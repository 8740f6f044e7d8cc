"""call-methylation cases shared by the CPU pin (tests/test_oracle_vs_ref.py: restatement == compiled reference) and the GPU
test (tests/test_gpu_methylation.py: device == compiled reference): synthetic reads aligned to a contig with a CIGAR that has
insertions, deletions and soft clips, forward and reverse strand — everything calculate_methylation_for_read reads
(src/basemods/nanopolish_basemods.cpp:238-457) built the way the BAM / FASTA / SquiggleRead would present it."""
import numpy as np

from nanopolish_b200 import synth
from oracle import eventalign_py as ea

K = 6
_COMP = str.maketrans("ACGT", "TGCA")


def revcomp(s):
    return s.translate(_COMP)[::-1]


def make_case(i, rs, rng, contig_pad=300):
    """read i of `rs` -> dict(read_sequence, b2e_start, b2e_stop, contig, ref_pos, flag, cigar, ...).
    The BAM query (what the CIGAR walks) is the read sequence, reverse complemented for flag 16; the contig is that query
    with the CIGAR's deletions inserted / insertions removed, between random flanks."""
    codes = rs.seq_codes[i]
    read_seq = synth._CODE2DNA[codes].tobytes().decode()
    nk = codes.shape[0] - K + 1
    which = rs.ev_kmer[i]
    first = np.searchsorted(which, np.arange(nk), side="left")
    last = np.searchsorted(which, np.arange(nk), side="right") - 1
    b2e_start = np.where(last >= first, first, -1).astype(np.int32)
    b2e_stop = np.where(last >= first, last, -1).astype(np.int32)
    rev = (i % 3 == 2)
    query = revcomp(read_seq) if rev else read_seq
    # CIGAR: soft clip, long matches broken by a 2-base deletion, a 3-base insertion, a 1-base deletion
    L = len(query)
    ops, ref_parts, q = [], [], 0
    def M(n):
        nonlocal q
        ops.append((n, 'M')); ref_parts.append(query[q:q + n]); q += n
    def I(n):
        nonlocal q
        ops.append((n, 'I')); q += n
    def D(n):
        ops.append((n, 'D')); ref_parts.append("".join("ACGT"[x] for x in rng.integers(0, 4, n)))
    def S(n):
        nonlocal q
        ops.append((n, 'S')); q += n
    S(7)
    seg = (L - 7 - 5 - 3) // 4
    M(seg); D(2); M(seg); I(3); M(seg); D(1); M(L - 7 - 5 - 3 - 3 * seg)
    S(5)
    assert q == L
    ref_body = "".join(ref_parts)
    left = "".join("ACGT"[x] for x in rng.integers(0, 4, contig_pad))
    right = "".join("ACGT"[x] for x in rng.integers(0, 4, contig_pad))
    contig = left + ref_body + right
    # a few IUPAC / lower-case bases in the fetched region: disambiguate() must deal with them
    cl = list(contig)
    for p in rng.integers(contig_pad + 50, contig_pad + len(ref_body) - 50, 4):
        cl[int(p)] = "acgtRYN"[int(rng.integers(0, 7))]
    contig = "".join(cl)
    return dict(read_sequence=read_seq, b2e_start=b2e_start, b2e_stop=b2e_stop, contig=contig, ref_pos=contig_pad,
                flag=16 if rev else 0, cigar=ea.pack_cigar(ops), name=f"read_{i}", ref_len=len(ref_body))


def event_alignment_record(case, k=K):
    """EventAlignmentRecord (src/alignment/nanopolish_alignment_db.cpp:50-91) for strand 0 -> (pairs [(ref_pos, event_idx)], rc)"""
    segs = ea.get_aligned_segments(case["ref_pos"], case["cigar"])
    assert len(segs) == 1
    rev = bool(case["flag"] & 16)
    read_length = len(case["read_sequence"])
    b2e = case["b2e_start"]
    def next_event(start, stop, stride):
        while start != stop:
            if b2e[start] != -1:
                return int(b2e[start])
            start += stride
        return -1
    out = []
    for ref_pos, read_pos in segs[0]:
        if read_pos < k or read_pos + k >= read_length:
            continue
        kp = read_length - read_pos - k if rev else read_pos
        before = next_event(kp, max(0, kp - 1000), -1)
        after = next_event(kp, min(kp + 1000, len(b2e) - 1), 1)
        out.append((ref_pos, after if before == -1 else before))
    if out and out[0][1] == out[-1][1]:
        out = []
    return out, (1 if rev else 0)


def fetched_reference(case):
    """get_reference_region_ts(fai, contig, pos, bam_endpos) -> gDNAAlphabet.disambiguate (faidx's end is inclusive)"""
    end = case["ref_pos"] + case["ref_len"]                    # bam_endpos
    return ea.disambiguate(case["contig"][case["ref_pos"]:end + 1])


def tsv_rows(contig_name, strand_char, read_name, rows):
    """write_methylation_results_as_tsv: rows = [(start, end, n_motif, ll_u float32, ll_m float32, sequence)]"""
    out = []
    for (sp, ep, nm, ll_u, ll_m, seq) in rows:
        m, u = float(ll_m) + 0.0, float(ll_u) + 0.0
        out.append("%s\t%s\t%d\t%d\t%s\t%.2f\t%.2f\t%.2f\t%d\t%d\t%s\n" % (contig_name, strand_char, sp, ep, read_name, m - u, m, u, 1, nm, seq))
    return "".join(out)


def expected_rows(sites, site_off, recs, ref, names, is_rev, contig, k):
    """the reference's writer (src/nanopolish_call_methylation.cpp:113-140) over site records, formatted by Python's correctly
    rounded %.2f — the C library's %.2lf"""
    out = []
    for r in range(recs.shape[0]):
        R = recs[r]
        seg = ref[int(R["ref_off"]):int(R["ref_off"]) + int(R["ref_len"])].tobytes().decode()
        for s in sites[int(site_off[r]):int(site_off[r + 1])]:
            ll_m, ll_u = float(s["ll_methylated"]) + 0.0, float(s["ll_unmethylated"]) + 0.0
            b = int(s["start_position"]) - int(R["ref_start_pos"]) - k + 1
            e = min(int(s["end_position"]) - int(R["ref_start_pos"]) + k, int(R["ref_len"]))
            out.append("%s\t%s\t%d\t%d\t%s\t%.2f\t%.2f\t%.2f\t%d\t%d\t%s\n" % (
                contig, "-" if is_rev[r] else "+", int(s["start_position"]), int(s["end_position"]), names[r], ll_m - ll_u, ll_m, ll_u, 1,
                int(s["n_motif"]), seg[b:e]))
    return "".join(out)
