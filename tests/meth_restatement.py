"""Plain-Python restatement of call-methylation's per-read enumeration — test infrastructure (the checker of
csrc/methylation.cu and the expectation of the host caller's TSV), never imported by the product.

Follows calculate_methylation_for_read, src/basemods/nanopolish_basemods.cpp:301-417, with the pieces it calls:
  Alphabet::match_to_site / is_motif_match / methylate / reverse_complement   src/common/nanopolish_alphabet.h:108-330
  AlignmentDB::_find_by_ref_bounds                                            src/alignment/nanopolish_alignment_db.cpp:688-731
  HMMInputSequence::get_kmer_rank                                             src/hmm/nanopolish_hmm_input_sequence.h:76-91
Pinned: tests/test_oracle_vs_ref.py runs it against the compiled reference's own calculate_methylation_for_read."""
import bisect

import numpy as np

from nanopolish_b200 import synth

ALPHABETS = {name: dict(bases=v[0].decode(), comp=v[1].decode(), sites=[s.decode() for s in v[2]], sites_m=[s.decode() for s in v[3]],
                        sites_mc=[s.decode() for s in v[4]]) for name, v in synth._METH_ALPHABETS.items()}
METHYLATED_SYMBOL = "M"


def match_to_site(s, i, site, rl):
    """nanopolish_alphabet.h:108-143 -> (offset, length, covers_methylated_site)"""
    offset = length = 0
    p = site.find(s) if i == 0 else -1            # strstr(site, str): the whole string inside the site, only asked at i == 0
    if p != -1:
        offset, length = p, len(s)
    else:
        cl = min(rl, len(s) - i)
        if s[i:i + cl] == site[:cl]:
            offset, length = 0, cl
    covers = length > 0 and METHYLATED_SYMBOL in s[i:i + length]
    return offset, length, covers


def is_motif_match(a, s, i):
    rl = len(a["sites"][0])
    return any(match_to_site(s, i, site, rl)[1] == rl for site in a["sites"])


def methylate(a, s):
    rl = len(a["sites"][0])
    out = list(s)
    i = 0
    while i < len(s):
        stride = 1
        for site, site_m in zip(a["sites"], a["sites_m"]):
            if match_to_site(s, i, site, rl)[1] == rl:
                out[i:i + rl] = list(site_m)
                stride = rl
                break
        i += stride
    return "".join(out)


def reverse_complement(a, s):
    rl = len(a["sites"][0]) if a["sites"] else 0
    comp = {b: c for b, c in zip(a["bases"], a["comp"])}
    out = [None] * len(s)
    i, j = 0, len(s) - 1
    while i < len(s):
        hit = None
        for si, site_m in enumerate(a["sites_m"]):
            off, ln, cov = match_to_site(s, i, site_m, rl)
            if ln > 0 and cov:
                hit = (si, off, ln)
                break
        if hit:
            si, off, ln = hit
            for t in range(off, off + ln):
                out[j] = a["sites_mc"][si][t]
                j -= 1
                i += 1
        else:
            out[j] = comp[s[i]]
            j -= 1
            i += 1
    return "".join(out)


def kmer_ranks(a, seq, rc_seq, k, rc):
    """get_kmer_rank(i, k, rc) for i = 0..len-k"""
    rank = {b: i for i, b in enumerate(a["bases"])}
    n = len(seq) - k + 1
    A = len(a["bases"])
    out = np.zeros(max(n, 0), np.uint32)
    for i in range(n):
        km = seq[i:i + k] if not rc else rc_seq[len(seq) - i - k:len(seq) - i]
        r = 0
        for ch in km:
            r = r * A + rank[ch]
        out[i] = r
    return out


def find_by_ref_bounds(ref_pos, read_pos, ref_start, ref_stop):
    i, j = bisect.bisect_left(ref_pos, ref_start), bisect.bisect_left(ref_pos, ref_stop)
    if i == len(ref_pos) or j == len(ref_pos):
        return None
    left = ref_pos[i] <= ref_start or (i > 0 and ref_pos[i - 1] <= ref_start)
    # right_bounded: ref_pos[j] >= ref_stop always holds for a lower_bound that is not end()
    if not left:
        return None
    return int(read_pos[i]), int(read_pos[j])


def enumerate_record(ref, ref_start_pos, pr_ref, pr_read, rc, alphabet, k, min_separation=10, min_flank=10, max_span=200,
                     min_event_span=10, region_start=-1, region_end=-1):
    """-> list of (start_position, end_position, n_motif, e1, e2, ranks_u, ranks_m, site_sequence)"""
    a = ALPHABETS[alphabet]
    motif_sites = [i for i in range(len(ref) - 1) if is_motif_match(a, ref, i)] if len(ref) else []
    groups, cur = [], 0
    while cur < len(motif_sites):
        end = cur + 1
        while end < len(motif_sites) and motif_sites[end] - motif_sites[end - 1] <= min_separation:
            end += 1
        groups.append((cur, end)); cur = end
    out = []
    for gs, ge in groups:
        first, last = motif_sites[gs], motif_sites[ge - 1]
        sub_start, sub_end, span = first - min_flank, last + min_flank, last - first
        if sub_start <= min_separation or span > max_span:
            continue
        subseq = ref[sub_start:sub_end + 1]                       # substr: cut at the end of the string
        b = find_by_ref_bounds(pr_ref, pr_read, sub_start + ref_start_pos, sub_end + ref_start_pos)
        if b is None or abs(b[1] - b[0]) <= min_event_span:
            continue
        start_position, end_position = first + ref_start_pos, last + ref_start_pos
        if (region_start != -1 and start_position < region_start) or (region_end != -1 and end_position >= region_end):
            continue
        m_subseq = methylate(a, subseq)
        ru = kmer_ranks(a, subseq, reverse_complement(a, subseq), k, rc)
        rm = kmer_ranks(a, m_subseq, reverse_complement(a, m_subseq), k, rc)
        out.append((start_position, end_position, ge - gs, b[0], b[1], ru, rm, ref[first - k + 1:last + k]))
    return out


def enumerate_batch(ref_bases, pairs, records, alphabet, k, **kw):
    """-> (rows [(record, start, end, n_motif)], jobs HMM_JOB_DT[2 * n], ranks u4[]) in the device's order"""
    rows, jrows, ranks_list = [], [], []
    flags = synth.HAF_ALLOW_PRE_CLIP | synth.HAF_ALLOW_POST_CLIP
    for ri, R in enumerate(records):
        ref = ref_bases[int(R["ref_off"]):int(R["ref_off"]) + int(R["ref_len"])].tobytes().decode()
        pr = pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])]
        for (sp, ep, nm, e1, e2, ru, rm, _seq) in enumerate_record(ref, int(R["ref_start_pos"]), pr["ref_pos"].tolist(), pr["read_pos"].tolist(),
                                                                   int(R["rc"]), alphabet, k, **kw):
            rows.append((ri, sp, ep, nm))
            for r in (ru, rm):
                jrows.append((int(R["read"]), int(R["model_id"]), e1, e2, int(R["rc"]), flags))
                ranks_list.append(r)
    jobs = np.zeros(len(jrows), synth.HMM_JOB_DT)
    off = 0
    for j, (read, mid, e1, e2, rc, fl) in enumerate(jrows):
        nk = ranks_list[j].shape[0]
        jobs[j] = (off, read, mid, e1, e2, nk, 1 if e1 <= e2 else -1, rc, fl, 0)
        off += nk
    ranks = np.concatenate(ranks_list).astype(np.uint32) if ranks_list else np.zeros(0, np.uint32)
    return rows, jobs, ranks
