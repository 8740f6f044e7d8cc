"""Plain-Python restatement of `nanopolish variants` candidate screening — test infrastructure (the checker of csrc/variants.cu).

Follows generate_candidate_single_base_edits (src/nanopolish_call_variants.cpp:288-361), AlignmentDB::get_event_subsequences
(src/alignment/nanopolish_alignment_db.cpp:172-221) and score_variant_thresholded (src/common/nanopolish_variant.cpp:765-799, the
single-thread order).  Pinned: tests/test_oracle_vs_ref.py runs its qualities against the compiled reference's score_variant_thresholded."""
import math

import numpy as np

from nanopolish_b200 import synth
from tests.meth_restatement import find_by_ref_bounds

BASES = "ACGT"


def candidates(ref: str, i0: int):
    """the Variants of position i (offset i0 into ref) in the order the reference generates them: (slot, ref_position offset, ref_seq, alt_seq)"""
    out = []
    b = ref[i0]
    for j in range(4):
        if BASES[j] != b:
            out.append((2 * j, i0, b, BASES[j]))                       # substitution
        if BASES[j] != b:
            out.append((2 * j + 1, i0, b, b + BASES[j]))               # insertion ("A" -> "AA" is redundant)
    if ref[i0 - 1] != ref[i0]:
        out.append((8, i0 - 1, ref[i0 - 1:i0 + 1], ref[i0 - 1]))       # deletion ("AA" -> "A" is redundant)
    return out


def pair_lists(records, pairs):
    """per record its aligned_events as (ref_pos list, read_pos list)"""
    out = []
    for R in records:
        pr = pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])]
        out.append((pr["ref_pos"].tolist(), pr["read_pos"].tolist()))
    return out


def event_sequences(records, pairs, cs, ce, lists=None):
    """get_event_subsequences: [(record index, e1, e2)] in record order (lists: pair_lists(records, pairs), computed once by callers
    that ask for many windows)"""
    out = []
    for r, (ref_pos, read_pos) in enumerate(lists if lists is not None else pair_lists(records, pairs)):
        if not ref_pos:
            continue
        b = find_by_ref_bounds(ref_pos, read_pos, cs, ce)
        if b is None:
            continue
        if abs(b[0] - b[1]) / abs(ce - cs) < 20:
            out.append((r, b[0], b[1]))
    return out


def apply(window: str, off: int, ref_seq: str, alt_seq: str) -> str:
    assert window[off:off + len(ref_seq)] == ref_seq
    return window[:off] + alt_seq + window[off + len(ref_seq):]


def position_scores(port_oracle, rs, model, ref: str, region_start: int, positions, records, pairs, flank=10, flags=0, indel_bias=1.0, k=6,
                    threads=1):
    """The oracle's profile_hmm_score of every (event sequence, haplotype) pair the reference's loop may score, for each position i of
    `positions`: None where the window leaves the region (the reference skips the position), else (candidates, event sequences,
    scores f4[n_sequences, 1 + n_candidates]: per event sequence the base haplotype, then the candidates in generation order).
    All positions go to the oracle as one batch."""
    n_ref = len(ref)
    lists = pair_lists(records, pairs)
    out, rows, ranks_list = [], [], []
    for i in positions:
        cs, ce = i - flank, i + 1 + flank
        if cs < region_start or ce > region_start + n_ref - 1:
            out.append(None)
            continue
        window = ref[cs - region_start:ce - region_start + 1]
        seqs = event_sequences(records, pairs, cs, ce, lists)
        cands = candidates(ref, i - region_start)
        hap = [window] + [apply(window, off - (cs - region_start), rseq, aseq) for (_, off, rseq, aseq) in cands]
        codes = [synth.encode(h, "nucleotide") for h in hap]
        fw = [synth.kmer_ranks_from_codes(c, k, 4) for c in codes]
        rv = [synth.dna_rc_kmer_ranks(c, k) for c in codes]
        for (r, e1, e2) in seqs:
            rc = int(records[r]["rc"])
            ranks_list += rv if rc else fw
            rows += [(int(records[r]["read"]), 0, e1, e2, rc, flags)] * len(hap)
        out.append((cands, seqs, len(hap)))
    sc = np.zeros(0, np.float32)
    if rows:
        jobs = synth._finish_jobs(rows, ranks_list)
        jobs.jobs["stride"] = np.where(jobs.jobs["rc"] == 1, -1, 1)          # EventAlignmentRecord::stride
        sc, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [model], jobs.kmer_ranks, jobs.jobs, indel_bias=indel_bias,
                                            threads=threads)
    at = 0
    for n, o in enumerate(out):
        if o is not None:
            cands, seqs, nh = o
            out[n] = (cands, seqs, sc[at:at + len(seqs) * nh].reshape(len(seqs), nh))
            at += len(seqs) * nh
    return out


def accumulate(cands, seqs, scores, threshold):
    """score_variant_thresholded's loop over the event sequences in order ->
    (qualities[9] with NaN for candidates the reference does not generate,
     DP rows the loop scores: 2 E for each (candidate, sequence) pair it adds, the base and the variant haplotype,
     event sequences read until the last candidate has left the threshold: all of them if one never does)"""
    q = [math.nan] * 9
    totals = [0.0] * len(cands)
    rows = used = 0
    for ri, (r, e1, e2) in enumerate(seqs):
        if all(abs(t) >= threshold for t in totals):
            break
        used = ri + 1
        base = float(scores[ri, 0])
        for c in range(len(cands)):
            if abs(totals[c]) < threshold:
                totals[c] += float(scores[ri, 1 + c]) - base
                rows += 2 * (abs(e1 - e2) + 1)
    for (slot, _, _, _), t in zip(cands, totals):
        q[slot] = t
    return q, rows, used


def screen_position(port_oracle, rs, model, ref: str, region_start: int, i: int, records, pairs, flank=10, threshold=100, flags=0, indel_bias=1.0, k=6):
    """-> (qualities[9] with NaN for candidates the reference does not generate, number of event sequences, the windows' (record, e1, e2))"""
    got = position_scores(port_oracle, rs, model, ref, region_start, [i], records, pairs, flank, flags, indel_bias, k)[0]
    if got is None:
        return [math.nan] * 9, 0, []
    cands, seqs, scores = got
    return accumulate(cands, seqs, scores, threshold)[0], len(seqs), seqs
