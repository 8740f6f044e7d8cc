"""Plain-Python restatement of screen_variants_by_score and expand_variants of `nanopolish variants --consensus` — test
infrastructure (the checker of csrc/screen_variants.cu and of the host mirror built on it), never imported by the product.

Follows src/nanopolish_call_variants.cpp:364-450 with the pieces it calls:
  AlignmentDB::are_coordinates_valid, get_reference_substring     src/alignment/nanopolish_alignment_db.cpp:119-141
  Haplotype::apply_variant on a fresh window                      src/nanopolish_haplotype.cpp:33-75
  AlignmentDB::get_event_subsequences                             src/alignment/nanopolish_alignment_db.cpp:172-221 (tests/hp_restatement.py)
  score_variant_thresholded with opt::methylation_types           src/common/nanopolish_variant.cpp:765-799 (its sets and fold:
                                                                  tests/var_meth_restatement.py), on one thread
The forward scores come from the caller: the compiled reference's own profile_hmm_score, or the device's nph_hmm_score_batch."""
import math

import numpy as np

from tests import hp_restatement as hr
from tests import var_meth_restatement as vmr

SCREENED, OUTSIDE, NOT_APPLIED = 0, 1, 2


def window(region_start: int, region_ref: str, ref_position: int, ref_seq: str, flank: int):
    """(calling_start, calling_end, the window's bases), or None where are_coordinates_valid fails (the reference skips the candidate)"""
    cs, ce = ref_position - flank, ref_position + len(ref_seq) + flank
    if cs < region_start or ce > region_start + len(region_ref) - 1:
        return None
    return cs, ce, region_ref[cs - region_start:ce - region_start + 1]


def variant_haplotype(win: str, flank: int, ref_seq: str, alt_seq: str):
    """(apply_variant's sequence on a fresh window, whether it applied): the window's bases at flank are compared byte for byte"""
    if win[flank:flank + len(ref_seq)] == ref_seq:
        return win[:flank] + alt_seq + win[flank + len(ref_seq):], True
    return win, False


def event_sequences(lists, cs, ce):
    """hr.event_sequences over pair lists made once: a record can bound [cs, ce] only if its first aligned base is at or before ce and
    its last at or after ce (otherwise a lower bound is missing, or the window is not left-bounded)"""
    out = []
    for r, (ref, read) in enumerate(lists):
        if not ref or ref[0] > ce or ref[-1] < ce:
            continue
        b = hr.pr.find_by_ref_bounds(ref, read, cs, ce)
        if b is None:
            continue
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.float64(abs(b[0] - b[1])) / np.float64(abs(ce - cs))
        if ratio < 20:
            out.append((r, b[0], b[1]))
    return out


def plan(region_start, region_ref, records, pairs, candidates, flank, types):
    """per candidate None (outside the region) or (status, base set, variant set, event sequences [(record, e1, e2)]); a set is
    [(type index or -1, string)] as generate_methylated_alternatives makes it"""
    lists = [([int(x) for x in p["ref_pos"]], [int(x) for x in p["read_pos"]])
             for p in (pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])] for R in records)]
    out = []
    for p, r, a in candidates:
        w = window(region_start, region_ref, p, r, flank)
        if w is None:
            out.append(None)
            continue
        cs, ce, win = w
        var, applied = variant_haplotype(win, flank, r, a)
        out.append((SCREENED if applied else NOT_APPLIED, vmr.alternatives(win, types), vmr.alternatives(var, types),
                    event_sequences(lists, cs, ce)))
    return out


def accumulate(base_scores, var_scores, ev, threshold):
    """score_variant_thresholded's loop over the event sequences in read order: (quality, the reference's DP rows).  base_scores[j],
    var_scores[j]: the float32 scores of read j's base and variant sets, in set order"""
    total, rows = 0.0, 0
    for (r, e1, e2), b, v in zip(ev, base_scores, var_scores):
        if abs(total) < threshold:
            total += float(vmr.score_set(v)) - float(vmr.score_set(b))
            rows += (len(b) + len(v)) * (abs(e1 - e2) + 1)
    return total, rows


def screened(pl, score_set_jobs, threshold):
    """per candidate (quality f8, n_reads, status, the reference's DP rows).  score_set_jobs(requests) -> float32 scores, one per
    request (record, e1, e2, type index or -1, sequence); every set of every candidate and read is asked (no early exit)"""
    reqs = []
    for x in pl:
        if x is None or x[0] != SCREENED:
            continue
        _, bs, vs, ev = x
        for rec, e1, e2 in ev:
            reqs += [(rec, e1, e2, t, s) for t, s in bs + vs]
    scores = score_set_jobs(reqs) if reqs else np.zeros(0, np.float32)
    out, j = [], 0
    for x in pl:
        if x is None:
            out.append((math.nan, 0, OUTSIDE, 0))
            continue
        st, bs, vs, ev = x
        if st == NOT_APPLIED:
            rows = sum(2 * len(bs) * (abs(e1 - e2) + 1) for _, e1, e2 in ev) if threshold > 0 else 0
            out.append((0.0, len(ev), NOT_APPLIED, rows))
            continue
        b_sc, v_sc = [], []
        for _ in ev:
            b_sc.append(scores[j:j + len(bs)]); j += len(bs)
            v_sc.append(scores[j:j + len(vs)]); j += len(vs)
        q, rows = accumulate(b_sc, v_sc, ev, threshold)
        out.append((q, len(ev), SCREENED, rows))
    return out


def quality_hex(q: float) -> str:
    return "%016x" % int(np.float64(q).view(np.uint64))


def kept_lines(candidates, results):
    """screen_variants_by_score's output list as the harness writes it: the candidates with quality > 0, INFO cleared"""
    return [f"{p}\t{r}\t{a}\t{quality_hex(q)}\t" for (p, r, a), (q, _, st, _) in zip(candidates, results) if st != OUTSIDE and q > 0]


def expand(contig, region_start, region_ref, candidates, min_flanking_sequence, var_contig=None):
    """expand_variants: [(ref_position, ref_seq, alt_seq)]; hr.RefAbort where the reference asserts"""
    region_end = region_start + len(region_ref) - 1
    out = []
    for p, r, a in candidates:
        out.append((p, r, a))
        if len(r) == 1 and len(a) == 1:
            continue
        end = p + len(r)
        if (var_contig or contig) == contig and p >= region_start and end <= region_end and region_end - end > min_flanking_sequence:
            d = region_ref[p - region_start:end - region_start + 1]
            if d[:len(r)] != r:
                raise hr.RefAbort("expand_variants: the extended deletion does not start with ref_seq")
            out.append((p, d, a))
        for b in "ACGT":
            out.append((p, r, a + b))
    return out
