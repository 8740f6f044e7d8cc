"""Plain-Python restatement of phase-reads' per-read variant loop — test infrastructure (the checker of csrc/phase_reads.cu),
never imported by the product.

Follows phase_single_read, src/nanopolish_phase_reads.cpp:178-347, with the pieces it calls:
  lower_bound / upper_bound under sortByPosition                 src/common/nanopolish_variant.h:106-111
  AlignmentDB::_find_by_ref_bounds                               src/alignment/nanopolish_alignment_db.cpp:688-731
  EventAlignmentRecord::stride                                   src/alignment/nanopolish_alignment_db.cpp:82
  Haplotype::apply_variant on the calling window                 src/nanopolish_haplotype.cpp:30-85
  HMMInputSequence::get_kmer_rank (DNA alphabet)                 src/hmm/nanopolish_hmm_input_sequence.h:76-91
  add_logs = p7_FLogsum and the quality arithmetic               src/common/logsum.h:55-66, nanopolish_phase_reads.cpp:293-317
The two forward scores per site come from the caller (the oracle)."""
import bisect
import math

import numpy as np

from nanopolish_b200 import synth

FLANK = 30                       # opt::min_flanking_sequence
WIN = 2 * FLANK + 1
_RANK = {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3}
_TBL = np.array([np.float32(math.log(1.0 + math.exp(-i / 1000.0))) for i in range(16000)], np.float32)   # p7_FLogsumInit
_LN10 = math.log(10)


def find_by_ref_bounds(ref_pos, read_pos, start, stop):
    """(e1, e2) or None: the two lower_bounds on the (ascending) ref_pos list and the left/right bound tests."""
    n = len(ref_pos)
    i = bisect.bisect_left(ref_pos, start)
    j = bisect.bisect_left(ref_pos, stop)
    if i == n or j == n:
        return None
    left = ref_pos[i] <= start or (i != 0 and ref_pos[i - 1] <= start)
    right = ref_pos[j] >= stop or (j + 1 < n and ref_pos[j + 1] >= start)
    return (read_pos[i], read_pos[j]) if left and right else None


def kmer_ranks(window: bytes, k: int, rc: bool):
    codes = [_RANK.get(c, 0) for c in window]
    out = []
    for q in range(len(codes) - k + 1):
        r = 0
        for t in range(k):
            r = r * 4 + ((3 - codes[q + k - 1 - t]) if rc else codes[q + t])
        out.append(r)
    return out


def add_logs(a: float, b: float) -> np.float32:
    """p7_FLogsum(a, b) on floats"""
    a, b = np.float32(a), np.float32(b)
    mx = a if a > b else b
    mn = a if a < b else b
    d = np.float32(mx - mn)
    if mn == -np.inf or not d < np.float32(15.7):
        return mx
    return np.float32(mx + _TBL[int(np.float32(d * np.float32(1000.0)))])


def quality(ref: float, alt: float, ref_base: bytes, alt_base: bytes):
    """(call byte, q_char) of :293-317"""
    log_sum = float(add_logs(alt, ref))
    is_alt = float(alt) > float(ref)
    log_p_wrong = (float(ref) if is_alt else float(alt)) - log_sum
    q = -10 * log_p_wrong / _LN10
    q = q if q < 30.0 else 30.0                   # std::min(MAX_Q_SCORE, q): a NaN q gives 30
    return (alt_base if is_alt else ref_base), int(q) + 33


def var_ranges(positions, records):
    """per record [lower_bound(ref_start_pos), upper_bound(bam_endpos)) in the sorted positions (one contig); bam_endpos is the
    last base of the fetched reference (faidx fetches [pos, endpos] inclusive)"""
    out = np.zeros((records.shape[0], 2), np.uint32)
    pos = list(int(p) for p in positions)
    for r, R in enumerate(records):
        lo = bisect.bisect_left(pos, int(R["ref_start_pos"]))
        hi = bisect.bisect_right(pos, int(R["ref_start_pos"]) + int(R["ref_len"]) - 1)
        out[r] = (lo, max(lo, hi))
    return out


def enumerate_batch(ref_bases, pairs, records, variants, var_range, k):
    """-> (sites [(record, variant)], jobs HMM_JOB_DT, ranks u4, windows [bytes]): two jobs per scored site, reference window first"""
    sites, jobs, ranks, windows = [], [], [], []
    n_ranks = 0
    for r, R in enumerate(records):
        pr = pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])]
        ref_pos = [int(x) for x in pr["ref_pos"]]
        read_pos = [int(x) for x in pr["read_pos"]]
        stride = (1 if read_pos[0] < read_pos[-1] else -1) if read_pos else 1
        rs = int(R["ref_start_pos"])
        ref = bytes(ref_bases[int(R["ref_off"]):int(R["ref_off"]) + int(R["ref_len"])])
        rc = bool(R["rc"])
        for v in range(int(var_range[r][0]), int(var_range[r][1])):
            V = variants[v]
            if not V["is_snp"]:
                continue
            p = int(V["ref_position"])
            b = find_by_ref_bounds(ref_pos, read_pos, p - FLANK, p + FLANK)
            if b is None:
                continue
            win = ref[p - FLANK - rs:p + FLANK + 1 - rs]
            if win[FLANK:FLANK + 1] != V["ref_base"]:
                continue                               # apply_variant fails: no call
            alt = win[:FLANK] + V["alt_base"] + win[FLANK + 1:]
            for w in (win, alt):
                rk = kmer_ranks(w, k, rc)
                jobs.append((n_ranks, int(R["read"]), int(R["model_id"]), b[0], b[1], len(rk), stride, int(rc),
                             synth.HAF_ALLOW_PRE_CLIP | synth.HAF_ALLOW_POST_CLIP, 0))
                ranks.append(rk)
                n_ranks += len(rk)
                windows.append(w)
            sites.append((r, v))
    jb = np.array(jobs, synth.HMM_JOB_DT) if jobs else np.zeros(0, synth.HMM_JOB_DT)
    rk = np.array([x for r in ranks for x in r], np.uint32)
    return sites, jb, rk, windows


def expected_calls(sites, scores, variants, n_records):
    """(call_off u8[n_records + 1], calls PHASE_CALL_DT) from the sites and their oracle scores"""
    calls = np.zeros(len(sites), synth.PHASE_CALL_DT)
    off = np.zeros(n_records + 1, np.uint64)
    for i, (r, v) in enumerate(sites):
        ref, alt = scores[2 * i], scores[2 * i + 1]
        c, q = quality(ref, alt, variants[v]["ref_base"], variants[v]["alt_base"])
        calls[i] = (r, v, ref, alt, c, q, (0, 0))
        off[r + 1] += 1
    return np.cumsum(off).astype(np.uint64), calls
