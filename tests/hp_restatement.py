"""Plain-Python restatement of `nanopolish variants --fix-homopolymers` — test infrastructure (the checker of csrc/homopolymer.cu
and of the homopolymer calls built on it), never imported by the product.

Follows fix_homopolymers, src/nanopolish_call_variants.cpp:541-780, with the pieces it calls:
  Haplotype::apply_variant, substr_by_reference, get_enclosing_reference_range_for_haplotype_range,
  get_reference_position_for_haplotype_base                       src/nanopolish_haplotype.cpp:30-158
  AlignmentDB::get_event_subsequences (_find_by_ref_bounds + the event/bp ratio test)
                                                                  src/alignment/nanopolish_alignment_db.cpp:172-221, :688-731
  DurationModel::generate_aligned_durations, log_gamma_sum        src/hmm/nanopolish_duration_model.cpp:17-58
  Variant::add_info                                               src/common/nanopolish_variant.h:82-92
The forward score and the Viterbi path of every job come from the caller (the compiled reference's profile_hmm_score and
profile_hmm_align), and the device's likelihood vectors can stand in for the restated ones (call_and_apply)."""
import bisect
import ctypes as C
import ctypes.util
import math

import numpy as np

from nanopolish_b200 import synth
from tests import phase_restatement as pr

K = 6
MIN_HP, MAX_HP = 3, 9
SHAPE = 2.461964
MIN_DURATION = 0.00025
NPOS = (1 << 64) - 1
_LIBM = C.CDLL(ctypes.util.find_library("m"))
_LIBM.lgamma.restype = C.c_double
_LIBM.lgamma.argtypes = [C.c_double]
_LIBM.log.restype = C.c_double
_LIBM.log.argtypes = [C.c_double]


class RefAbort(Exception):
    """where the reference would trip an assert"""


class Haplotype:
    """nph::Haplotype / the reference's Haplotype: the sequence and, per base, its reference position (None: inserted)"""

    def __init__(self, ref_position: int, reference: str):
        self.ref_position, self.reference, self.seq = ref_position, reference, reference
        self.cmap = list(range(ref_position, ref_position + len(reference)))
        self.variants = []
        self._index = None

    def copy(self):
        h = Haplotype.__new__(Haplotype)
        h.ref_position, h.reference, h.seq, h.cmap, h.variants = self.ref_position, self.reference, self.seq, list(self.cmap), list(self.variants)
        h._index = None
        return h

    @property
    def ref_end(self):
        return self.ref_position + len(self.reference)

    def _lower_bound(self, r):
        """the first base with a reference position >= r (the reference's linear scan; the positions ascend, so a bisection
        over the bases that have one finds the same base)"""
        if self._index is None:
            self._index = ([c for c in self.cmap if c is not None], [i for i, c in enumerate(self.cmap) if c is not None])
        j = bisect.bisect_left(self._index[0], r)
        return self._index[1][j] if j < len(self._index[0]) else len(self.cmap)

    def apply_variant(self, pos, ref_seq, alt_seq, quality=0.0, info="") -> bool:
        i = self._lower_bound(pos)
        if i == len(self.cmap) or self.cmap[i] != pos or self.seq[i:i + len(ref_seq)] != ref_seq:
            return False
        self.seq = self.seq[:i] + alt_seq + self.seq[i + len(ref_seq):]
        self.cmap[i:i + len(ref_seq)] = [None] * len(alt_seq)
        self._index = None
        self.variants.append((pos, ref_seq, alt_seq, quality, info))
        return True

    def position_of(self, i):
        return self.cmap[i]

    def substr_by_reference(self, start, end):
        if not (self.ref_position <= start <= self.ref_end and self.ref_position <= end <= self.ref_end):
            raise RefAbort("substr_by_reference outside the haplotype")
        s, e = self._lower_bound(start), self._lower_bound(end)
        while s >= len(self.cmap) or self.cmap[s] is None or self.cmap[s] > start:
            if s == 0:
                raise RefAbort("substr_by_reference walks before the first base")
            s -= 1
        if e == len(self.cmap):
            raise RefAbort("substr_by_reference: end not in the haplotype")
        start, end = self.cmap[s], self.cmap[e]
        out = Haplotype(start, self.reference[start - self.ref_position:end + 1 - self.ref_position])
        out.seq, out.cmap = self.seq[s:e + 1], self.cmap[s:e + 1]
        return out

    def enclosing(self, lo, hi):
        """(lo, hi, ref_lo, ref_hi) after moving lo down and hi up over inserted bases, or None (npos)"""
        while lo > 0 and self.cmap[lo] is None:
            lo -= 1
        while hi < len(self.cmap) and self.cmap[hi] is None:
            hi += 1
        if lo == 0 or hi >= len(self.cmap):
            return None
        return lo, hi, self.cmap[lo], self.cmap[hi]


def windows(hap: Haplotype, region_start: int, region_end: int, min_flank: int, trace=None):
    """the homopolymers fix_homopolymers scores, in scan order: dicts with the run, the calling window and nph_hp_window's fields.
    trace (a list): gets (test, outcome, run start, run length) for every test a run meets, the scan's edges (see tests)"""
    s, n, i, out = hap.seq, len(hap.seq), 0, []
    t = trace.append if trace is not None else (lambda x: None)
    while i < n:
        b, start = s[i], i
        while i < n and s[i] == b:
            i += 1
        if i >= n:
            t(("last_run", True, start, i - start))
            break
        end, length = i, i - start
        t(("length", MIN_HP <= length <= MAX_HP, start, length))
        if length < MIN_HP or length > MAX_HP:
            continue
        t(("flank_lo", start >= min_flank, start - min_flank, length))
        if start < min_flank:
            continue
        t(("flank_hi", end + min_flank < n, end + min_flank - n, length))
        if end + min_flank >= n:
            continue
        r = hap.enclosing(start - min_flank, end + min_flank)
        t(("npos", r is None, start, length))
        if r is None:
            continue
        hcs, hce, rcs, rce = r
        t(("region_lo", rcs >= region_start, rcs - region_start, length))
        if rcs < region_start:
            continue
        t(("region_hi", rce < region_end, rce - region_end, length))
        if rce >= region_end or rcs < hap.ref_position or rce >= hap.ref_end:
            continue
        calling = hap.substr_by_reference(rcs, rce).seq
        out.append(dict(hp_start=start, hp_end=end, hp_length=length, hp_base=b, rcs=rcs, rce=rce, calling=calling,
                        edit_offset=start - hcs, k0=start - hcs - K + 1))
    return out


def window_array(wins):
    """(calling_seqs u1, HP_WINDOW_DT) of windows()"""
    w = np.zeros(len(wins), synth.HP_WINDOW_DT)
    buf, off = [], 0
    for i, x in enumerate(wins):
        w[i] = (off, len(x["calling"]), x["rcs"], x["rce"], x["edit_offset"], x["k0"], x["hp_length"], x["hp_base"].encode(), (0, 0, 0), K)
        buf.append(x["calling"].encode())
        off += len(x["calling"])
    return np.frombuffer(b"".join(buf) or b"\0", np.uint8).copy(), w


def event_sequences(records, pairs, rcs, rce, max_ratio=20):
    """get_event_subsequences: [(record, e1, e2)] in record order (max_ratio = inf: without the ratio test)"""
    out = []
    for r, R in enumerate(records):
        p = pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])]
        if p.shape[0] == 0:
            continue
        b = pr.find_by_ref_bounds([int(x) for x in p["ref_pos"]], [int(x) for x in p["read_pos"]], rcs, rce)
        if b is None:
            continue
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.float64(abs(b[0] - b[1])) / np.float64(abs(rce - rcs))
        if ratio < max_ratio:
            out.append((r, b[0], b[1]))
    return out


def variant_sequence(win, L):
    c, at, diff = win["calling"], win["edit_offset"], L - win["hp_length"]
    if diff < 0:
        return c[:at] + c[at - diff:]
    return c[:at] + win["hp_base"] * diff + c[at:]


def get_time(start_time, e):
    return np.float32(start_time[e] - start_time[0])


def likelihoods(win, seqs, reads, start_time, duration, score, align):
    """(event_lik[7], duration_lik[7]) of one window over its event sequences.  score(seq, r, e1, e2) -> float32,
    align(seq, r, e1, e2) -> [(event_idx, kmer_idx, state)] in the reference's vector order; start_time / duration per event"""
    e_lik, d_lik = [0.0] * 7, [0.0] * 7
    for r, e1, e2 in seqs:
        if abs(e1 - e2) < 10:
            continue
        off = int(reads[r]["event_off"])
        t = start_time[off:]
        local_time = float(abs(np.float32(get_time(t, e1) - get_time(t, e2))))
        local_avg = local_time / float(len(win["calling"]))
        rate = (1 / local_avg) * SHAPE if local_avg != 0 else math.inf
        for L in range(MIN_HP, MAX_HP + 1):
            v = variant_sequence(win, L)
            slots = [0.0] * (len(v) - K + 1)
            for ev, km, st in align(v, r, e1, e2):
                if st != "K":
                    slots[km] += float(duration[off + ev])
            e_lik[L - 3] += float(score(v, r, e1, e2))
            sum_duration = 0.0
            for k in range(win["k0"] + 2, win["k0"] + L + 2):
                sum_duration += slots[k]
            if sum_duration > MIN_DURATION:
                na = L * SHAPE
                g = (na * _LIBM.log(rate)) - _LIBM.lgamma(na) + (na - 1) * _LIBM.log(sum_duration) - rate * sum_duration
            else:
                g = 0.0
            d_lik[L - 3] += g
    return e_lik, d_lik


def call_rule(hp_length, e_lik, d_lik):
    """(call, quality, size_diff, kept) of :686-727: the first strict maximum from -inf (call stays npos when nothing beats it),
    max - score[hp_length], kept unless < 10 (a NaN is kept), size_diff = int(call - hp_length)"""
    max_score, call = -math.inf, NPOS
    score_by = {}
    for L in range(MIN_HP, MAX_HP + 1):
        s = d_lik[L - 3] + e_lik[L - 3]
        score_by[L] = s
        if s > max_score:
            max_score, call = s, L
    score = max_score - score_by[hp_length]
    size_diff = (call - hp_length) & 0xffffffff
    size_diff = size_diff - (1 << 32) if size_diff >= 1 << 31 else size_diff
    return call, score, size_diff, not score < 10


def call_and_apply(hap: Haplotype, fixed: Haplotype, win, total_reads, e_lik, d_lik, trace=None):
    """the call of :686-777 on one window's vectors, applied to `fixed` (positions from `hap`, the input haplotype).  trace (a
    list): gets ("call", call, quality, size_diff) and ("tries", positions tried before the one applied or the last, applied)"""
    call, score, size_diff, kept = call_rule(win["hp_length"], e_lik, d_lik)
    if trace is not None:
        trace.append(("call", call, score, size_diff))
    if not kept:
        return
    info = f"TotalReads={total_reads};AlleleCount=1"
    b = win["hp_base"]
    tried = 0
    for k in range(win["hp_start"], win["hp_end"] + 1):
        if size_diff == 0:
            break
        p = hap.position_of(k)
        if p is not None:
            if size_diff > 0:
                ref_seq = fixed.substr_by_reference(p, p).seq
                if len(ref_seq) == 1 and ref_seq == b and fixed.apply_variant(p, ref_seq, ref_seq + b, score, info):
                    break
            else:
                ref_seq = fixed.substr_by_reference(p, p + 1).seq
                if len(ref_seq) == 2 and ref_seq == b + b and fixed.apply_variant(p, ref_seq, ref_seq[0], score, info):
                    break
        tried += 1
    if trace is not None and size_diff != 0:
        trace.append(("tries", tried, tried <= win["hp_end"] - win["hp_start"]))


def duration_decides(win, e_lik, d_lik) -> bool:
    """the call is made (quality >= 10) and the event likelihoods alone would not make it: another length, or a quality below 10"""
    def call(v):
        best = max(range(7), key=lambda i: (v[i], -i))
        return best, v[best] - v[win["hp_length"] - 3]
    both, q = call([d + e for d, e in zip(d_lik, e_lik)])
    ev, qe = call(list(e_lik))
    return q >= 10 and (ev != both or qe < 10)


def fix_homopolymers(hap: Haplotype, wins, vectors, trace=None):
    """the fixed haplotype from the windows and their (total_reads, e_lik, d_lik)"""
    fixed = hap.copy()
    for w, (n, e, d) in zip(wins, vectors):
        call_and_apply(hap, fixed, w, n, e, d, trace)
    return fixed


def qbits(q: float) -> str:
    return format(int(np.float64(q).view(np.uint64)), "016x")


def fixed_text(fixed: Haplotype, n_input: int) -> str:
    """the fixed sequence and its new variants in npref_fix_homopolymers' format"""
    return fixed.seq + "\n" + "".join(f"{p}\t{r}\t{a}\t{qbits(q)}\t{i}\n" for p, r, a, q, i in fixed.variants[n_input:])
