"""call_haplotype_from_candidates (src/nanopolish_call_variants.cpp:782-880) restated in Python over any profile_hmm_score — test
infrastructure.

restated(...) groups the candidates, builds each group's combinations with a small Haplotype, collects each window's event sequences
(tests/hp_restatement.py), asks `score` for every (event sequence, haplotype, alternative) and then runs score_variant_group's
VariantGroup bookkeeping and simple_call on the float32 scores: the genotype search vectorised over the sets (each set's keys are still
summed one after another, in key order), the supports with math.exp (the C library's exp), the INFO fields with the C library's
"%g", and its own restatement of kt_fisher_exact.  SupportFractionByBase (--calculate-all-support) is not restated."""
import ctypes
import ctypes.util
import itertools
import math

import numpy as np

from tests import hp_restatement as hr
from tests import var_meth_restatement as vmr

LOG2 = math.log(2)
# the C library's lgamma (Python's math.lgamma is its own approximation); math.exp and math.log call the C library's
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.lgamma.restype = ctypes.c_double
_libm.lgamma.argtypes = [ctypes.c_double]
_TBL = None


def _tbl():
    global _TBL
    if _TBL is None:
        _TBL = vmr.logsum_table()
    return _TBL


def flogsum(a, b):
    """p7_FLogsum on float32 arrays, elementwise"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    mx = np.where(a > b, a, b)
    mn = np.where(a < b, a, b)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (mx - mn).astype(np.float32)
        take = ~((mn == -np.inf) | ~(d < np.float32(15.7)))
        idx = np.where(take, (d * np.float32(1000.0)), 0).astype(np.int64)
        return np.where(take, (mx + _tbl()[idx]).astype(np.float32), mx).astype(np.float32)


class Hap:
    """Haplotype over a window of the unedited reference: bases and their reference positions (None: inserted)"""

    def __init__(self, seq, start):
        self.seq, self.pos = list(seq), list(range(start, start + len(seq)))

    def copy(self):
        h = Hap("", 0)
        h.seq, h.pos = list(self.seq), list(self.pos)
        return h

    def apply(self, p, r, a) -> bool:
        idx = next((i for i, x in enumerate(self.pos) if x is not None and x >= p), len(self.pos))
        if idx == len(self.pos) or self.pos[idx] != p or "".join(self.seq[idx:idx + len(r)]) != r:
            return False
        self.seq[idx:idx + len(r)] = list(a)
        self.pos[idx:idx + len(r)] = [None] * len(a)
        return True

    def string(self):
        return "".join(self.seq)


def n_choose_k(n, k):
    """nChoosek with the reference's int arithmetic"""
    if k > n:
        return 0
    if k * 2 > n:
        k = n - k
    if k == 0:
        return 1
    r = n
    for i in range(2, k + 1):
        r = r * (n - i + 1) // i
    return r


def combinations(vs, base, max_haplotypes):
    """score_variant_group's combinations: [(variant ids, haplotype string)], combination 0 the empty one"""
    n, total, max_r = len(vs), 0, 1
    while max_r <= n:
        c = n_choose_k(n, max_r)
        if c + total < max_haplotypes:
            total += c
        else:
            break
        max_r += 1
    max_r -= 1
    out = []
    for r in range(max_r + 1):
        for ids in itertools.combinations(range(n), r):
            h = base.copy()
            if _apply_all(h, [vs[i] for i in ids]):
                out.append((ids, h.string()))
    return out


def _apply_all(h, vs):
    for v in vs:                                     # apply_variants stops applying at the first refusal
        if not h.apply(*v):
            return False
    return True


def groups(cands, flank, min_distance):
    """(first, end, calling_start, calling_end) of every group, called or not"""
    out, cur = [], 0
    while cur < len(cands):
        end = cur + 1
        while end < len(cands) and cands[end][0] - cands[end - 1][0] <= min_distance:
            end += 1
        out.append((cur, end, cands[cur][0] - flank, cands[end - 1][0] + len(cands[end - 1][1]) + flank))
        cur = end
    return out


def fisher_two(n11, n12, n21, n22):
    """kt_fisher_exact's two-sided p-value, restated"""
    row1, col1, n = n11 + n12, n11 + n21, n11 + n12 + n21 + n22
    hi, lo = min(row1, col1), max(0, row1 + col1 - n)
    if lo == hi:
        return 1.0

    def lch(a, b):
        lg = _libm.lgamma
        return 0.0 if b == 0 or a == b else lg(a + 1) - lg(b + 1) - lg(a - b + 1)

    def direct(v):
        return math.exp(lch(row1, v) + lch(n - row1, col1 - v) - lch(n, col1))

    st = {"x": n11, "p": direct(n11)}

    def at(v):
        n22 = v + n - row1 - col1
        if v % 11 and n22:
            x = st["x"]
            if v == x + 1:
                st["p"] *= float(row1 - x) / v * (col1 - x) / n22
                st["x"] = v
                return st["p"]
            if v == x - 1:
                st["p"] *= float(x) / (row1 - v) * (x + n - row1 - col1) / (col1 - v)
                st["x"] = v
                return st["p"]
        st["x"], st["p"] = v, direct(v)
        return st["p"]

    q = st["p"]
    left = right = 0.0
    p, i = at(lo), lo + 1
    while p < 0.99999999 * q:
        left += p
        p, i = at(i), i + 1
    if p < 1.00000001 * q:
        left += p
    p, j = at(hi), hi - 1
    while p < 0.99999999 * q:
        right += p
        p, j = at(j), j - 1
    if p < 1.00000001 * q:
        right += p
    two = left + right
    return 1.0 if two > 1.0 else two


def g(v) -> str:
    """std::ostream << double (printf "%g")"""
    if math.isnan(v):
        return "-nan" if math.copysign(1.0, v) < 0 else "nan"
    return "%g" % v


def sor(rf, rr, af, ar):
    rf, rr, af, ar = rf + 1, rr + 1, af + 1, ar + 1
    r = (rf * ar) / (af * rr)
    return math.log(r + (1.0 / r)) + math.log(min(rf, rr) / max(rf, rr)) - math.log(min(af, ar) / max(af, ar))


def genotype_search(t, n_comb, ploidy):
    """(best index or None, best score, base score) of simple_call's search over t[c][key] = float32(s - log 2)"""
    sets = np.array(list(itertools.combinations_with_replacement(range(n_comb), ploidy)), np.int64).reshape(-1, ploidy)
    score = np.zeros(sets.shape[0], np.float64)
    for q in range(t.shape[1]):
        v = np.full(sets.shape[0], -np.inf, np.float32)
        for j in range(ploidy):
            v = flogsum(v, t[sets[:, j], q])
        score = score + v.astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok = score > -np.inf
    best = None
    if ok.any():
        m = np.max(score[ok])
        best = int(np.flatnonzero(ok & (score == m))[0])
    return sets, best, (float(score[best]) if best is not None else -math.inf), float(score[0])


def restated(region_start, region_ref, recs, pairs, names, cands, score, flank=30, min_distance=10, max_haplotypes=1000, ploidy=2,
             genotype_only=False, types=()):
    """the reference's output lines (as nphh_call_haplotype / npref_call_haplotype write them, without SupportFractionByBase).
    score(reqs) -> float32 scores of [(record, e1, e2, type index or -1, string)]; names[record] the record's read name"""
    derived = Hap(region_ref, region_start)
    region_end = region_start + len(region_ref) - 1
    calls = []
    for first, end, cs, ce in groups(cands, flank, min_distance):
        if ce - cs > 200:
            continue
        assert cs >= region_start and ce <= region_end, "a window outside the region (the reference asserts)"
        vs = cands[first:end]
        combos = combinations(vs, Hap(region_ref[cs - region_start:ce - region_start + 1], cs), max_haplotypes)
        reads = hr.event_sequences(recs, pairs, cs, ce)
        sets_of = [vmr.alternatives(seq, types) for _, seq in combos]
        reqs = [(r, e1, e2, t, s) for r, e1, e2 in reads for alts in sets_of for t, s in alts]
        sc = score(reqs) if reqs else np.zeros(0, np.float32)
        at = 0
        key_of = [names[r] + ":0" for r, _, _ in reads]
        keys = sorted(set(key_of))
        kidx = {k: i for i, k in enumerate(keys)}
        s = np.zeros((len(combos), len(keys)), np.float32)
        read_sum = [None] * len(keys)
        rc = [0] * len(keys)
        for (r, _, _), k in zip(reads, key_of):
            q = kidx[k]
            for c, alts in enumerate(sets_of):
                v = vmr.score_set(sc[at:at + len(alts)])
                at += len(alts)
                s[c, q] = v
                read_sum[q] = v if read_sum[q] is None else flogsum(read_sum[q], v)[()]
            rc[q] = int(recs[r]["rc"])
        if len(combos) <= 1:
            continue
        t = (s.astype(np.float64) - LOG2).astype(np.float32)
        sets, best, best_score, base_score = genotype_search(t, len(combos), ploidy)
        best_set = [] if best is None else list(sets[best])
        if best_score - base_score < 20:
            best_set = list(sets[0])
        nk, nv = len(keys), len(vs)
        rva = [[0.0] * nv for _ in range(nk)]
        rvs = [0.0] * nv
        for c, (ids, _) in enumerate(combos):
            for q in range(nk):
                post = math.exp(float(s[c, q]) - float(read_sum[q]))
                for vi in ids:
                    rva[q][vi] += post
                    rvs[vi] += post
        for vi in range(nv):
            st = [0.0, 0.0, 0.0, 0.0]
            for q in range(nk):
                st[rc[q]] += 1 - rva[q][vi]
                st[2 + rc[q]] += rva[q][vi]
            count = sum(vi in combos[c][0] for c in best_set)
            if not (genotype_only or count > 0):
                continue
            with np.errstate(invalid="ignore", divide="ignore"):
                frac = float(np.float64(rvs[vi]) / np.float64(nk))
                by_strand = (float(np.float64(st[2]) / np.float64(st[0] + st[2])), float(np.float64(st[3]) / np.float64(st[1] + st[3])))
            two = fisher_two(int(st[0]), int(st[1]), int(st[2]), int(st[3]))
            fs = int(-4.343 * math.log(two) + .499) if two > 0 else -1
            fs = 1000 if fs < 0 else fs
            info = (f"TotalReads={nk};AlleleCount={count};SupportFraction={g(frac)};SupportFractionByStrand={g(by_strand[0])},{g(by_strand[1])};"
                    f"StrandSupport={','.join(str(int(_round(x))) for x in st)};StrandFisherTest={fs};SOR={g(sor(*st))}")
            quality = best_score - base_score if count > 0 else 0.0
            gt = ("/".join("0" if a < ploidy - count else "1" for a in range(ploidy))) if nk > 0 else "."
            calls.append((vs[vi], quality, info, gt))
    out = []
    for (p, r, a), quality, info, gt in calls:
        if derived.apply(p, r, a):
            out.append(f"{p}\t{r}\t{a}\t{np.float64(quality).view(np.uint64):016x}\t{info}\t{gt}")
    return [derived.string()] + out


def _round(x):
    """std::round: halves away from zero"""
    f = math.floor(abs(x))
    return math.copysign(f + (1 if abs(x) - f >= 0.5 else 0), x)
