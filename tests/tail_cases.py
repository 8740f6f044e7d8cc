"""Edge cases of the poly(A) and detect-polyi tail caller (nanopolish_b200/csrc/polya.cu, nph_polya_batch and
nph_detect_polyi_batch), each built deterministically from a seed and a design, and the claims each one makes about where it
sits: on the kernel's 256-step emission tiles, the boundaries and ties its folded backtrack has to get right, the bytes its
radix selection of the median decides on, the scalings and samples it reads, the poly(I) stage's 1 536-sample flat tiles and
Bernoulli switch, and the QC thresholds in double.

Cases that need a boundary, a tail length or a switch at an exact index are fitted with the port oracle (npo_polya_trace in
oracle/np_oracle.c), never with the compiled reference, so every case can be rebuilt where oracle/_ref/ does not exist.
check_tail_edges confirms every claim on the port oracle's trace and fails if a designed edge is not reached."""
from __future__ import annotations

import copy
import hashlib
from dataclasses import dataclass, field

import numpy as np

from tests import polya_cases as pc
from tests import polyi_cases as qc
from tests.polya_cases import PolyaRead

# ---- the kernel's constants (polya.cu), checked against the source by test_tail_edges_oracle ---------------------------
TILE = 256                       # kTile: steps per emission tile
EMIT_WARPS = 3                   # kEmitWarps
THREADS = 32 * (1 + EMIT_WARPS)  # kThreads: the CTA, also the radix selection's stride over k-mers
N_ST = 6
FLAT = N_ST * TILE               # kFlat: samples per flat tile of the poly(I) passes
MIN_REGION = 200.0               # n_adapter / n_polya below it: NOREGION
MAX_ADAPTER = 300.0              # adapter_length above it: ADAPTER
MAX_CLIP = 200                   # suffix_clip above it: SUFFCLIP
MIN_TAIL = 100                   # stop - start below it: no Bernoulli stage
MODES = ("polya", "polyi")
S, L, A, P, Cl, T = range(6)
RULES = ("L", "A", "P<-P", "P<-A", "C", "T")
RULE_STATE = (L, A, P, P, Cl, T)  # the state whose backpointer each rule sets

# the clean levels the designed reads are drawn at (the HMM's own means, scale 1, shift 0, var 1)
CLEAN = {"S": (70.2737, 1.0), "L": (110.973, 1.5), "A": (63.3126, 1.0), "P": (108.883, 1.0), "T": (79.679, 1.5)}


@dataclass
class TailCase:
    name: str
    mode: str                    # "polya" or "polyi"
    read: PolyaRead
    claims: set = field(default_factory=set)
    family: str = ""


def fingerprint(c: TailCase) -> str:
    r = c.read
    h = hashlib.sha1()
    for a in (r.samples.astype(np.float32), r.duration.astype(np.float32), r.map_start.astype(np.int32), r.map_stop.astype(np.int32)):
        h.update(a.tobytes())
    h.update(repr((c.mode, r.name, float(r.sample_rate).hex(), float(r.scale).hex(), float(r.shift).hex(), float(r.var).hex(),
                   int(r.suffix_clip), bool(r.loaded), r.contig, int(r.pos))).encode())
    return h.hexdigest()


def dkey(d: float) -> int:
    """the radix selection's key of a double (polya.cu dkey)"""
    u = int(np.float64(d).view(np.uint64))
    return (~u & (2 ** 64 - 1)) if u >> 63 else (u | (1 << 63))


def first_diff_byte(a: float, b: float) -> int:
    """the highest key byte (7..0) where a and b differ, -1 if equal"""
    x = dkey(a) ^ dkey(b)
    return -1 if x == 0 else (x.bit_length() - 1) // 8


def deciding_byte(median) -> int:
    """the lowest key byte at which the selection still separates the median from a sorted neighbour: the pass a selection
    that stopped early would get wrong (-1: both neighbours equal the median or are absent)"""
    lo, m, hi = (float(v) for v in median)
    bs = [first_diff_byte(m, v) for v in (lo, hi) if not np.isnan(v)]
    bs = [b for b in bs if b >= 0]
    return min(bs) if bs else -1


# ---- read builders --------------------------------------------------------------------------------------------------------
def events(rng, n_kmers: int, sample_rate: float = 3012.0):
    dur, ms, me = pc.event_table(rng, n_kmers, sample_rate)
    return dur, ms, me


def clean_read(rng, name: str, lens, labels="SLAPT", sd_scale=1.0, n_kmers=None, sample_rate=3012.0, **kw) -> PolyaRead:
    """regions of the given lengths at CLEAN levels, quantised; scale 1, shift 0, var 1 unless given"""
    parts = []
    for lab, ln in zip(labels, lens):
        mu, sd = CLEAN[lab]
        parts.append(rng.normal(mu, sd * sd_scale, int(ln)))
    v = pc.quantise(np.concatenate(parts))
    nk = int(n_kmers if n_kmers is not None else max(20, v.shape[0] // 40))
    dur, ms, me = events(rng, nk, sample_rate)
    kw.setdefault("scale", 1.0); kw.setdefault("shift", 0.0); kw.setdefault("var", 1.0)
    sc, sh, va = kw.pop("scale"), kw.pop("shift"), kw.pop("var")
    return PolyaRead(name, v, sample_rate, sc, sh, va, dur, ms, me, **kw)


def changes(labels) -> dict:
    """{(from, to): [steps c with labels[c-1] = from, labels[c] = to]}"""
    lab = np.asarray(labels)
    c = np.nonzero(lab[1:] != lab[:-1])[0] + 1
    out = {}
    for s in c:
        out.setdefault((int(lab[s - 1]), int(lab[s])), []).append(int(s))
    return out


BOUNDARY = {0: (S, L), 1: (L, A), 2: (A, P), 3: (P, T)}


def fit_boundary(port, mode, make, lens, k: int, step: int, tries: int = 12):
    """Move boundary k (0: S->L, 1: L->A, 2: A->P, 3: P->T) of the read make(lens) until the backtracked label changes there
    exactly at `step`, moving samples between region k and region k + 1.  Returns the read, or None."""
    lens = list(lens)
    for _ in range(tries):
        r = make(lens)
        t = port.tail_trace(r, mode == "polyi")
        got = changes(t["labels"]).get(BOUNDARY[k], [])
        if step in got:
            return r
        if not got:
            return None
        d = step - got[-1]
        lens[k] += d
        lens[k + 1] -= d
        if lens[k] < 1 or lens[k + 1] < 1:
            return None
    return None


def fit_tail_len(port, mode, r: PolyaRead, want: int, one=None, tries: int = 8):
    """grow or shrink the read's tail ([adapter + 1, polya)) until it holds `want` samples (polyi_cases.fit_tail, with the port)"""
    fill = np.float32(one if one is not None else CLEAN["P"][0])
    for _ in range(tries):
        seg = port.tail_trace(r, mode == "polyi")["seg"]
        ad, pa = int(seg[2]), int(seg[3])
        got = pa - (ad + 1)
        if got == want:
            return r
        d = want - got
        if d > 0:
            r.samples = np.concatenate([r.samples[:pa], np.full(d, fill, np.float32), r.samples[pa:]])
        else:
            r.samples = np.concatenate([r.samples[:pa + d], r.samples[pa:]])
    return None


def split_double(d: float):
    """floats f1, f2, f3 whose event-order sum ((0 + f1) + f2) + f3 is the double d exactly"""
    f1 = np.float32(d)
    r1 = d - float(f1)
    f2 = np.float32(r1)
    f3 = np.float32(r1 - float(f2))
    assert ((0.0 + float(f1)) + float(f2)) + float(f3) == d, d
    return [f1, f2, f3]


def duration_table(values, rng=None):
    """durations and a map whose k-th k-mer's event-order FP64 sum is values[k] exactly (None: unmapped); k-mer order shuffled"""
    vals = list(values)
    if rng is not None:
        rng.shuffle(vals)
    dur, ms, me = [], [], []
    for v in vals:
        if v is None:
            ms.append(-1); me.append(-1)
            continue
        fs = [np.float32(v)] if float(np.float32(v)) == v else split_double(v)
        ms.append(len(dur)); dur.extend(fs); me.append(len(dur) - 1)
    if not dur:
        dur = [np.float32(1.0)]
    return np.array(dur, np.float32), np.array(ms, np.int32), np.array(me, np.int32)


def with_durations(r: PolyaRead, values, rng=None) -> PolyaRead:
    r.duration, r.map_start, r.map_stop = duration_table(values, rng)
    return r


def median_design(rng, nk: int, med: float, lo: float | None, hi: float | None, below=1e-3, above=1.0):
    # below * 1.01^k stays under lo, above * 1.01^k over hi
    """nk k-mer durations whose sorted element nk / 2 is med, with neighbours lo and hi (None: far away)"""
    r = nk // 2
    vals = [below * (1 + 0.01 * i) for i in range(max(r - 1, 0))] + ([lo if lo is not None else below * 0.5] if r > 0 else [])
    vals += [med]
    rest = nk - len(vals)
    if rest > 0:
        vals += [hi if hi is not None else above] + [above * (1 + 0.01 * i) for i in range(rest - 1)]
    assert len(vals) == nk
    return vals


# ---- the cases ------------------------------------------------------------------------------------------------------------
def tile_cases(port, mode, rng):
    out = []
    for n in (2, 3, 256, 257, 258, 512, 513, 514, 99839, 99840, 99841):
        r = pc.synth_read(rng, f"{mode}-n{n}", n, n_kmers=max(3, n // 40))
        out.append(TailCase(r.name, mode, r, {f"n={n}"}, "tiles"))
    # row 0 emits sample n-1: a last sample far from sample 0 (a START sample at the end of a read that opens at the LEADER level)
    for n in (2, 257, 3000):
        r = pc.synth_read(rng, f"{mode}-lastsample{n}", n, n_kmers=max(3, n // 40))
        r.samples[0] = np.float32(CLEAN["L"][0]); r.samples[-1] = np.float32(40.0)
        out.append(TailCase(r.name, mode, r, {"row0-last-sample"}, "tiles"))
    # a NaN last sample makes row 0's START score NaN, and with it every comparison of the walk false: only row 0 reads it
    for n in (2, 3000):
        r = pc.synth_read(rng, f"{mode}-lastnan{n}", n, n_kmers=max(3, n // 40))
        r.samples[-1] = np.float32(np.nan)
        out.append(TailCase(r.name, mode, r, {"row0-nan"}, "tiles"))
    # label changes at steps 255, 256 and 257 (around the first tile edge) for every boundary, and the P -> T change at n-2 and n-1
    base = [300, 600, 900, 900, 600]
    for k in range(4):
        for step in (255, 256, 257):
            lens = list(base)
            pre = sum(lens[:k])
            if step - pre < 1:
                short = [max(1, (step - 1) // (k + 1))] * (k + 1)
                short[k] = step - sum(short[:k])
                lens[:k + 1] = short
            else:
                lens[k] = step - pre
            name = f"{mode}-b{k}@{step}"
            make = lambda ls, name=name, seed=int(rng.integers(1 << 30)): clean_read(np.random.default_rng(seed), name, ls)
            r = fit_boundary(port, mode, make, lens, k, step)
            if r is not None:
                out.append(TailCase(name, mode, r, {f"{'SLAP'[k]}>{'LAPT'[k]}@{step}"}, "tiles"))
    # the earliest S -> L change: step 2 (row 0's LEADER score is -inf, so step 1's pointer into LEADER is always START)
    make = lambda ls, seed=int(rng.integers(1 << 30)): clean_read(np.random.default_rng(seed), f"{mode}-b0@2", ls)
    r = fit_boundary(port, mode, make, [1, 600, 900, 900, 600], 0, 2)
    if r is not None:
        out.append(TailCase(r.name, mode, r, {"S>L@2"}, "tiles"))
    for back in (2, 1):
        name = f"{mode}-pt@n-{back}"
        make = lambda ls, name=name, seed=int(rng.integers(1 << 30)): clean_read(np.random.default_rng(seed), name, ls)
        n = 3000
        r = fit_boundary(port, mode, make, [300, 600, 900, 1200 - back, back], 3, n - back)
        if r is not None:
            out.append(TailCase(name, mode, r, {f"P>T@n-{back}"}, "tiles"))
    return out


def backtrack_cases(port, mode, rng):
    out = []
    lens = [300, 600, 900, 1200, 600]
    # single CLIFF samples (a value in (70, 140) far from POLYA) at and around the tile edges, and alternations P C P C P
    r = clean_read(rng, f"{mode}-pcp-tile", lens)
    for i in (2047, 2305) + tuple(range(2559, 2568, 2)):          # POLYA runs over [1800, 3000); 2048 = 8 tiles
        r.samples[i] = np.float32(135.0)
    out.append(TailCase(r.name, mode, r, {"PCP", "PCP@tile", "PCPCP"}, "backtrack"))
    # a CLIFF run that ends the tail: C C C within the last 8 POLYA samples, then TRANSCRIPT
    for off in range(4, 12):
        r = clean_read(np.random.default_rng(77), f"{mode}-cliff-end", lens)
        r.samples[2996 - off:2999 - off] = np.float32(135.0)
        if "cliff-before-end" in tail_edges(TailCase(r.name, mode, r), port.tail_trace(r, mode == "polyi")):
            break
    out.append(TailCase(r.name, mode, r, {"cliff-before-end"}, "backtrack"))
    # more than 256 cliffs
    r = clean_read(rng, f"{mode}-cliffs300", [300, 600, 900, 3000, 600])
    idx = 1800 + np.arange(0, 3000, 9)[:320]
    r.samples[idx] = np.float32(135.0)
    out.append(TailCase(r.name, mode, r, {"cliffs>256"}, "backtrack"))
    # -inf scores: a stdv so small that every Gaussian emission but START's underflows, samples outside CLIFF's range, and
    # the shortest reads (rows 1..3 have -inf ADAPTER / POLYA / CLIFF scores)
    for var, n in ((1e-30, 600), (1e-38, 600), (0.05, 2500), (0.02, 1500)):
        r = pc.synth_read(rng, f"{mode}-var{var:g}", n, var=var, scale=1.0, shift=0.0)
        out.append(TailCase(r.name, mode, r, {"inf-ties"} if var < 1e-20 else set(), "backtrack"))
    r = clean_read(rng, f"{mode}-nocliff-range", lens)
    r.samples[1800:3000][::3] = np.float32(150.0)
    out.append(TailCase(r.name, mode, r, set(), "backtrack"))
    for n in (4, 5, 6, 7):
        for s in range(3):
            r = pc.synth_read(np.random.default_rng(1000 * n + s), f"{mode}-short{n}-{s}", n, n_kmers=3)
            out.append(TailCase(r.name, mode, r, set(), "backtrack"))
    # exact finite ties in rules L and A that the backtrack reads, one float sample scanned ulp by ulp next to a boundary
    for rule, make, start in TIE_DESIGNS:
        r = tie_scan(port, mode, f"{mode}-tie-{RULES[rule]}", make, start, rule)
        if r is not None:
            out.append(TailCase(r.name, mode, r, {f"tie:{RULES[rule]}"}, "backtrack"))
    return out


# A tie in rule L at step 2: START -> START -> LEADER against START -> LEADER -> LEADER, which differ in the emissions of
# sample 1 (eS - eL) by logf(0.9) - logf(0.1); in rule A at step 5, LEADER -> ADAPTER at 4 against at 5.  Sample 1 (rule L) or
# 4 (rule A) is the scanned one; the rest holds the read in START, LEADER, ADAPTER, POLYA and TRANSCRIPT.
TIE_DESIGNS = (
    (0, lambda v: [79.7, v] + [110.973] * 300 + [63.3126] * 600 + [108.883] * 300 + [79.679] * 100, 93.35),
    (1, lambda v: [79.7, 70.27, 110.973, 110.973, v] + [63.3126] * 600 + [108.883] * 300 + [79.679] * 100, 98.05),
)


def tie_scan(port, mode, name, make, start, rule, max_ulps=4096):
    """the read make(v) (scale 1, shift 0, var 1, 30 mapped k-mers) for the float v nearest `start`, scanning up and down ulp by
    ulp, whose backtrack reads a finite tie of `rule`; None if there is none within max_ulps"""
    up = dn = np.float32(start)
    dur, ms, me = events(np.random.default_rng(1), 30)
    for _ in range(max_ulps):
        for v in (up, dn):
            r = PolyaRead(name, np.array(make(v), np.float32), 3012.0, 1.0, 0.0, 1.0, dur, ms, me)
            if rule in read_ties(port.tail_trace(r, mode == "polyi"), finite=True):
                return r
        up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
    return None


def finite_tie_search(port, mode, n_try=400, seed=5):
    """candidate quantised constant / periodic signals whose backtracked path reads an exactly tied finite comparison:
    {rule: (name, values, scalings)}"""
    rng = np.random.default_rng(seed)
    found = {}
    grid = pc.quantise(np.arange(40.0, 200.0, float(pc.ADC_STEP)))
    for i in range(n_try):
        per = int(rng.integers(1, 4))
        vals = [float(grid[int(rng.integers(grid.shape[0]))]) for _ in range(per)]
        sc = (1.0, 0.0, 1.0) if i % 2 == 0 else (float(rng.choice([0.5, 1.0, 2.0])), float(rng.choice([0.0, 1.0, -2.0])),
                                                  float(rng.choice([0.5, 1.0, 2.0])))
        dur, ms, me = events(rng, 20)
        r = PolyaRead("s", np.resize(np.array(vals, np.float32), 800), 3012.0, *sc, dur, ms, me)
        t = port.tail_trace(r, mode == "polyi")
        for rule in read_ties(t, finite=True):
            found.setdefault(rule, (f"{RULES[rule]}-{i}", vals, sc))
    return found


def read_ties(t, finite: bool) -> set:
    """the rules whose tied comparison (finite or -inf) the backtrack read: a tie at step j of rule r with labels[j+1] = r's state"""
    lab, ties = t["labels"], t["ties"]
    n = lab.shape[0]
    out = set()
    for r, st in enumerate(RULE_STATE):
        bit = (1 << (2 * r)) if finite else (2 << (2 * r))
        j = np.nonzero(ties[1:n - 1] & bit)[0] + 1
        if j.size and (lab[j + 1] == st).any():
            out.add(r)
    return out


def median_cases(rng, mode):
    out = []
    sr = 3012.0
    base = lambda name, n=600: pc.synth_read(rng, name, n)
    for nk in (1, 2, 3, 127, 128, 129, 255, 256, 257, 2999, 3000):
        r = base(f"{mode}-nk{nk}")
        vals = list((rng.integers(3, 40, nk) / sr).astype(np.float32).astype(np.float64))
        out.append(TailCase(r.name, mode, with_durations(r, vals, rng), {f"nk={nk}"}, "median"))
    r = base(f"{mode}-nk-equal")
    out.append(TailCase(r.name, mode, with_durations(r, [float(np.float32(7 / sr))] * 301), {"all-equal"}, "median"))
    # the median and its lower neighbour first differ at key byte b; low bytes need multi-event spans
    m = 0.00996503781659
    for b in range(8):
        k = dkey(m)
        lo_key = k - (1 << (8 * b)) if ((k >> (8 * b)) & 255) else k - (2 << (8 * b))
        u = lo_key & ~(1 << 63)
        lo = float(np.uint64(u).view(np.float64))
        for nk in (301, 300):
            r = base(f"{mode}-byte{b}-nk{nk}")
            # the upper neighbour differs at byte 7 (a float near 1e38), so the lower one decides at byte b
            vals = median_design(rng, nk, m, lo, None, below=lo * 1e-3, above=float(np.float32(1e38)))
            out.append(TailCase(r.name, mode, with_durations(r, vals, rng), {f"byte={b}"}, "median"))
    # unmapped k-mers (0.0) at and around the median
    for name, nz in (("zero-median", 151), ("zero-below", 150), ("zero-lower", 149)):
        r = base(f"{mode}-{name}")
        vals = [None] * nz + list((rng.integers(3, 40, 301 - nz) / sr).astype(np.float32).astype(np.float64))
        out.append(TailCase(r.name, mode, with_durations(r, vals, rng), {name}, "median"))
    # negative durations: a negative median, and negatives below a positive one
    for name, neg in (("neg-median", 200), ("neg-below", 100)):
        r = base(f"{mode}-{name}")
        vals = [-float(np.float32(v)) for v in rng.uniform(1e-3, 1e-2, neg)] + list(rng.uniform(1e-3, 1e-2, 301 - neg).astype(np.float32).astype(np.float64))
        out.append(TailCase(r.name, mode, with_durations(r, vals, rng), {name}, "median"))
    # a median span whose event-order sum differs in its last bit from every other order of its events
    trip = [np.float32(1.0), np.float32(float.fromhex("0x1.f8p-53")), np.float32(2.0 ** -53)]
    r = base(f"{mode}-order-sum")
    dur = np.array([np.float32(5e-3)] * 150 + trip + [np.float32(2.0)] * 150, np.float32)
    ms = np.array(list(range(150)) + [150] + list(range(153, 303)), np.int32)
    me = np.array(list(range(150)) + [152] + list(range(153, 303)), np.int32)
    r.duration, r.map_start, r.map_stop = dur, ms, me
    out.append(TailCase(r.name, mode, r, {"order-sum"}, "median"))
    return out


def order_sum_differs(dur) -> bool:
    """the FP64 sum of three events in event order differs from both sums that add a different event last (the orders that
    only swap the first two give the same sum)"""
    a, b, c = (float(v) for v in dur)
    ev = (a + b) + c
    return ev != (a + c) + b and ev != (b + c) + a


def scaling_cases(rng, mode):
    out = []
    lens = [300, 600, 900, 1200, 600]
    halfway = [("scale-half", dict(scale=1.0 + 2.0 ** -24)), ("shift-half", dict(shift=2.0 + 2.0 ** -23)),
               ("var-half", dict(var=1.0 + 3 * 2.0 ** -24)), ("scale-neg", dict(scale=-1.0, shift=180.0)), ("scale-zero", dict(scale=0.0)),
               ("var-subnormal", dict(var=1e-40)), ("scale-shift-double", dict(scale=1.0 + 2.0 ** -30, shift=0.1))]
    for name, kw in halfway:
        r = clean_read(rng, f"{mode}-{name}", lens, **kw)
        out.append(TailCase(r.name, mode, r, {name}, "scalings"))
    # NaN, +-inf and +-0 samples in every region
    r = clean_read(rng, f"{mode}-special", lens)
    starts = np.cumsum([0] + lens[:-1])
    for s0, ln in zip(starts, lens):
        for j, v in enumerate((np.nan, np.inf, -np.inf, 0.0, -0.0)):
            r.samples[s0 + ln // 2 + 7 * j] = np.float32(v)
    out.append(TailCase(r.name, mode, r, {"special-samples"}, "scalings"))
    return out


def polyi_cases(port, rng):
    """detect-polyi only: tails at the flat tiles, a long tail, Bernoulli switches at designed steps, an all-A tail"""
    mode = "polyi"
    out = []
    ones = lambda m: [1] * m
    for m in (1535, 1536, 1537, 3071, 3072, 3073):
        r = fit_tail_len(port, mode, qc.crafted_read(rng, f"tail{m}", m + 1), m, one=109.0)
        if r is not None:
            r.samples[int(port.tail_trace(r, True)["seg"][2]) + 1:][:m] = qc._tail([0] * (m // 2) + [1] * (m - m // 2), 109.0).astype(np.float32)
            out.append(TailCase(r.name, mode, r, {f"m={m}"}, "polyi"))
    # one long noisy tail: the sequential float mean differs from the FP64 and pairwise means
    r = qc.crafted_read(rng, "tail150k", 150000)
    lo = 2400
    r.samples[lo:lo + 150000] = pc.quantise(rng.normal(108.7, 4.5, 150000))
    out.append(TailCase(r.name, mode, r, {"long-mean"}, "polyi"))
    # the Bernoulli switch (the first A) at designed steps: fitted by moving the I/A split
    for want in (2, 1535, 1536, 1537, "m-7"):
        m = 3300
        r = fit_tail_len(port, mode, qc.crafted_read(rng, f"switch{want}", m + 1), m, one=109.0)
        if r is None:
            continue
        tail0 = int(port.tail_trace(r, True)["seg"][2]) + 1
        target = m - 7 if want == "m-7" else want
        nz = 0 if want == 2 else target
        for _ in range(12):
            bits = [0] * nz + [1] * (m - nz)
            r.samples[tail0:tail0 + m] = qc._tail(bits, 109.0).astype(np.float32)
            got = port.tail_trace(r, True)["polya_first"]
            if got == target or got < 0:
                break
            nz += target - got
            nz = max(0, min(m, nz))
        out.append(TailCase(r.name, mode, r, {f"switch={want}"}, "polyi"))
    r = fit_tail_len(port, mode, qc.crafted_read(rng, "all-a", 1201), 1200, one=109.0)
    r.samples[int(port.tail_trace(r, True)["seg"][2]) + 1:][:1200] = qc._tail(ones(1200), 109.0).astype(np.float32)
    out.append(TailCase(r.name, mode, r, {"all-A"}, "polyi"))
    # a tail whose double-scaled samples differ from the float-scaled ones (pass 0 scales with the unrounded double scalings)
    r = qc.crafted_read(rng, "double-scaling", 3000)
    r.scale, r.shift = 1.0 + 2.0 ** -25 + 2.0 ** -40, 2.0 ** -19 + 2.0 ** -60
    r.samples[2400:5400] = pc.quantise(rng.normal(108.7, 4.5, 3000))
    out.append(TailCase(r.name, mode, r, {"double-scaling"}, "polyi"))
    r = pass0_case(port)
    if r is not None:
        out.append(TailCase(r.name, mode, r, {"pass0-decides"}, "polyi"))
    for c in out:
        c.name = c.read.name = f"{mode}-{c.read.name}"
    return out


def qc_cases(port, rng, mode):
    """the QC thresholds: n_adapter and n_polya at 199 / 200, adapter_length at 300.0 and one ulp above, len at 0 and below,
    and two failures at once"""
    out = []
    sr = 4096.0
    med = 2.0 ** -8           # rate 256: adapter_length = adapter samples / 16
    fixed = lambda r: with_durations(r, [med] * 301)

    def make_fit(name, k, step, lens, **kw):
        mk = lambda ls, seed=int(rng.integers(1 << 30)): fixed(clean_read(np.random.default_rng(seed), name, ls, sample_rate=sr, **kw))
        return fit_boundary(port, mode, mk, lens, k, step)

    def fit_count(name, k, count, lens):
        """region k (2: ADAPTER, n_adapter = adapter + 1 - leader; 3: POLYA, n_polya = polya - (adapter + 1)) holds `count`"""
        step = sum(lens[:k + 1])
        for _ in range(6):
            r = make_fit(name, k, step, lens)
            if r is None:
                return None
            seg = [int(v) for v in port.tail_trace(r, mode == "polyi")["seg"]]
            got = (seg[2] + 1 - seg[1]) if k == 2 else (seg[3] - seg[2] - 1)
            if got == count:
                return r
            step += count - got
        return None

    for na in (199, 200):
        r = fit_count(f"{mode}-nadapter{na}", 2, na, [300, 600, na, 1200, 600])
        if r is not None:
            out.append(TailCase(r.name, mode, r, {f"n_adapter={na}"}, "qc"))
    for npa in (199, 200, 80, 79, 81):
        r = fit_count(f"{mode}-npolya{npa}", 3, npa, [300, 600, 900, npa, 600])
        if r is not None:
            out.append(TailCase(r.name, mode, r, {f"n_polya={npa}", "len=0" if npa == 80 else "len<0" if npa == 79 else "len>0"}, "qc"))
    # adapter_length = (adapter - leader + 1) / sample_rate * rate: 4 800 samples at 4096 Hz and rate 256 is 300.0
    r = fit_count(f"{mode}-adapter300", 2, 4800, [300, 600, 4800, 1200, 600])
    if r is not None:
        t = port.tail_trace(r, mode == "polyi")
        k = int(t["seg"][2]) - int(t["seg"][1]) + 1
        if k == 4800:
            out.append(TailCase(r.name, mode, r, {"adapter=300"}, "qc"))
            r2 = PolyaRead(f"{mode}-adapter300+ulp", r.samples.copy(), sr, r.scale, r.shift, r.var, r.duration, r.map_start, r.map_stop)
            for j in range(1, 64):
                r2.sample_rate = float(np.nextafter(sr, 0.0)) - (j - 1) * 2.0 ** -40
                if k / r2.sample_rate * 256.0 == float(np.nextafter(300.0, 400.0)):
                    break
            out.append(TailCase(r2.name, mode, r2, {"adapter=300+ulp"}, "qc"))
            for clip in (200, 201):
                r3 = PolyaRead(f"{mode}-adapter300-clip{clip}", r.samples, sr, r.scale, r.shift, r.var, r.duration, r.map_start, r.map_stop,
                               suffix_clip=clip)
                out.append(TailCase(r3.name, mode, r3, {f"clip={clip}"}, "qc"))
            r4 = PolyaRead(f"{mode}-adapter+clip", r2.samples, r2.sample_rate, r.scale, r.shift, r.var, r.duration, r.map_start, r.map_stop,
                           suffix_clip=500)
            out.append(TailCase(r4.name, mode, r4, {"two-failures"}, "qc"))
    r = make_fit(f"{mode}-noregion+adapter", 2, 900 + 6000, [300, 600, 6000, 150, 600])     # also SUFFCLIP
    if r is not None:
        r.suffix_clip = 300
        out.append(TailCase(r.name, mode, r, {"two-failures"}, "qc"))
    return out


def float_scalings(r: PolyaRead) -> PolyaRead:
    """r with its scale and shift narrowed to float: what a pass 0 that scaled with the float scalings would see (the
    segmentation takes them as floats either way)"""
    q = copy.copy(r)
    q.scale, q.shift = float(np.float32(r.scale)), float(np.float32(r.shift))
    return q


def _bit(s):
    """BernoulliHMM's bit of one centred float sample (polyi_cases.restate_bits)"""
    f = np.float32
    with np.errstate(all="ignore"):
        xx = f(100.0) if (s > f(200.0) or s < f(40.0)) else s
        return f(qc._logf(qc._pdf(xx, f(108.498), f(5.257))) / qc._logf(qc._pdf(xx, f(108.883), f(3.257)))) > f(1.0)


def _centred(x, shift, scale):
    """the centred values of tail samples x: pass 0's scaling in double narrowed to float, the sequential float mean"""
    y = ((x.astype(np.float64) - shift) / scale).astype(np.float32)
    mean = np.float32(np.add.accumulate(y, dtype=np.float32)[-1] / np.float32(y.shape[0]))
    return ((y - mean).astype(np.float32) + np.float32(108.0)).astype(np.float32)


def pass0_case(port, m=1000, nz=500, trials=50):
    """A poly(I) tail of nz 0 bits then 1 bits whose first 1 sample sits at the bit's upper threshold, such that its bit is 1
    under pass 0's double scalings and 0 under the float-narrowed ones; the Bernoulli switch then moves by one.  The scalings
    are drawn until the two centred values straddle the threshold (a scaling that shifts every sample by the same ulp cancels
    in y - mean), and the sample is found by bisection on the double path's bit."""
    rng = np.random.default_rng(29)
    r = fit_tail_len(port, "polyi", qc.crafted_read(rng, "pass0", m + 1), m, one=109.0)
    t0 = int(port.tail_trace(r, True)["seg"][2]) + 1
    r.samples[t0:t0 + m] = qc._tail([0] * nz + [1] * (m - nz), 109.0).astype(np.float32)
    key = lambda t: (t["polyi_last"], t["polya_first"], t["detected"], tuple(int(v) for v in t["seg"]))
    f = np.float32
    for _ in range(trials):
        r.scale, r.shift = 1.0 + float(rng.uniform(-3e-7, 3e-7)), float(rng.uniform(-2e-5, 2e-5))
        x = r.samples[t0:t0 + m].copy()

        def bit_d(v):
            x[nz] = v
            return _bit(_centred(x, r.shift, r.scale)[nz])
        lo, hi = f(113.0), f(115.5)
        if bit_d(lo) == bit_d(hi):
            continue
        b_lo = bit_d(lo)
        while np.nextafter(lo, hi) != hi:
            mid = f((float(lo) + float(hi)) / 2)
            if mid in (lo, hi):
                break
            lo, hi = (mid, hi) if bit_d(mid) == b_lo else (lo, mid)
        for v in (lo, hi):
            x[nz] = v
            q = float_scalings(r)
            if _bit(_centred(x, r.shift, r.scale)[nz]) != _bit(_centred(x, q.shift, q.scale)[nz]):
                r.samples[t0 + nz] = v
                if key(port.tail_trace(r, True)) != key(port.tail_trace(float_scalings(r), True)):
                    return r
        r.samples[t0 + nz] = f(109.0)
    return None


def all_cases(port) -> list:
    """every case of every family, polya first; deterministic"""
    out = []
    for mode in MODES:
        rng = np.random.default_rng(20261017 if mode == "polya" else 20261018)
        out += tile_cases(port, mode, rng)
        out += backtrack_cases(port, mode, rng)
        out += median_cases(rng, mode)
        out += scaling_cases(rng, mode)
        out += qc_cases(port, rng, mode)
        if mode == "polyi":
            out += polyi_cases(port, rng)
    for m in MODES:
        r = pc.synth_read(np.random.default_rng(3), f"{m}-failed-load", 300)
        r.loaded = False
        out.append(TailCase(r.name, m, r, {"failed-load"}, "batches"))
    return out


# ---- claims ---------------------------------------------------------------------------------------------------------------
def tail_edges(c: TailCase, t, port=None) -> set:
    """the edges case c reaches, from its port-oracle trace t (None for a failed load); with the port oracle, also whether
    pass 0's double scalings decide its poly(I) answer"""
    r = c.read
    e = set()
    if not r.loaded:
        return {"failed-load"}
    n = r.samples.shape[0]
    e.add(f"n={n}")
    lab = t["labels"]
    ch = changes(lab)
    if n > 1 and abs(float(r.samples[0]) - float(r.samples[-1])) > 30:
        e.add("row0-last-sample")
    if n > 1 and np.isnan(r.samples[-1]) and not np.isnan(r.samples[0]):
        e.add("row0-nan")
    for (a, b), steps in ch.items():
        nm = "SLAPCT"
        for s in steps:
            for want in (2, 255, 256, 257):
                if s == want:
                    e.add(f"{nm[a]}>{nm[b]}@{want}")
            if s == n - 2:
                e.add(f"{nm[a]}>{nm[b]}@n-2")
            if s == n - 1:
                e.add(f"{nm[a]}>{nm[b]}@n-1")
    pcp = [i for i in range(1, n - 1) if lab[i] == Cl and lab[i - 1] == P and lab[i + 1] == P]
    if pcp:
        e.add("PCP")
    if any(i % TILE in (TILE - 1, 0, 1) for i in pcp):
        e.add("PCP@tile")
    if any(i + 2 in pcp for i in pcp):
        e.add("PCPCP")
    pa = int(t["seg"][3])
    if 0 < pa < n and lab[pa] == P and (lab[max(0, pa - 8):pa] == Cl).any():
        e.add("cliff-before-end")
    if int(t["seg"][4]) > 256:
        e.add("cliffs>256")
    fin, inf = read_ties(t, True), read_ties(t, False)
    e |= {f"tie:{RULES[k]}" for k in fin} | {f"inf-tie:{RULES[k]}" for k in inf}
    if inf:
        e.add("inf-ties")
    nk = r.map_start.shape[0]
    e.add(f"nk={nk}")
    med = t["median"]
    b = deciding_byte(med)
    if b >= 0:
        e.add(f"byte={b}")
    sums = _sums(r)
    if len(set(sums)) == 1 and nk > 1:
        e.add("all-equal")
    if med[1] == 0.0:
        e.add("zero-median")
    if not np.isnan(med[0]) and med[0] == 0.0 and med[1] > 0:
        e.add("zero-below")
    if (np.array(sums) == 0.0).sum() >= nk // 2 - 2 and med[1] > 0:
        e.add("zero-lower")
    if med[1] < 0:
        e.add("neg-median")
    if min(sums) < 0 < med[1]:
        e.add("neg-below")
    for k in range(nk):
        s0, s1 = int(r.map_start[k]), int(r.map_stop[k])
        if s0 != -1 and s1 - s0 == 2 and sums[k] == med[1] and order_sum_differs(r.duration[s0:s1 + 1]):
            e.add("order-sum")
    f32 = np.float32
    if float(f32(r.scale)) != r.scale and abs(float(f32(r.scale)) - r.scale) * 2 == abs(float(np.spacing(f32(r.scale)))):
        e.add("scale-half")
    if float(f32(r.shift)) != r.shift and abs(float(f32(r.shift)) - r.shift) * 2 == abs(float(np.spacing(f32(r.shift)))):
        e.add("shift-half")
    if float(f32(r.var)) != r.var and abs(float(f32(r.var)) - r.var) * 2 == abs(float(np.spacing(f32(r.var)))):
        e.add("var-half")
    if r.scale < 0:
        e.add("scale-neg")
    if r.scale == 0:
        e.add("scale-zero")
    if 0 < float(f32(r.var) * f32(3.2570)) < float(np.finfo(np.float32).tiny):
        e.add("var-subnormal")
    if float(f32(r.scale)) != r.scale and float(f32(r.shift)) != r.shift:
        e.add("scale-shift-double")
    x = r.samples
    if np.isnan(x).any() and (x == np.inf).any() and (x == -np.inf).any() and ((x == 0) & ~np.signbit(x)).any() and ((x == 0) & np.signbit(x)).any():
        e.add("special-samples")
    # detect-polyi
    if c.mode == "polyi" and t["bernoulli"]:
        ad, pa = int(t["seg"][2]), int(t["seg"][3])
        m = pa - ad - 1
        e.add(f"m={m}")
        y = ((r.samples[ad + 1:pa].astype(np.float64) - r.shift) / r.scale).astype(np.float32)
        if m > 100000:
            seq = t["tail_mean"]
            if seq != f32(y.astype(np.float64).mean()) and seq != f32(np.sum(y, dtype=np.float32) / f32(m)):
                e.add("long-mean")
        yf = ((r.samples[ad + 1:pa] - f32(r.shift)) / f32(r.scale)).astype(np.float32)
        if (yf != y).any():
            e.add("double-scaling")
            if port is not None:
                key = lambda u: (u["polyi_last"], u["polya_first"], u["detected"], tuple(int(v) for v in u["seg"]))
                if key(t) != key(port.tail_trace(float_scalings(r), True)):
                    e.add("pass0-decides")
        sw = t["polya_first"]
        for want in (2, 1535, 1536, 1537):
            if sw == want:
                e.add(f"switch={want}")
        if sw == m - 7:
            e.add("switch=m-7")
        if t["bits"].all():
            e.add("all-A")
    # QC
    seg = [int(v) for v in t["seg"]]
    ld, ad, pa = seg[1], seg[2], seg[3]
    nad, npo = (ad + 1) - ld, pa - (ad + 1)
    e.add(f"n_adapter={nad}")
    e.add(f"n_polya={npo}")
    al = (ad - (ld - 1)) / r.sample_rate * t["read_rate"]
    if al == 300.0:
        e.add("adapter=300")
    if al == float(np.nextafter(300.0, 400.0)):
        e.add("adapter=300+ulp")
    e.add(f"clip={r.suffix_clip}")
    ln = npo / r.sample_rate * t["read_rate"] + -5.0
    e.add("len=0" if ln == 0.0 else "len<0" if ln < 0 else "len>0" if ln > 0 else "len=nan")
    fails = (nad < 200 or npo < 200) + (al > 300.0) + (r.suffix_clip > 200)
    if fails >= 2:
        e.add("two-failures")
    return e


def _sums(r: PolyaRead):
    out = []
    for s0, s1 in zip(r.map_start, r.map_stop):
        acc = 0.0
        if s0 != -1:
            for j in range(s0, s1 + 1):
                acc += float(r.duration[j])
        out.append(acc)
    return out


# every edge each family must reach (the builders' claims are per case; these are what the suite as a whole must cover)
EDGES = {
    "tiles": [f"n={n}" for n in (2, 3, 256, 257, 258, 512, 513, 514, 99839, 99840, 99841)] + ["row0-last-sample", "row0-nan", "S>L@2"]
             + [f"{a}>{b}@{s}" for a, b in ("SL", "LA", "AP", "PT") for s in (255, 256, 257)] + ["P>T@n-2", "P>T@n-1"],
    "backtrack": ["PCP", "PCP@tile", "PCPCP", "cliff-before-end", "cliffs>256", "inf-ties", "tie:L", "tie:A"],
    "median": [f"nk={n}" for n in (1, 2, 3, 127, 128, 129, 255, 256, 257, 2999, 3000)] + ["all-equal"]
              + [f"byte={b}" for b in range(8)] + ["zero-median", "zero-below", "zero-lower", "neg-median", "neg-below", "order-sum"],
    "scalings": ["scale-half", "shift-half", "var-half", "scale-neg", "scale-zero", "var-subnormal", "scale-shift-double",
                 "special-samples"],
    "qc": ["n_adapter=199", "n_adapter=200", "n_polya=199", "n_polya=200", "len=0", "len<0", "adapter=300", "adapter=300+ulp",
           "clip=200", "clip=201", "two-failures"],
    "polyi": [f"m={m}" for m in (1535, 1536, 1537, 3071, 3072, 3073)] + ["long-mean", "double-scaling", "pass0-decides", "all-A"]
             + [f"switch={w}" for w in (2, 1535, 1536, 1537, "m-7")],
    "batches": ["failed-load"],
}
# the ties the backtrack must read at -inf in both modes.  Rules L and A never tie at -inf where the backtrack reads them:
# - L compares START -> LEADER, and START's score is never -inf (its emission is at least logf(0.5 * 0.00476));
# - the backtrack reads rule A at step j only where p[j+1] = ADAPTER, and that label came from a pointer that chose ADAPTER
#   by a strict < (POLYA's A branch at step j+1, or rule A itself at step j+1), so ADAPTER's score at row j is finite, and
#   with it the larger of the two values rule A compares at step j.
# Finite ties in L and A come from tie_scan; test_builders_reach_every_edge prints which rules the quantised search reaches.
INF_TIE_RULES = ("P<-P", "P<-A", "C", "T")


def check_tail_edges(port, cases=None):
    """every claim of every case holds on the port oracle's trace; returns ({family: {claim: [cases]}}, traces)"""
    cases = cases if cases is not None else all_cases(port)
    cover, traces, bad = {}, {}, []
    for c in cases:
        t = port.tail_trace(c.read, c.mode == "polyi") if c.read.loaded else None
        traces[c.name] = t
        got = tail_edges(c, t, port)
        missing = c.claims - got
        if missing:
            bad.append((c.name, sorted(missing)))
        fam = cover.setdefault(c.family, {})
        for k in sorted(c.claims):
            fam.setdefault(k, [])
            if k in got:
                fam[k].append(c.name)
        for k in sorted(got):
            if k.startswith(("tie:", "inf-tie:")):
                cover.setdefault("ties", {}).setdefault(k, []).append(c.name)
    assert not bad, f"designed edges not reached: {bad[:8]}"
    for fam, edges in EDGES.items():
        got = cover.get(fam, {})
        for m in (("polyi",) if fam == "polyi" else MODES):
            missing = [k for k in edges if not any(nm.startswith(m) for nm in got.get(k, []))]
            assert not missing, f"{fam} ({m}): edges no case reaches: {missing}"
    for m in MODES:
        missing = [k for k in INF_TIE_RULES if not any(nm.startswith(m) for nm in cover["ties"].get(f"inf-tie:{k}", []))]
        assert not missing, f"{m}: -inf ties the backtrack never reads: {missing}"
    return cover, traces


def coverage_table(cover: dict, title: str) -> str:
    rows = [f"{title}: edge".ljust(34) + "cases"]
    for k, v in cover.items():
        rows.append(k.ljust(34) + (f"{len(v):4d}  {', '.join(v[:3])}{' ...' if len(v) > 3 else ''}" if v else "MISSING"))
    return "\n".join(rows)


# ---- answers: the reference's, the port oracle's and the device's in one comparable form --------------------------------
GOLDEN = "ref_tail_edges.pkl.xz"


class TailRefs:
    """oracle/_ref/libnpref_polya.so and libnpref_polyi.so"""

    def __init__(self):
        self.polya, self.polyi = pc.RefPolya(), qc.RefPolyi()

    def answer(self, c: TailCase):
        if c.mode == "polya":
            seg, rl, q, row = self.polya.read(c.read)
            bern, det = (-1, -1), -1
        else:
            seg, rl, q, bern, det, row = self.polyi.read(c.read)
            bern, det = bern or (-1, -1), -1 if det is None else det
        if seg is None:
            return (None, None, None, q, -1, -1, -1, row)
        return (tuple(int(v) for v in seg), float(rl[0]).hex(), float(rl[1]).hex(), int(q), int(bern[0]), int(bern[1]), int(det), row)


def live_refs():
    """oracle/_ref/libnpref_polya.so and libnpref_polyi.so"""
    import os
    return TailRefs() if os.path.exists(pc.REF_POLYA) and os.path.exists(qc.REF_POLYI) else None


def result_answer(c: TailCase, g):
    """a device result (POLYA_RES_DT or POLYI_RES_DT record) in the answer form, its row from the TSV writer"""
    from nanopolish_b200 import detect_polyi, polya
    r = c.read
    s = g if c.mode == "polya" else g["seg"]
    row = polya.row(r.name, r.contig, r.pos, g) if c.mode == "polya" else detect_polyi.row(r.name, r.contig, r.pos, g)
    if int(s["qc"]) == polya.READ_FAILED_LOAD:
        return (None, None, None, int(s["qc"]), -1, -1, -1, row)
    seg = tuple(int(s[k]) for k in ("start", "leader", "adapter", "polya", "cliffs"))
    bern = (-1, -1, -1) if c.mode == "polya" else (int(g["polyi_last"]), int(g["polya_first"]), int(g["detected"]))
    return (seg, float(s["read_rate"]).hex(), float(s["polya_length"]).hex(), int(s["qc"])) + bern + (row,)


def port_answer(port, c: TailCase):
    """the port oracle's answer, through the same result record and row writer as the device's"""
    from nanopolish_b200.synth import POLYA_RES_DT, POLYI_RES_DT
    g = np.zeros(1, POLYA_RES_DT if c.mode == "polya" else POLYI_RES_DT)[0]
    s = g if c.mode == "polya" else g["seg"]
    if not c.read.loaded:
        s["read_rate"] = s["polya_length"] = -1.0
        s["qc"] = 4
        if c.mode == "polyi":
            g["polyi_last"] = g["polya_first"] = g["detected"] = -1
        return result_answer(c, g)
    t = port.tail_trace(c.read, c.mode == "polyi")
    for k, v in zip(("start", "leader", "adapter", "polya", "cliffs"), t["seg"]):
        s[k] = v
    s["read_rate"], s["polya_length"], s["qc"] = t["read_rate"], t["polya_length"], t["qc"]
    if c.mode == "polyi":
        g["polyi_last"], g["polya_first"], g["detected"] = t["polyi_last"], t["polya_first"], t["detected"]
    return result_answer(c, g)
