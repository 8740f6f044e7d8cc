"""Edge reads for the CUDA event detector (csrc/event_detect.cu), and a restatement of the geometry and paths it takes.

The fused kernel walks a read as LANES = 32 * WPR segments, each warmed up from a fresh peak-detector state, verifies every
segment's starting state against its left neighbour and re-walks until the chain agrees; boundaries go into per-lane slices of
the read's room.  A read whose prefix sums are not provably exact (the guard), whose boundaries crowd a lane's slice, or whose
long window is wider than the fused kernel stages takes the streaming fallback.  This module states those rules (`seg_len`,
`lane_ranges`, `slice_size`, `heuristic_wpr`, `guard`, `predict`), builds reads that sit on their edges (`edge_reads`), each
listing the edges it claims, and `check_edges` confirms every claim on the port oracle's run (npo_detect_events_trace for the
t-statistics and the step that emitted each boundary, npo_peak_walk for the warm-up, snapshot and repair walks).

Bound on the room: both detectors are masked at step 0 and take the first t-statistic as their running minimum at step 1, so
the first boundary is at 2 or later.  A detector that emits peak p at step i (> p) starts its next peak no earlier than
i + 1, and the long detector is reset at every step the short one holds a peak over its threshold, so consecutive
boundaries are >= 2 samples apart, and the last one is at n - 2 or earlier.  A read of n >= 2 samples therefore has at most
floor((n - 2) / 2) boundaries, i.e. at most floor(n / 2) events, 8 fewer than load_from_raw's room of n / 2 + 8.  The
"densest" parameter set (w1 = w2 = 1, negative thresholds and peak height) reaches the bound: a boundary every two samples."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200 import synth

# ---- event_detect.cu's constants ----------------------------------------------------------------------------------------
FUSED_MAX_W2 = 14          # kFusedMaxW2: wider long windows take the streaming kernel
MAX_W2 = 16                # kMaxW2: wider ones are refused
PEAK_WARPS = 4             # kPeakWarps: warps per CTA of the fused kernel
FUSED_WARM = 128           # kFusedWarm: warm-up samples before each segment
TEMPLATED = ((3, 6), (7, 14))
FLT_MAX = np.float32(3.4028235e38)

PEAK_STATE_DT = np.dtype([("masked_to", "<u8", 2), ("peak_pos", "<i8", 2), ("peak_value", "<f4", 2), ("valid_peak", "<i4", 2)])
assert PEAK_STATE_DT.itemsize == 48


def same(got, want):
    """identical boundaries and bit-identical length / mean / stdv"""
    assert got.shape[0] == want.shape[0]
    assert np.array_equal(got["start"], want["start"])
    for f in ("length", "mean", "stdv"):
        assert np.array_equal(got[f].view(np.uint32), want[f].view(np.uint32)), f


def params(w1, w2, t1=None, t2=9.0, ph=None):
    p = np.zeros(1, synth.EVENT_PARAMS_DT)
    rna = w2 >= 10
    p[0] = (w1, w2, (2.5 if rna else 1.4) if t1 is None else t1, t2, (1.0 if rna else 0.2) if ph is None else ph, 0)
    return p


# the parameter sets every edge read runs under: name -> (record, window class)
PARAMS = {}
for _w1, _w2 in [(1, 1), (1, 2), (2, 2), (2, 14), (3, 7), (4, 9), (5, 5), (6, 13), (13, 14), (14, 14)]:
    PARAMS[f"w{_w1},{_w2}"] = params(_w1, _w2)
PARAMS["dna"] = params(3, 6)
PARAMS["rna"] = params(7, 14)
PARAMS["w1,16"] = params(1, 16)
PARAMS["w15,16"] = params(15, 16)
PARAMS["ph0"] = params(3, 6, ph=0.0)
PARAMS["ph-neg"] = params(4, 9, ph=-0.5)
PARAMS["thr0"] = params(3, 6, t1=0.0, t2=0.0)
PARAMS["thr-huge"] = params(3, 6, t1=3e38, t2=3e38)
PARAMS["thr-huge-w5"] = params(2, 5, t1=3e38, t2=3e38)
PARAMS["ph-huge"] = params(3, 6, ph=3e38)
PARAMS["densest"] = params(1, 1, t1=-1.0, t2=-1.0, ph=-1.0)


def window_class(p) -> str:
    w1, w2 = int(p[0]["window_length1"]), int(p[0]["window_length2"])
    if w2 > FUSED_MAX_W2:
        return "fallback"
    return "templated" if (w1, w2) in TEMPLATED else "generic"


CLASSES = ("generic", "templated", "fallback")
WPRS = (1, 2, 4)


# ---- geometry ---------------------------------------------------------------------------------------------------------
def seg_len(n: int, lanes: int) -> int:
    return ((n + lanes - 1) // lanes + 31) // 32 * 32


def lane_ranges(n: int, lanes: int, warm: int):
    """[(a0, b0, b1)] of every lane that owns samples: warm-up from a0, owned range [b0, b1)"""
    seg = seg_len(n, lanes)
    out = []
    for gl in range(lanes):
        b0 = gl * seg
        if b0 >= n:
            break
        out.append((b0 - warm if b0 > warm else 0, b0, min(n, b0 + seg)))
    return out


def slice_size(event_cap: int, lanes: int) -> int:
    return (event_cap - 1) // lanes


def warm_of(env_value) -> int:
    """$NPH_EVENTS_WARMUP rounded up to a multiple of 32, kFusedWarm without it"""
    return FUSED_WARM if env_value is None else (int(env_value) + 31) // 32 * 32


def heuristic_wpr(n_reads: int, longest: int, sm_count: int, warm: int = FUSED_WARM) -> int:
    """nph_detect_events_device's warps per read without $NPH_EVENTS_WPR"""
    wpr = 1
    while wpr < 4 and n_reads * wpr < sm_count * 20 and longest // (64 * wpr) >= 2 * warm:
        wpr *= 2
    return wpr


@dataclass
class Guard:
    lg: int
    span_x: int
    span_q: int
    okx: bool
    okq: bool
    evn: int = 0
    evx: int = 0

    @property
    def exact(self):
        return self.okx and self.okq


def guard(x) -> Guard:
    """the fused kernel's exactness guard on a read's samples"""
    x = np.ascontiguousarray(x, np.float32)
    lg = int(x.shape[0]).bit_length()                                  # ceil(log2(n + 1))
    vb = x.view(np.uint32) & np.uint32(0x7FFFFFFF)
    qb = (x * x).astype(np.float32).view(np.uint32)
    vmax, qmax = int(vb.max()), int(qb.max())
    vmin = int(vb[vb != 0].min()) if vmax else 0xFFFFFFFF
    qmin = int(qb[qb != 0].min()) if qmax else 0xFFFFFFFF
    evx, evn, eqx, eqn = vmax >> 23, vmin >> 23, qmax >> 23, qmin >> 23
    sx, sq = lg + evx + 24 - evn, lg + eqx + 24 - eqn
    okx = vmax == 0 or (evn >= 97 and evx <= 157 and sx <= 53)
    okq = qmax == 0 or (eqn >= 66 and eqx <= 188 and sq <= 53)
    return Guard(lg, sx, sq, okx, okq, evn, evx)


# ---- the walk, restated over the port oracle's peak detector --------------------------------------------------------------
def fresh_state():
    s = np.zeros(1, PEAK_STATE_DT)
    s["peak_pos"] = -1
    s["peak_value"] = FLT_MAX
    return s


@dataclass
class Prediction:
    path: str                       # "fast", "guard", "slice" (fused kernel refused the read) or "wide" (w2 > 14)
    repairs: int = 0                # repair rounds the fused kernel walks
    counts: list = field(default_factory=list)    # boundaries per owning lane
    R: int = 0
    cross_warp: bool = False        # a lane at a warp's first position was re-walked from the previous warp's last lane
    pv0_only: bool = False          # some snapshot differed from its left neighbour's state in the short peak value alone
    snap_mismatch: bool = False


class Trace:
    """the port oracle's run of one read under one parameter set"""

    def __init__(self, port, x, prm):
        self.x = np.ascontiguousarray(x, np.float32)
        self.prm = prm
        self.events, self.t1, self.t2, self.steps = port.detect_events_trace(self.x, prm)
        self.port = port
        self._walks = {}

    @property
    def boundaries(self):
        return self.events["start"][1:].astype(np.int64)

    def walk(self, a, b, state):
        key = (a, b, state.tobytes())
        if key not in self._walks:
            s = state.copy()
            pk, _ = self.port.peak_walk(self.t1, self.t2, self.prm, a, b, s)
            self._walks[key] = (s, len(pk))
        s, c = self._walks[key]
        return s.copy(), c


def _differs_in_pv0_only(a, b) -> bool:
    a2, b2 = a.copy(), b.copy()
    a2["peak_value"][0][0] = b2["peak_value"][0][0] = 0
    return a.tobytes() != b.tobytes() and a2.tobytes() == b2.tobytes()


def predict(tr: Trace, lanes: int, warm: int, event_cap: int) -> Prediction:
    """the path the device takes for one read, its repair rounds and its lanes' boundary counts"""
    n = tr.x.shape[0]
    p = tr.prm[0]
    if int(p["window_length2"]) > FUSED_MAX_W2:
        return Prediction("wide")
    rngs = lane_ranges(n, lanes, warm)
    sts, snaps, counts = [], [], []
    for a0, b0, b1 in rngs:
        snap, _ = tr.walk(a0, b0, fresh_state())
        st, c = tr.walk(b0, b1, snap)
        sts.append(st); snaps.append(snap); counts.append(c)
    g = guard(tr.x)
    pr = Prediction("fast", R=slice_size(event_cap, lanes))
    if g.exact:
        for _ in range(lanes):
            bad = [gl for gl in range(1, len(rngs)) if snaps[gl].tobytes() != sts[gl - 1].tobytes()]
            if not bad:
                break
            pr.snap_mismatch = True
            pr.pv0_only |= any(_differs_in_pv0_only(snaps[gl], sts[gl - 1]) for gl in bad)
            pr.cross_warp |= any(gl % 32 == 0 for gl in bad)
            upd = {}
            for gl in bad:
                left = sts[gl - 1]
                st, c = tr.walk(rngs[gl][1], rngs[gl][2], left)
                upd[gl] = (st, left, c)
            for gl, (st, left, c) in upd.items():
                sts[gl], snaps[gl], counts[gl] = st, left, c
            pr.repairs += 1
        # once verified, every lane counts the sequential detector's boundaries in its range
        steps = tr.steps.astype(np.int64)
        assert counts == [int(((steps >= b0) & (steps < b1)).sum()) for _, b0, b1 in rngs]
    pr.counts = counts
    if not g.exact:
        pr.path = "guard"
    elif any(c > pr.R for c in counts):
        pr.path = "slice"
    return pr


# ---- edge reads -------------------------------------------------------------------------------------------------------
@dataclass
class EdgeRead:
    name: str
    x: np.ndarray
    claims: frozenset          # edge kinds this read is built to reach (checked by check_edges)


def _steps(n, seed, lo=60.0, hi=120.0, dwell=9.0, noise=1.0):
    rng = np.random.default_rng(seed)
    x = np.empty(n, np.float64)
    i = 0
    while i < n:
        d = max(1, int(rng.exponential(dwell)) + 1)
        x[i:i + d] = rng.uniform(lo, hi)
        i += d
    return (x + noise * rng.standard_normal(n)).astype(np.float32)


def adc(n, seed, noise=1.5, dwell=9.0, digitisation=8192.0, rng_pa=1400.0, offset=10.0, lo=40.0, hi=250.0):
    """ADC-quantised current: (adc + offset) * range / digitisation, levels in [lo, hi] pA"""
    scale = np.float32(rng_pa / digitisation)
    pa = _steps(n, seed, lo + 2, hi - 2, dwell, noise).astype(np.float64)
    code = np.clip(np.rint(pa / float(scale) - offset), lo / float(scale) - offset, hi / float(scale) - offset)
    return ((code + offset).astype(np.float32) * scale).astype(np.float32)


def _span_read(n, seed, big_q_exp, tail_small=False):
    """levels alternating between x in [1, 1.41) (x*x in [1, 2)) and x with x*x in [2^e, 2^(e+1)), e = big_q_exp: the square
    span is ceil(log2(n + 1)) + e + 24.  tail_small puts the small levels only in the last quarter, after a prefix of large
    samples whose square sum passes 2^(e + lg) (so the sequential double prefix sum rounds there)"""
    rng = np.random.default_rng(seed)
    lo_b, hi_b = 2.0 ** (big_q_exp / 2), 2.0 ** ((big_q_exp + 1) / 2)
    x = np.empty(n, np.float32)
    i, k = 0, 0
    while i < n:
        d = min(int(rng.integers(4, 14)), n - i)
        small = (k % 2 == 1) if not tail_small else (i > 3 * n // 4 and k % 2 == 1)
        if small:
            x[i:i + d] = rng.uniform(1.0, 1.41, d).astype(np.float32)
        else:
            lvl = rng.uniform(hi_b * 0.93, hi_b * 0.995) if tail_small else rng.uniform(lo_b * 1.01, hi_b * 0.99)
            x[i:i + d] = (lvl + rng.uniform(-0.004, 0.004, d) * hi_b).astype(np.float32)
        i += d; k += 1
    big = x > 2
    x[big] = np.clip(x[big], np.float32(lo_b * 1.0001), np.float32(hi_b * 0.9999))
    x[0] = np.float32(lo_b * 1.0001) if tail_small else x[0]
    return x


def edge_reads() -> list:
    R = []
    add = lambda name, x, *claims: R.append(EdgeRead(name, np.ascontiguousarray(x, np.float32), frozenset(claims)))
    # segment geometry, for each lane count: around multiples of 32 * LANES, last owning lane of 1 and of fewer than w2 samples
    for wpr in WPRS:
        L = 32 * wpr
        for k in (1, 3):
            for d in (-1, 0, 1):
                add(f"n=32L*{k}{d:+d}@L{L}", _steps(32 * L * k + d, 100 * L + 10 * k + d), f"n=32L{d:+d}")
        add(f"last-lane-1@L{L}", _steps(32 * L + 1, 7 * L + 1), "last-lane=1")
        add(f"last-lane-5@L{L}", _steps(32 * L + 5, 7 * L + 5), "last-lane<w2")
    add("idle-lanes", _steps(700, 3), "idle-lanes", "warm>seg")
    # n = 2w - 1 and 2w for every window length, and one-sample reads
    windows = {int(p[0][f]) for p in PARAMS.values() for f in ("window_length1", "window_length2")} - {1}
    for n in range(1, 34):
        add(f"short-{n}", _steps(n, 500 + n, dwell=3.0), *(["n=2w-1"] if (n + 1) // 2 in windows and n % 2 else []),
            *(["n=2w"] if n // 2 in windows and n % 2 == 0 else []))
    # a stepped stretch, then a plateau longer than the warm-up: the chain re-verifies lane after lane (m1 differs)
    for wpr in WPRS:
        L = 32 * wpr
        x = _steps(64 * L, 900 + L)
        x[2048:] = np.float32(93.25)
        add(f"plateau@L{L}", x, "repair", "repair-rounds>1", "repair-cross-warp")
    add("steps-9000", _steps(9000, 77), "repair")
    add("steps-20000", _steps(20000, 78), "repair")
    # the guard: square span 53 at n = 2^12 - 1, 54 at 2^12 (lg steps), 54 from the exponent range with a rounding prefix sum
    x53 = _span_read(4096, 11, 17)
    add("span53-n4095", x53[:4095], "span=53", "lg-pass")
    add("span54-n4096", x53, "span=54", "lg-fail", "q-binds")
    add("span54-rounds", _span_read(4095, 12, 18, tail_small=True), "span=54", "q-binds", "prefix-rounds")
    # the exponent window of the samples
    rng = np.random.default_rng(21)
    lvl = lambda n, a, b: (np.repeat(rng.uniform(a, b, n // 8 + 1), 8)[:n]).astype(np.float32)
    tiny = (lvl(3000, 1.0, 1.99) * np.float32(2.0 ** -30)).astype(np.float32)
    add("x=2^-30", tiny, "x-min-2^-30")
    t2 = tiny.copy(); t2[1500] = np.float32(2.0 ** -30 * 0.75)
    add("x<2^-30", t2, "x-below-2^-30")
    huge = (lvl(3000, 1.0, 1.99) * np.float32(2.0 ** 30)).astype(np.float32)
    add("x~2^31", huge, "x-max-2^31")
    h2 = huge.copy(); h2[1700] = np.float32(2.0 ** 31)
    add("x=2^31", h2, "x-at-2^31")
    # zeros, -0.0, negative and mixed-sign samples on the fast path (quarter-pA steps)
    z = np.round(_steps(5000, 31) * 4) / 4
    z[::37] = 0.0; z[5::41] = -0.0
    add("zeros", z, "zeros", "neg-zero")
    add("negative", -np.round(_steps(5000, 32) * 4) / 4, "negative")
    add("mixed-sign", np.round(_steps(5000, 33, lo=-50.0, hi=50.0) * 4) / 4, "mixed-sign")
    # ADC-quantised current: noisy, and noise-free steps (exact ties, zero variance, zero difference of means)
    add("adc-noisy", adc(12000, 41), "adc")
    add("adc-flat-steps", adc(6000, 42, noise=0.0, dwell=20.0), "adc", "cv-clamped", "delta=0", "tstat-tie")
    add("adc-flat-short", adc(3000, 43, noise=0.0, dwell=4.0), "adc", "cv-clamped", "delta=0", "tstat-tie")
    # period [a a a b b b]: every long window pair has equal means (t2 = 0) and no short one does, so under a peak height too large
    # to rise a warmed-up lane differs from the sequential state in the short detector's running minimum alone
    add("period-6", np.tile(np.array([80.0, 80.0, 80.0, 95.5, 95.5, 95.5], np.float32), 1000), "pv0-only")
    # small reads whose room is below one boundary per lane (R = 0)
    for n in (24, 40, 49):
        add(f"r0-{n}", _steps(n, 600 + n, dwell=4.0), "R=0")
    return R


def room(n: int) -> int:
    """load_from_raw's room per read"""
    return n // 2 + 8


def batch(reads, caps=None):
    """(raw, RAW_READ_DT) of a batch of edge reads, each with the room load_from_raw gives it unless caps says otherwise"""
    rr = np.zeros(len(reads), synth.RAW_READ_DT)
    so = eo = 0
    for i, r in enumerate(reads):
        n = r.x.shape[0]
        cap = room(n) if caps is None else int(caps[i])
        rr[i] = (so, eo, n, cap)
        so += n; eo += cap
    return np.concatenate([r.x for r in reads]), rr


# ---- claims -----------------------------------------------------------------------------------------------------------
FUSED = ("generic", "templated")
# edge kind -> the window classes it applies to (every WPR unless WPR_OF says otherwise)
APPLIES = {
    "n=32L-1": FUSED, "n=32L+0": FUSED, "n=32L+1": FUSED, "last-lane=1": FUSED, "last-lane<w2": FUSED, "idle-lanes": FUSED,
    "warm>seg": FUSED, "repair": FUSED, "repair-rounds>1": FUSED, "repair-cross-warp": FUSED, "slice-overflow": FUSED, "R=0": FUSED,
    "span=53": FUSED, "span=54": FUSED, "lg-pass": FUSED, "lg-fail": FUSED, "q-binds": FUSED, "prefix-rounds": FUSED,
    "x-min-2^-30": FUSED, "x-below-2^-30": FUSED, "x-max-2^31": FUSED, "x-at-2^31": FUSED,
    "pv0-only": ("templated",), "zeros": CLASSES, "neg-zero": CLASSES, "negative": CLASSES, "mixed-sign": CLASSES, "adc": CLASSES,
    "cv-clamped": CLASSES, "delta=0": CLASSES, "tstat-tie": CLASSES, "n=2w-1": CLASSES, "n=2w": CLASSES, "no-boundary": CLASSES,
}
WPR_OF = {"repair-cross-warp": (2, 4)}


def _tstat_parts(x, w):
    """compute_tstat's combined_var (before the clamp) and delta_mean at every position it fills, in the reference's promotions"""
    n = x.shape[0]
    if n < 2 * w or w < 2:
        return np.zeros(0, np.float32), np.zeros(0, np.float32)
    S = np.concatenate([[0.0], np.cumsum(x.astype(np.float64))])
    Q = np.concatenate([[0.0], np.cumsum((x * x).astype(np.float32).astype(np.float64))])
    i = np.arange(w, n - w + 1)
    wf = np.float32(w)
    sum1, sq1 = S[i] - S[i - w], Q[i] - Q[i - w]
    sum2, sq2 = (S[i + w] - S[i]).astype(np.float32), (Q[i + w] - Q[i]).astype(np.float32)
    m1 = (sum1 / np.float64(wf)).astype(np.float32)
    m2 = (sum2 / wf).astype(np.float32)
    cv = sq1 / np.float64(wf) - (m1 * m1).astype(np.float64) + (sq2 / wf).astype(np.float64) - (m2 * m2).astype(np.float64)
    return cv.astype(np.float32), (m2 - m1).astype(np.float32)


def read_edges(r: EdgeRead, tr: Trace, pred: Prediction, lanes: int, warm: int, cap: int) -> set:
    """the edge kinds one read reaches under one parameter set and one lane count"""
    x, n = r.x, r.x.shape[0]
    p = tr.prm[0]
    w1, w2 = int(p["window_length1"]), int(p["window_length2"])
    e = set()
    rngs = lane_ranges(n, lanes, warm)
    seg = seg_len(n, lanes)
    if len(rngs) < lanes:
        e.add("idle-lanes")
    last = rngs[-1][2] - rngs[-1][1]
    if last == 1:
        e.add("last-lane=1")
    if last < w2:
        e.add("last-lane<w2")
    if n >= 32 * lanes - 1:
        d = (n + 1) % (32 * lanes) - 1
        if d in (-1, 0, 1):
            e.add(f"n=32L{d:+d}")
    if any(b0 - a0 > seg for a0, b0, _ in rngs):
        e.add("warm>seg")
    if pred.repairs >= 1:
        e.add("repair")
    if pred.repairs >= 2:
        e.add("repair-rounds>1")
    if pred.cross_warp:
        e.add("repair-cross-warp")
    if pred.pv0_only:
        e.add("pv0-only")
    if pred.path == "slice":
        e.add("slice-overflow")
        if pred.R == 0:
            e.add("R=0")
    g = guard(x)
    span = max(g.span_x, g.span_q)
    if g.exact and span == 53:
        e.add("span=53")
    if not g.exact and g.okx and span == 54:
        e.add("span=54")
    if g.okx and not g.okq:
        e.add("q-binds")
    if g.exact and span == 53 and n == (1 << (g.lg)) - 1:
        e.add("lg-pass")
    if not g.exact and span == 54 and n == 1 << (g.lg - 1):
        e.add("lg-fail")
    if g.evn == 97 and g.exact:
        e.add("x-min-2^-30")
    if g.evn == 96 and not g.okx:
        e.add("x-below-2^-30")
    if g.evx == 157 and g.exact:
        e.add("x-max-2^31")
    if g.evx == 158 and not g.okx:
        e.add("x-at-2^31")
    if len(tr.boundaries) and float((x * x).max()) < 2.0 ** 30:
        # the sequential FP64 prefix of the squares rounds at some boundary (exact sums as integers in units of 2^-23)
        q = (x * x).astype(np.float32)
        qi = np.concatenate([[0], np.cumsum(np.rint(q.astype(np.float64) * 2.0 ** 23).astype(np.int64))])
        Qd = np.concatenate([[0.0], np.cumsum(q.astype(np.float64))])
        if np.all(q.astype(np.float64) * 2.0 ** 23 == np.rint(q.astype(np.float64) * 2.0 ** 23)):
            if any(int(qi[b]) != int(Qd[b] * 2.0 ** 23) for b in tr.boundaries):
                e.add("prefix-rounds")
    if (x == 0).any() and (x.view(np.uint32) == 0).any() and g.exact:
        e.add("zeros")
    if (x.view(np.uint32) == 0x80000000).any() and g.exact:
        e.add("neg-zero")
    if (x < 0).all() and g.exact:
        e.add("negative")
    if (x < 0).any() and (x > 0).any() and g.exact:
        e.add("mixed-sign")
    if r.name.startswith("adc") and g.exact:
        e.add("adc")
    for w, t in ((w1, tr.t1), (w2, tr.t2)):
        if w >= 2 and n == 2 * w - 1:
            e.add("n=2w-1")
        if w >= 2 and n == 2 * w:
            e.add("n=2w")
        cv, dm = _tstat_parts(x, w)
        if (cv < np.float32(1.1754944e-38)).any():
            e.add("cv-clamped")
        if ((dm == 0) & (cv >= np.float32(2.0 ** -60))).any():
            e.add("delta=0")
        if w >= 2 and ((t[1:] == t[:-1]) & (t[1:] > 0)).any():
            e.add("tstat-tie")
    if len(tr.boundaries) == 0:
        e.add("no-boundary")
    return e


CONFIGS = [(1, None), (2, None), (4, None), (1, "1"), (2, "31"), (4, "33"), (2, "0")]      # (WPR, $NPH_EVENTS_WARMUP)


def fingerprint(x, prm) -> str:
    return hashlib.sha1(np.ascontiguousarray(x, np.float32).tobytes() + prm.tobytes()).hexdigest()


def events_hash(start, length, mean, stdv) -> str:
    h = hashlib.sha1()
    for a, dt in ((start, np.uint64), (length, np.float32), (mean, np.float32), (stdv, np.float32)):
        h.update(np.ascontiguousarray(a, dt).tobytes())
    return h.hexdigest()


def check_edges(port, reads=None, configs=CONFIGS):
    """Run every read under every parameter set and configuration on the port oracle, confirm each read's claims and the
    invariants, and return (coverage {(wpr, class): set of edges}, claimed cells, predictions {(read, param, config): Prediction})."""
    reads = edge_reads() if reads is None else reads
    cover = {(w, c): set() for w in WPRS for c in CLASSES}
    preds = {}
    reached_by_read = {r.name: set() for r in reads}
    for pname, prm in PARAMS.items():
        cls = window_class(prm)
        for r in reads:
            tr = Trace(port, r.x, prm)
            b = tr.boundaries
            n = r.x.shape[0]
            # strictly increasing, >= 2 apart, within [2, n - 2]: at most max(1, n // 2) events, inside the room
            assert np.all(np.diff(b) >= 2) and (len(b) == 0 or (b[0] >= 2 and b[-1] <= n - 2)), f"{r.name} {pname}: boundaries {b}"
            assert tr.events.shape[0] <= max(1, n // 2) <= room(n), f"{r.name} {pname}: {tr.events.shape[0]} events"
            if pname == "densest" and n >= 2:
                assert len(b) == (n - 2) // 2, f"{r.name}: densest set gives {len(b)} boundaries"
            for wpr, wenv in configs:
                lanes, warm = 32 * wpr, warm_of(wenv)
                pr = predict(tr, lanes, warm, room(n))
                preds[(r.name, pname, (wpr, wenv))] = pr
                e = read_edges(r, tr, pr, lanes, warm, room(n))
                if wenv is not None and int(wenv) % 32:
                    e.add(f"warm={wenv}")
                for k in e:
                    if cls in APPLIES.get(k, CLASSES) and wpr in WPR_OF.get(k, WPRS):
                        cover[(wpr, cls)].add(k)
                reached_by_read[r.name] |= e
    for r in reads:
        assert r.claims <= reached_by_read[r.name], f"{r.name} misses {sorted(r.claims - reached_by_read[r.name])}"
    claimed = set()
    for r in reads:
        for k in r.claims | {"slice-overflow", "no-boundary"}:
            for w in WPR_OF.get(k, WPRS):
                for c in APPLIES[k]:
                    claimed.add((w, c, k))
    return cover, claimed, preds


def coverage_table(cover, claimed) -> str:
    kinds = sorted({k for _, _, k in claimed} | set().union(*cover.values()))
    cells = [(w, c) for w in WPRS for c in CLASSES]
    head = "edge".ljust(20) + " ".join(f"{w}/{c[:5]}".rjust(10) for w, c in cells)
    rows = [head]
    for k in kinds:
        rows.append(k.ljust(20) + " ".join(("x" if k in cover[(w, c)] else ("MISSING" if (w, c, k) in claimed else ".")).rjust(10)
                                           for w, c in cells))
    return "\n".join(rows)


def batch_stats(preds, reads, pname, config):
    """the device's $NPH_EVENTS_STATS line for one batch: (repair walks, streaming fallback, guard/slice)"""
    ps = [preds[(r.name, pname, config)] for r in reads]
    return (sum(p.repairs for p in ps), sum(p.path != "fast" for p in ps), sum(p.path in ("guard", "slice") for p in ps))
