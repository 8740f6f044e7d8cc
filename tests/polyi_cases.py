"""detect-polyi test inputs and checkers: synthetic poly(I)/poly(A) reads, crafted edge reads, the compiled reference's
detect-polyi pieces (oracle/_ref/libnpref_polyi.so, built by oracle/polya.mk) and a plain Python restatement of its
segmentation HMM and Bernoulli stage.  Reads, packing and glibc's expf / logf come from polya_cases: a read here is the same
PolyaRead that estimate_polya_for_single_read and dpi_estimate_polya_for_single_read both see after loading."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from tests import polya_cases as pc
from tests.polya_cases import PolyaRead, _expf, _logf, f32

REF_POLYI = os.path.join(pc.ROOT, "oracle", "_ref", "libnpref_polyi.so")


class RefPolyi(pc.RefTail):
    """The reference's own detect-polyi functions (oracle/detect_polyi_harness.cpp)."""

    def __init__(self):
        super().__init__(REF_POLYI, "polyi", 2)

    def read(self, r: PolyaRead):
        """(seg u64[5], (read_rate, polya_length), qc, (polyi, polya), detected, row); the numbers are None for a failed load"""
        bern = np.zeros(2, np.int32); det = C.c_int()
        seg, rl, qc, row = super().read(r, bern.ctypes.data, C.byref(det))
        if seg is None:
            return None, None, 4, None, None, row
        return seg, rl, qc, (int(bern[0]), int(bern[1])), det.value, row


# ---- synthetic reads ------------------------------------------------------------------------------------------------------
def synth_polyi_read(rng, name: str, n_samples: int, polyi_frac=None, **kw) -> PolyaRead:
    """A polya_cases read whose tail is split at one level into a wide (sigma ~5.3, poly(I)) part and then a narrow
    (sigma ~3.3, poly(A)) part; polyi_frac is the wide part's share (0: poly(A) only, 1: poly(I) only)."""
    f = rng.dirichlet([1.0, 1.5, 3.0, 3.0, 6.0])
    lens = np.maximum(1, np.floor(f * n_samples)).astype(np.int64)
    lens[-1] = n_samples - lens[:-1].sum()
    if lens[-1] < 1 or n_samples < 5:
        return pc.synth_read(rng, name, n_samples, **kw)
    r = pc.synth_read(rng, name, n_samples, regions=list(zip("SLAPT", (int(v) for v in lens))), **kw)
    frac = float(rng.choice([0.0, 0.3, 0.5, 0.8, 1.0])) if polyi_frac is None else polyi_frac
    lo = int(lens[:3].sum())
    hi = lo + int(lens[3])
    k = lo + int(round((hi - lo) * frac))
    v = np.concatenate([rng.normal(108.498, 5.3, k - lo), rng.normal(108.883, 3.3, hi - k)])
    r.samples[lo:hi] = pc.quantise(r.shift + r.scale * v + (r.var - 1.0) * (v - 108.7) * 0.5)
    return r


# ---- crafted reads: exact bit sequences in the tail ------------------------------------------------------------------------
# With scale 1, shift 0 and var 1 a sample is its own scaled value.  A tail whose samples are `one` = 109 (bit 1) or
# alternately one - 6 and one + 6 (bit 0) has a mean near `one`, so the centred values are near 108 (lI / lA ~1.2 > 1) and
# near 102 / 114 (< 1), far from the bit's thresholds (~105.1 and ~113.2), while the mixture POLYA emission still beats
# TRANSCRIPT on all three.
def _tail(bits, one=109.0) -> np.ndarray:
    out = np.empty(len(bits), np.float64)
    z = 0
    for i, b in enumerate(bits):
        if b:
            out[i] = one
        else:
            out[i] = one + (-6.0 if z & 1 == 0 else 6.0); z += 1
    return out


def crafted_read(rng, name: str, tail_len: int, head=(300, 600, 1500), n_transcript=600, one=109.0, **kw) -> PolyaRead:
    """START / LEADER / ADAPTER drawn at the HMM's levels, then tail_len samples at `one`, then TRANSCRIPT near 80."""
    s = rng.normal(70.2737, 1.5, head[0])
    ld = rng.normal(110.973, 2.0, head[1])
    ad = rng.normal(63.3126, 1.5, head[2])
    tr = rng.normal(79.679, 2.0, n_transcript)
    v = np.concatenate([s, ld, ad, np.full(tail_len, one), tr]).astype(np.float32)
    nk = max(20, v.shape[0] // 40)
    dur, ms, me = pc.event_table(rng, nk, 3012.0, zero_median=kw.pop("zero_median", False))
    r = PolyaRead(name, v, 3012.0, 1.0, 0.0, 1.0, dur, ms, me, **kw)
    r.one = one
    return r


def fit_tail(ref: RefPolyi, r: PolyaRead, want_len: int, bits_fn=None, tries: int = 6) -> PolyaRead:
    """Grow or shrink the designed tail until the reference's segmentation gives a tail of want_len samples
    ([adapter + 1, polya)), then lay bits_fn(want_len) over exactly those samples (the caller asserts what it needed)."""
    tail_lo = None
    for _ in range(tries):
        seg = ref.read(r)[0]
        ad, pa = int(seg[2]), int(seg[3])
        got = pa - (ad + 1)
        tail_lo = ad + 1
        if got == want_len:
            break
        d = want_len - got
        if d > 0:
            r.samples = np.concatenate([r.samples[:pa], np.full(d, r.one, np.float32), r.samples[pa:]])
        else:
            r.samples = np.concatenate([r.samples[:pa + d], r.samples[pa:]])
    if bits_fn is not None:
        r.samples[tail_lo:tail_lo + want_len] = _tail(bits_fn(want_len), r.one).astype(np.float32)
    return r


def centred(r: PolyaRead, start: int, stop: int, i: int):
    """the centred value s of sample i of the tail [start, stop) (:663-664)"""
    return f32(f32(f32((float(r.samples[i]) - r.shift) / r.scale) - _restated_mean(r, start, stop)) + f32(108.0))


def place_centred(r: PolyaRead, start: int, stop: int, targets):
    """Set tail samples so that their centred values are exactly the given floats: {index: s}.  The tail's mean moves with
    them, so this iterates, stepping each sample by ulps until its centred value is exact (scale 1, shift 0)."""
    for _ in range(8):
        done = True
        mean = _restated_mean(r, start, stop)
        for i, s in targets.items():
            y = f32(f32(s) - f32(108.0) + mean)
            for _ in range(64):
                r.samples[i] = y
                got = f32(f32(y - mean) + f32(108.0))
                if got == f32(s):
                    break
                y = np.nextafter(y, np.float32(np.inf) if got < f32(s) else np.float32(-np.inf))
            done &= _restated_mean(r, start, stop) == mean
        if done and all(centred(r, start, stop, i) == f32(s) for i, s in targets.items()):
            return r
    raise AssertionError(f"{r.name}: centred values not placed")


def edge_reads(rng, ref: RefPolyi):
    """Reads at the corners of detect-polyi's arithmetic (the conditions test_detect_polyi_oracle asserts are reached).  Crafted
    against the compiled reference, so they need it."""
    out = []
    zeros_then_ones = lambda nz: (lambda m: [0] * nz + [1] * (m - nz))
    ones = lambda m: [1] * m
    zeros = lambda m: [0] * m
    # tails of 99, 100 and 101 samples (stop - start < 100 gives {-1, -1})
    for m in (99, 100, 101):
        out.append(fit_tail(ref, crafted_read(rng, f"tail_{m}", m + 1), m, ones))
    # polyi at 200 and 201 (POLYI-ONLY needs polyi > 200), with a long poly(A) part after it: A+I and POLYA-ONLY
    for k in (199, 200, 201, 202):
        out.append(fit_tail(ref, crafted_read(rng, f"polyi_{k}", 701), 700, zeros_then_ones(k)))
    # region_length - polya at 200 and 201 (POLYA-ONLY needs > 200), after a poly(I) part
    for nz in (498, 499, 500, 501):
        out.append(fit_tail(ref, crafted_read(rng, f"polya_rest_{nz}", 701), 700, zeros_then_ones(nz)))
    # an all-poly(I) tail (POLYI-ONLY) and a short one that finds nothing (NONE)
    out.append(fit_tail(ref, crafted_read(rng, "all_polyi", 801), 800, zeros))
    out.append(fit_tail(ref, crafted_read(rng, "short_polya", 251), 250, ones))
    # centred samples at and just beyond the clamp bounds.  In [184, 200] both densities underflow, so lI / lA is
    # -inf / -inf = NaN and the bit 0.  The raw samples must stay inside the POLYA region for the segmentation, which clamps
    # raw values outside [40, 200] to 100: a tail at 109 puts s = 200 at a raw 201 (clamped there too), a tail at 107 puts
    # s = 40 at a raw 39.  Near 40 the centred value moves in steps of 2^-17 (y - mean is rounded at 68), so its neighbours
    # are two float ulps away.
    for name, one, ss in (("clamp_high", 109.0, (200.0, 200.00002, 199.99998)), ("clamp_low", 107.0, (40.0, 39.999992, 40.000008))):
        r = fit_tail(ref, crafted_read(rng, name, 1201, one=one), 1200)
        lo = int(ref.read(r)[0][2]) + 1
        out.append(place_centred(r, lo, lo + 1200, {lo + 300 + 40 * i: np.float32(s) for i, s in enumerate(ss)}))
    # the shortest reads; short_5 reaches the sentinel fallback, so its tail is [n-1, n-1) (NONE)
    for n in (2, 3, 4, 5):
        out.append(pc.synth_read(rng, f"short_{n}", n, n_kmers=3))
    # a median duration of 0 on a read with a detected tail
    out.append(fit_tail(ref, crafted_read(rng, "zero_median", 701, zero_median=True), 700, zeros_then_ones(300)))
    # a read that failed to load
    r = pc.synth_read(rng, "failed_load", 100)
    r.loaded = False
    out.append(r)
    return out


def _restated_mean(r: PolyaRead, start: int, stop: int):
    acc = f32(0.0)
    for x in r.samples[start:stop]:
        acc = f32(acc + f32((float(x) - r.shift) / r.scale))
    return f32(acc / f32(stop - start))


# ---- Python restatement (float32, glibc's expf / logf) ----------------------------------------------------------------------
_ISP = f32(0.3989422804014327)


def _pdf(x, mean, sd):
    a = (x - mean) / sd
    return (_ISP / sd) * _expf((f32(-0.5) * a) * a)


def restate_segment(samples, scale, shift, var, sentinel_rule=True):
    """DPISegmentationHMM::segment_squiggle (src/nanopolish_detect_polyi.cpp:177-518): polya_cases.restate_segment with the
    POLYA emission an even mixture of two Gaussians (:291-295)."""
    scale, shift, var = f32(scale), f32(shift), f32(var)
    G = {"s": (70.2737, 3.7743), "l": (110.973, 5.237), "a0": (79.347, 8.3702), "a1": (63.3126, 2.7464), "p0": (108.883, 3.257),
         "p1": (108.498, 5.257), "t0": (79.679, 6.966), "t1": (105.784, 16.022)}
    g = {}
    for k, (m, s) in G.items():
        sd = var * f32(s)
        g[k] = (shift + scale * f32(m), sd, _logf(sd))
    lisp = f32(np.log(0.3989422804014327))
    pdf = lambda x, k: _pdf(x, g[k][0], g[k][1])

    def lpdf(x, k):
        m, s, ls = g[k]
        a = (x - m) / s
        return (lisp - ls) + ((f32(-0.5) * a) * a)

    def emit(x):
        x = f32(x)
        xx = f32(100.0) if (x > f32(200.0) or x < f32(40.0)) else x
        return [_logf(f32(0.5) * pdf(xx, "s") + f32(0.5) * f32(0.00476)), lpdf(xx, "l"),
                _logf(f32(0.874) * pdf(xx, "a0") + f32(0.126) * pdf(xx, "a1")),
                _logf(f32(0.5) * pdf(xx, "p0") + f32(0.5) * pdf(xx, "p1")),
                f32(-4.2485) if (xx > f32(70.0) and xx < f32(140.0)) else f32(-np.inf),
                _logf(f32(0.346) * pdf(xx, "t0") + f32(0.654) * pdf(xx, "t1"))]

    lt = lambda p: _logf(f32(p))
    SS, SL, LL, LA, AA, AP, PP, PC, PT, CP, CC, TT = (lt(0.10), lt(0.90), lt(0.90), lt(0.10), lt(0.95), lt(0.05), lt(0.89),
                                                      lt(0.01), lt(0.10), lt(0.99), lt(0.01), lt(1.00))
    mx = lambda a, b: b if a < b else a
    n = len(samples)
    e = emit(samples[n - 1])
    v = [f32(0.0) + e[0], f32(-np.inf) + e[1], f32(-np.inf), f32(-np.inf), f32(-np.inf), f32(-np.inf)]
    bp = [None] * n
    with np.errstate(all="ignore"):
        for i in range(1, n):
            e = emit(samples[i])
            s_s, s_l, l_l, l_a = v[0] + SS, v[0] + SL, v[1] + LL, v[1] + LA
            a_a, a_p, p_p, p_c, p_t = v[2] + AA, v[2] + AP, v[3] + PP, v[3] + PC, v[3] + PT
            c_c, c_p, t_t = v[4] + CC, v[4] + CP, v[5] + TT
            v = [s_s + e[0], mx(l_l, s_l) + e[1], mx(a_a, l_a) + e[2], mx(p_p, mx(a_p, c_p)) + e[3], mx(c_c, p_c) + e[4], mx(p_t, t_t) + e[5]]
            bP = 3 if (a_p < p_p and c_p < p_p) else (2 if (p_p < a_p and c_p < a_p) else 4)
            bp[i] = (0, 1 if s_l < l_l else 0, 2 if l_a < a_a else 1, bP, 4 if p_c < c_c else 3, 5 if p_t < t_t else 3)
    reg = [0] * n
    reg[n - 1] = 5
    for j in range(n - 2, 0, -1):
        reg[j] = bp[j][reg[j + 1]]
    ix = [0, 1, 2, 3, 0]
    for i in range(n):
        nx = reg[i + 1] if i + 1 < n else -1
        if reg[i] == 0 and nx == 1: ix[0] = i
        if reg[i] == 1 and nx == 2: ix[1] = i
        if reg[i] == 2 and nx == 3: ix[2] = i
        if reg[i] == 3 and nx == 5: ix[3] = i
        if reg[i] == 4: ix[4] += 1
    if sentinel_rule and (ix[1] == 1 or ix[2] == 2 or ix[3] == 3):
        ix[1], ix[2], ix[3] = (n - 3) % (1 << 64), n - 2, n - 1
    return tuple(ix)


def restate_bits(r: PolyaRead, start: int, stop: int):
    """BernoulliHMM::log_lkhd_ratio_sequence (:652-675) over samples [start, stop), scaled in double (:737-740)"""
    y = [f32((float(x) - r.shift) / r.scale) for x in r.samples[start:stop]]
    mean = f32(0.0)
    for v in y:
        mean = f32(mean + v)
    mean = f32(mean / f32(len(y)))
    bits = []
    with np.errstate(all="ignore"):
        for v in y:
            s = f32(f32(v - mean) + f32(108.0))
            xx = f32(100.0) if (s > f32(200.0) or s < f32(40.0)) else s
            lI = _logf(_pdf(xx, f32(108.498), f32(5.257)))
            lA = _logf(_pdf(xx, f32(108.883), f32(3.257)))
            bits.append(1 if f32(lI / lA) > f32(1.0) else 0)
    return bits


def restate_bernoulli(r: PolyaRead, start: int, stop: int):
    """BernoulliHMM::segmentation (:728-756) with its viterbi (:678-725) as written: (polyi, polya)"""
    if stop - start < 100:
        return -1, -1
    b = restate_bits(r, start, stop)
    n = len(b)
    lt = lambda p: _logf(f32(p))
    II, IA, AA = lt(0.90), lt(0.10), lt(1.00)
    em = {(0, 1): lt(0.72304), (0, 0): _logf(f32(1.0) - f32(0.72304)), (1, 1): lt(0.92154), (1, 0): _logf(f32(1.0) - f32(0.92154))}
    vI, vA = f32(0.0) + em[(0, b[0])], f32(-np.inf) + em[(1, b[0])]
    bpA = [1] * n
    with np.errstate(all="ignore"):
        for i in range(1, n):
            i2i, i2a, a2a = vI + II, vI + IA, vA + AA
            vI, vA = i2i + em[(0, b[i])], (a2a if i2a < a2a else i2a) + em[(1, b[i])]
            bpA[i] = 0 if a2a < i2a else 1
    reg = [0] * n
    reg[n - 1] = 1 if vI < vA else 0
    for j in range(n - 2, 0, -1):
        reg[j] = 0 if reg[j + 1] == 0 else bpA[j]
    polyi = polya = -1
    for i, lab in enumerate(reg):
        if lab == 0:
            polyi = i
        if lab == 1 and polya < 0:
            polya = i
    return polyi, polya


def restate_detected(polyi: int, polya: int, region_length: int) -> int:
    """post_boolhmm_detetection_qc (:973-997) as NPH_POLYI_*"""
    polyi_found = polyi > 200
    polya_found = polya > 0 and region_length - polya > 200
    return (2 if polyi_found else 0) | (1 if polya_found else 0)
