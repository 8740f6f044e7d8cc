"""Poly(A) test inputs and checkers: synthetic direct-RNA-like reads, the compiled reference's poly(A) pieces
(oracle/_ref/libnpref_polya.so, built by oracle/polya.mk) and a small Python restatement of segment_squiggle.

A read here is what estimate_polya_for_single_read sees after loading: the whole raw signal in acquisition order, the
scalings, the event durations and the base-to-event map."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200.synth import EVENT_RANGE_DT, POLYA_JOB_DT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_POLYA = os.path.join(ROOT, "oracle", "_ref", "libnpref_polya.so")
ADC_STEP = np.float32(1400.0 / 8192.0)     # picoamps per ADC step: range / digitisation

# (level, stdv) of each region at the HMM's own parameters (src/nanopolish_polya_estimator.cpp:232-250)
LEVELS = {"S": (70.2737, 3.7743), "L": (110.973, 5.237), "A": (79.347, 8.3702), "P": (108.883, 3.257), "T": (95.0, 14.0)}


@dataclass
class PolyaRead:
    name: str
    samples: np.ndarray                  # float32
    sample_rate: float
    scale: float
    shift: float
    var: float
    duration: np.ndarray                 # float32 per event
    map_start: np.ndarray                # int32 per k-mer
    map_stop: np.ndarray
    suffix_clip: int = 0
    contig: str = "chr1"
    pos: int = 0
    loaded: bool = True
    flag: int = 0


def quantise(v) -> np.ndarray:
    return (np.round(np.asarray(v, np.float64) / float(ADC_STEP)).astype(np.float32) * ADC_STEP).astype(np.float32)


def event_table(rng, n_kmers: int, sample_rate: float, unmapped: float = 0.05, zero_median: bool = False):
    """Event durations (whole samples / rate, as load_from_raw forms them) and a monotone base-to-event map."""
    n_events = max(1, int(n_kmers * rng.uniform(1.2, 2.0)))
    dur = (rng.integers(3, 40, n_events).astype(np.float64) / sample_rate).astype(np.float32)
    start = np.full(n_kmers, -1, np.int32)
    stop = np.full(n_kmers, -1, np.int32)
    if not zero_median:
        e = 0
        for k in range(n_kmers):
            if rng.random() < unmapped or e >= n_events:
                continue
            span = int(rng.integers(0, 3))
            s = e
            t = min(n_events - 1, e + span)
            start[k], stop[k] = s, t
            e = t + int(rng.integers(0, 2))
    return dur, start, stop


def synth_read(rng, name: str, n_samples: int, regions=None, n_kmers=None, cliffs: float = 0.002, spikes: float = 0.0005,
               sample_rate: float = 3012.0, **kw) -> PolyaRead:
    """START / LEADER / ADAPTER / POLYA (with CLIFF spikes) / TRANSCRIPT at the HMM's levels, through the read's scalings,
    quantised to an ADC grid (so exact ties occur), plus out-of-range spikes."""
    scale = float(kw.pop("scale", rng.uniform(0.9, 1.1)))
    shift = float(kw.pop("shift", rng.uniform(-3.0, 3.0)))
    var = float(kw.pop("var", rng.uniform(0.8, 1.3)))
    if regions is None:
        f = rng.dirichlet([1.0, 1.5, 3.0, 3.0, 6.0])
        regions = [("S", f[0]), ("L", f[1]), ("A", f[2]), ("P", f[3]), ("T", f[4])]
    lens = np.array([r[1] for r in regions], np.float64)
    lens = np.maximum(1, np.round(lens / lens.sum() * n_samples)).astype(np.int64)
    lens[-1] += n_samples - lens.sum()
    while lens[-1] < 1:
        i = int(np.argmax(lens[:-1])); lens[i] -= 1; lens[-1] += 1
    parts = []
    for (lab, _), ln in zip(regions, lens):
        mu, sd = LEVELS[lab]
        if lab == "A":
            lo = rng.random(ln) < 0.126
            seg = np.where(lo, rng.normal(63.3126, 2.7464, ln), rng.normal(79.347, 8.3702, ln))
        else:
            seg = rng.normal(mu, sd, ln)
        if lab == "P" and cliffs > 0:
            m = rng.random(ln) < cliffs
            seg[m] = rng.uniform(71.0, 139.0, m.sum())
        parts.append(shift + scale * seg * 1.0 + (var - 1.0) * (seg - mu) * 0.5)
    v = np.concatenate(parts)[:n_samples]
    if spikes > 0:
        m = rng.random(n_samples) < spikes
        v[m] = rng.choice([10.0, 35.0, 230.0, 400.0], m.sum())
    samples = quantise(v)
    nk = int(n_kmers if n_kmers is not None else max(20, n_samples // 40))
    dur, ms, me = event_table(rng, nk, sample_rate, zero_median=kw.pop("zero_median", False))
    return PolyaRead(name, samples, sample_rate, scale, shift, var, dur, ms, me, **kw)


def pack(reads):
    """The arrays of one nph_polya_batch call."""
    raw, dur, b2e = [], [], []
    jobs = np.zeros(len(reads), POLYA_JOB_DT)
    so = eo = ro = 0
    for i, r in enumerate(reads):
        j = jobs[i]
        j["sample_off"], j["event_off"], j["rank_off"] = so, eo, ro
        j["n_samples"], j["n_kmers"], j["n_events"] = r.samples.shape[0], r.map_start.shape[0], r.duration.shape[0]
        j["suffix_clip"], j["sample_rate"], j["scale"], j["shift"], j["var"] = r.suffix_clip, r.sample_rate, r.scale, r.shift, r.var
        j["loaded"] = 1 if r.loaded else 0
        raw.append(r.samples); dur.append(r.duration)
        m = np.zeros(r.map_start.shape[0], EVENT_RANGE_DT); m["start"] = r.map_start; m["stop"] = r.map_stop
        b2e.append(m)
        so += r.samples.shape[0]; eo += r.duration.shape[0]; ro += r.map_start.shape[0]
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs)) if xs else np.zeros(0, dt)
    return cat(raw, np.float32), jobs, cat(dur, np.float32), cat(b2e, EVENT_RANGE_DT)


class RefPolya:
    """The reference's own poly(A) functions (oracle/polya_harness.cpp)."""

    def __init__(self):
        self.lib = C.CDLL(REF_POLYA)
        vp, sz = C.c_void_p, C.c_size_t
        self.lib.npref_polya_read.restype = C.c_longlong
        self.lib.npref_polya_read.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_uint32, vp, sz, C.c_double, C.c_double,
                                              C.c_double, C.c_double, vp, sz, vp, vp, sz, vp, vp, vp, vp, sz]
        self.lib.npref_polya_failed_row.restype = C.c_longlong
        self.lib.npref_polya_failed_row.argtypes = [C.c_char_p, C.c_char_p, C.c_int, vp, sz]
        self.lib.npref_polya_time.restype = C.c_double
        self.lib.npref_polya_time.argtypes = [vp, sz, C.c_double, C.c_double, C.c_double, C.c_double, vp, sz, vp, vp, sz]

    def read(self, r: PolyaRead):
        """(seg u64[5], (read_rate, polya_length), qc, row)"""
        buf = C.create_string_buffer(1024)
        if not r.loaded:
            n = self.lib.npref_polya_failed_row(r.name.encode(), r.contig.encode(), r.pos, buf, 1024)
            return None, None, 4, buf.raw[:n].decode()
        seg = np.zeros(5, np.uint64); rl = np.zeros(2, np.float64); qc = C.c_int()
        s = np.ascontiguousarray(r.samples, np.float32); d = np.ascontiguousarray(r.duration, np.float32)
        a = np.ascontiguousarray(r.map_start, np.int32); b = np.ascontiguousarray(r.map_stop, np.int32)
        n = self.lib.npref_polya_read(r.name.encode(), r.contig.encode(), r.pos, r.suffix_clip, s.ctypes.data, s.shape[0],
                                      r.sample_rate, r.scale, r.shift, r.var, d.ctypes.data, d.shape[0], a.ctypes.data, b.ctypes.data,
                                      a.shape[0], seg.ctypes.data, rl.ctypes.data, C.byref(qc), buf, 1024)
        assert n > 0
        return seg, (rl[0], rl[1]), qc.value, buf.raw[:n].decode()

    def time(self, r: PolyaRead) -> float:
        s = np.ascontiguousarray(r.samples, np.float32); d = np.ascontiguousarray(r.duration, np.float32)
        a = np.ascontiguousarray(r.map_start, np.int32); b = np.ascontiguousarray(r.map_stop, np.int32)
        return self.lib.npref_polya_time(s.ctypes.data, s.shape[0], r.sample_rate, r.scale, r.shift, r.var, d.ctypes.data, d.shape[0],
                                         a.ctypes.data, b.ctypes.data, a.shape[0])


def edge_reads(rng):
    """Reads at the corners of the reference's arithmetic."""
    out = []
    base = lambda name, n, **kw: synth_read(rng, name, n, **kw)
    # values exactly at the clamp and CLIFF bounds, and out-of-range spikes
    r = base("exact_bounds", 3000)
    idx = rng.choice(3000, 400, replace=False)
    r.samples[idx] = rng.choice(np.array([40.0, 70.0, 140.0, 200.0, 39.999996, 200.00002, 0.0, -5.0, 1e4], np.float32), 400)
    out.append(r)
    # mixtures that underflow to -inf (START/ADAPTER/TRANSCRIPT far from every level after scaling) and a tiny stdv
    r = base("underflow", 2500, var=0.05, scale=1.0, shift=0.0)
    out.append(r)
    # constant signals
    for v in (40.0, 70.0, 100.0, 108.883, 139.0, 200.0):
        r = base(f"constant_{v}", 1500)
        r.samples[:] = np.float32(v)
        out.append(r)
    # the shortest reads
    for n in (2, 3, 4, 5):
        out.append(base(f"short_{n}", n, n_kmers=3))
    # boundaries at the sentinel indices 1, 2, 3: one sample of START, then LEADER etc.
    for k in (1, 2, 3, 4):
        out.append(base(f"sentinel_{k}", 2400, regions=[("S", k), ("L", k), ("A", 800), ("P", 800), ("T", 800)]))
    # missing regions
    out.append(base("no_polya", 3000, regions=[("S", 300), ("L", 600), ("A", 1500), ("T", 600)]))
    out.append(base("no_adapter", 3000, regions=[("S", 300), ("L", 600), ("P", 1500), ("T", 600)]))
    out.append(base("only_transcript", 3000, regions=[("T", 1)]))
    out.append(base("only_start", 2000, regions=[("S", 1)]))
    # many POLYA <-> CLIFF alternations
    out.append(base("cliffs", 6000, regions=[("S", 300), ("L", 600), ("A", 1500), ("P", 3000), ("T", 600)], cliffs=0.2))
    # suffix clips at the threshold, on reads that otherwise pass
    for clip in (200, 201):
        out.append(base(f"suffclip_{clip}", 12000, regions=[("S", 500), ("L", 1500), ("A", 3000), ("P", 4000), ("T", 3000)],
                        suffix_clip=clip, cliffs=0.0, spikes=0.0))
    # a median duration of 0 (every k-mer unmapped): infinite read rate, NaN length -> 0
    out.append(base("zero_median", 8000, regions=[("S", 500), ("L", 1500), ("A", 2000), ("P", 2500), ("T", 1500)], zero_median=True))
    # a zero median on a read without a poly(A) region: the sentinel fallback makes the tail 0 samples, 0 * inf is NaN, length 0
    out.append(base("zero_median_no_tail", 6000, regions=[("S", 500), ("L", 1500), ("A", 2000), ("T", 2000)], zero_median=True))
    # a long adapter at a fast read rate (ADAPTER)
    r = base("long_adapter", 20000, regions=[("S", 300), ("L", 700), ("A", 15000), ("P", 2500), ("T", 1500)], cliffs=0.0, spikes=0.0)
    r.duration[:] = np.float32(3.0 / r.sample_rate)
    out.append(r)
    # a read that failed to load
    r = base("failed_load", 100)
    r.loaded = False
    out.append(r)
    return out


# ---- Python restatement of segment_squiggle (float32, glibc's expf / logf) ---------------------------------------------
_libm = C.CDLL("libm.so.6")
_libm.expf.restype = C.c_float; _libm.expf.argtypes = [C.c_float]
_libm.logf.restype = C.c_float; _libm.logf.argtypes = [C.c_float]
f32 = np.float32


def _expf(x):
    return f32(_libm.expf(float(x)))


def _logf(x):
    return f32(_libm.logf(float(x)))


def restate_segment(samples, scale, shift, var, sentinel_rule=True):
    """segment_squiggle (src/nanopolish_polya_estimator.cpp:204-509) in plain Python: (start, leader, adapter, polya, cliffs).
    sentinel_rule=False: the boundaries before the sentinel rule (:500-506) replaces them."""
    scale, shift, var = f32(scale), f32(shift), f32(var)
    G = {"s": (70.2737, 3.7743), "l": (110.973, 5.237), "a0": (79.347, 8.3702), "a1": (63.3126, 2.7464), "p": (108.883, 3.257),
         "t0": (79.679, 6.966), "t1": (105.784, 16.022)}
    g = {}
    for k, (m, s) in G.items():
        sd = var * f32(s)
        g[k] = (shift + scale * f32(m), sd, _logf(sd))
    lisp = f32(np.log(0.3989422804014327))
    isp = f32(0.3989422804014327)

    def pdf(x, k):
        m, s, _ = g[k]
        a = (x - m) / s
        return (isp / s) * _expf((f32(-0.5) * a) * a)

    def lpdf(x, k):
        m, s, ls = g[k]
        a = (x - m) / s
        return (lisp - ls) + ((f32(-0.5) * a) * a)

    def emit(x):
        x = f32(x)
        xx = f32(100.0) if (x > f32(200.0) or x < f32(40.0)) else x
        return [_logf(f32(0.5) * pdf(xx, "s") + f32(0.5) * f32(0.00476)), lpdf(xx, "l"),
                _logf(f32(0.874) * pdf(xx, "a0") + f32(0.126) * pdf(xx, "a1")), lpdf(xx, "p"),
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


def restate_rate(r: PolyaRead) -> float:
    d = []
    for s, t in zip(r.map_start, r.map_stop):
        acc = 0.0
        if s != -1:
            for j in range(s, t + 1):
                acc += float(r.duration[j])
        d.append(acc)
    d.sort()
    m = d[len(d) // 2]
    return float("inf") if m == 0.0 else 1.0 / m
