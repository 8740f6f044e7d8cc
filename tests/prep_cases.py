"""Edge cases for the two ends of the raw-read prologue (csrc/squiggle_prep.cu) and the fused load_from_raw driver
(csrc/load_from_raw.cu), and a restatement of the constants and launch geometry they depend on.

trim_kernel takes each chunk's median and MAD with a 128-slot bitonic warp sort (slots past the chunk hold +inf), finds the
varseg_thresh quantile of the MADs by a rank count over the block (ties broken by chunk index), and keeps the chunks between
the first and the last MAD strictly above it.  recalibrate_kernel builds each job's base-to-event map in place with atomics,
picks the 'M' events with ballots over 32-k-mer tiles and a rank carried from tile to tile, sums the normal equations on lane 0
and solves them with Eigen's full-pivot LU written out.  The builders below place inputs on the edges of those steps; each
case lists the edges it claims, and `check_trim_edges` / `check_cal_edges` confirm every claim from the port oracle's own
intermediate values (npo_trim_trace: the MADs, the threshold, the kept chunks; npo_recalibrate_trace: the five sums, the
pivot, the rank branch and the 'M' k-mers), never from what the builder meant to build.

Two edges that look reachable are not, and are stated here instead:
  * no chunk count n < 2^22 makes nextafterf(1, 0) * (n - 1) round up to n - 1 in float (the product is always at least half
    an ulp below n - 1, and rounds down), so a varseg_thresh below 1 never takes quantilef's "p is exactly 1" branch; the
    case with nextafterf(1, 0) interpolates with a remainder just below 1 instead.
  * the reference cannot be asked about a read whose trim keeps no chunk (trim_raw_by_mad asserts), one with fewer samples
    than a chunk (it reads an empty array) or one whose kept end is below trim_end (rt.end wraps as a size_t); such cases
    are compared device against port only and are listed by `trim_deviations`."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200 import synth

# ---- squiggle_prep.cu / load_from_raw.cu constants ---------------------------------------------------------------------
MAX_CHUNK = 128              # kMaxChunk: samples per chunk a warp holds (4 slots x 32 lanes)
TRIM_THREADS = 256           # kTrimThreads: one block per read, 8 warps
TRIM_WARPS = TRIM_THREADS // 32
CAL_WARPS = 8                # kCalWarps: one warp per calibration job
TILE = 32                    # k-mers per ballot tile of the 'M' selection
CONV_WARPS = 8               # kConvWarps: one warp per live read in convert_kernel
BLOCKS_PER_SM = 8            # every grid is capped at sm_count * 8 blocks
MIN_M = 200                  # minNumEventsToRescale
MAX_VAR = 2.5                # MIN_CALIBRATION_VAR
MAX_EPB = 5.0                # events_per_base above which the read fails QC
LFR_TRIM = (200, 10, 100, 0.0)   # load_from_raw's trim_start, trim_end, varseg_chunk, varseg_thresh
MAD_SCALE = np.float32(1.4826)
FLT_MAX = np.float32(3.4028235e38)
K = 6                        # calibration cases use 6-mer nucleotide models


def trim_grid(n_reads: int, sm_count: int) -> int:
    return min(n_reads, sm_count * BLOCKS_PER_SM)


def warp_grid(n_jobs: int, sm_count: int, warps: int = CAL_WARPS) -> int:
    """recalibrate_kernel's and convert_kernel's grid: a warp per job, at most sm_count * 8 blocks"""
    return min((n_jobs + warps - 1) // warps, sm_count * BLOCKS_PER_SM)


def warp_jobs_loop(sm_count: int) -> int:
    """the smallest job count for which some warp takes a second job"""
    return CAL_WARPS * sm_count * BLOCKS_PER_SM + 1


def event_room(n_samples: int) -> int:
    return n_samples // 2 + 8


def quantile_pos(p, n):
    """quantilef's index and remainder, in float as the reference computes them"""
    pos = np.float32(np.float32(p) * np.float32(n - 1))
    idx = int(pos)
    return idx, np.float32(pos - np.float32(idx)), idx < n - 1


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _up(x):
    return np.nextafter(np.float32(x), np.float32(np.inf))


# ---- trim cases -------------------------------------------------------------------------------------------------------
@dataclass
class TrimCase:
    name: str
    x: np.ndarray
    ts: int
    te: int
    chunk: int
    perc: float
    claims: set = field(default_factory=set)

    @property
    def params(self):
        return (self.ts, self.te, self.chunk, float(self.perc))


def fingerprint(x, *params) -> str:
    return hashlib.sha1(_f32(x).tobytes() + repr(tuple(params)).encode()).hexdigest()


def range_hash(ok, s, e) -> str:
    return hashlib.sha1(repr((int(ok), int(s), int(e))).encode()).hexdigest()


def mads_hash(mads, thresh) -> str:
    return hashlib.sha1(_f32(mads).tobytes() + _f32([thresh]).tobytes()).hexdigest()


def _noise_chunks(rng, nchunk, chunk, lo=60.0, hi=130.0, sd=8.0):
    """a step trace: a new level every ~9 samples plus noise, so every chunk has a MAD well above a quiet one's"""
    n = nchunk * chunk
    lev = rng.uniform(lo, hi, n // 9 + 2).repeat(9)[:n]
    return _f32(lev + rng.normal(0.0, sd, n))


def _quiet(rng, n, level=200.0, sd=0.5):
    return _f32(level + rng.normal(0.0, sd, n))


def mad_chunk(d, rng, chunk=101):
    """an odd chunk with median exactly 0.0 and unscaled MAD exactly d (float): 50 samples below zero, 0.0, 50 above; the
    absolute deviations are the samples' magnitudes, 49 below d, d itself, 50 above"""
    d = np.float32(d)
    assert chunk == 101
    small = _f32(rng.uniform(0.1, 0.9, 49) * d)
    large = _f32(rng.uniform(1.1, 3.0, 50) * d)
    neg = np.concatenate([-small[:25], -large[:25]])
    pos = np.concatenate([small[25:], [d], large[25:]])
    x = _f32(np.concatenate([neg, [0.0], pos]))
    rng.shuffle(x)
    return x


def mad_of_d(d):
    return np.float32(np.float32(d) * MAD_SCALE)


def d_for_mad(target):
    """the smallest float d with fl(d * 1.4826f) == target (searched upwards from target / 1.4826)"""
    d = np.float32(target / 1.4826) * np.float32(0.99999)
    while mad_of_d(d) < target:
        d = _up(d)
    assert mad_of_d(d) == target, "no d gives that MAD"
    return d


def _mix(remf, lo, hi, double_product=False):
    """quantilef's interpolation: (1.0 - remf) * lo in double plus remf * hi in float (or, double_product, in double)"""
    a = np.float64(1.0 - np.float64(remf)) * np.float64(lo)
    b = np.float64(remf) * np.float64(hi) if double_product else np.float64(np.float32(remf * hi))
    return np.float32(a + b)


def _mix_product_read(rng):
    """a read whose one kept chunk is kept only because remf * hi is rounded in float: varseg_thresh nextafterf(1, 0) puts the
    threshold between the two largest MADs lo < hi with a remainder just below 1; the float product gives the float below hi,
    the double product would give hi itself.  The chunk with MAD hi leads the read."""
    p = np.nextafter(np.float32(1), np.float32(0))
    srch = np.random.default_rng(6279)
    while True:
        n = int(srch.integers(3, 40))
        idx, remf, _ = quantile_pos(p, n)
        hi = np.float32(srch.uniform(8, 16))
        lo = np.float32(hi * (1 - srch.uniform(0, 1e-4)))
        if idx != n - 2 or not lo < hi or _mix(remf, lo, hi) != np.nextafter(hi, np.float32(0)) or _mix(remf, lo, hi, True) != hi:
            continue
        try:
            dl, dh = d_for_mad(lo), d_for_mad(hi)
        except AssertionError:
            continue
        rest = [mad_chunk(d, rng) for d in np.float32(rng.uniform(0.5, 0.9, n - 2)) * dl]
        return (np.concatenate([mad_chunk(dh, rng)] + rest + [mad_chunk(dl, rng)]),)


def trim_cases() -> list:
    rng = np.random.default_rng(2024)
    cases = []

    def add(name, x, ts, te, chunk, perc, *claims):
        cases.append(TrimCase(name, _f32(x), ts, te, chunk, float(np.float32(perc)), set(claims)))

    # every chunk size the warp sort takes, odd (exact median) and even (interpolated): a quiet leader, a body, a quiet tail
    for c in range(2, MAX_CHUNK + 1):
        body = _noise_chunks(rng, 7, c)
        x = np.concatenate([_quiet(rng, c), body, _quiet(rng, c, 190.0), rng.normal(100, 5, c - 1 if c % 3 == 0 else 0)])
        add(f"chunk{c}", x, c // 3, c // 5, c, 0.0 if c % 2 else 0.37, "chunk-odd" if c % 2 else "chunk-even")

    # sample counts around the chunk
    for c in (100, 37):
        for ns, tag in ((0, "ns=0"), (c - 1, "ns=chunk-1"), (c, "ns=chunk"), (7 * c - 1, "ns=m*chunk-1"), (7 * c, "ns=m*chunk"),
                        (7 * c + c - 1, "ns=m*chunk+chunk-1")):
            x = np.concatenate([_quiet(rng, min(ns, c)), _noise_chunks(rng, 8, c)])[:ns]
            add(f"ns{ns}-c{c}", x, 20, 10, c, 0.0, tag)

    # chunk counts: warp stride (8k +- 1), the rank count's block stride (255-257, 513), and one long read
    for nch in (1, 2, 3, 7, 9, 15, 17, 255, 256, 257, 513):
        x = np.concatenate([_quiet(rng, 16), _noise_chunks(rng, max(nch - 1, 0), 16)])
        add(f"nchunk{nch}", x, 5, 3, 16, 0.0 if nch < 100 else 0.2)
    x = np.concatenate([_quiet(rng, 8 * 40), _noise_chunks(rng, 10_000, 8), _quiet(rng, 8 * 25)])
    add("nchunk-long", x, 200, 10, 8, 0.05)

    # perc
    body = np.concatenate([_quiet(rng, 100), _noise_chunks(rng, 12, 100, sd=3.0), _noise_chunks(rng, 8, 100, sd=12.0)])
    add("perc0", body, 200, 10, 100, 0.0, "perc=0")
    add("perc1", np.concatenate([_noise_chunks(rng, 6, 64, sd=3), _noise_chunks(rng, 1, 64, sd=20), _noise_chunks(rng, 5, 64, sd=3)]),
        10, 10, 64, 1.0, "perc=1")
    add("perc-exact-0.25", _noise_chunks(rng, 9, 50), 0, 0, 50, 0.25, "perc-exact-index")
    add("perc-exact-0.75", _noise_chunks(rng, 13, 51), 3, 3, 51, 0.75, "perc-exact-index")
    n = 201
    add("perc-rem-near-1", _noise_chunks(rng, n, 20), 7, 7, 20, np.float32(7.995 / (n - 1)), "perc-rem-near-1")
    add("perc-1-ulp", _noise_chunks(rng, 40, 30), 0, 0, 30, np.nextafter(np.float32(1), np.float32(0)), "perc-1-ulp")
    add("perc-min-float", body, 0, 0, 100, np.float32(1.4e-45), "perc=min-float")
    add("mix-product", *_mix_product_read(rng), 3, 2, 101, np.nextafter(np.float32(1), np.float32(0)), "mix-product-decides")

    # ranges decided by one ulp: with perc 0 the threshold is the smallest MAD, the MAD of a middle chunk R
    for end in ("lead", "trail"):
        d0 = np.float32(3.0)
        thr = mad_of_d(d0)
        R = mad_chunk(d0, rng)
        big = [_noise_chunks(rng, 1, 101, lo=-10, hi=10, sd=20.0) for _ in range(4)]
        eq = mad_chunk(d0, rng)                          # same MAD as R: at the threshold, so trimmed
        above = mad_chunk(d_for_mad(_up(thr)), rng)      # one ulp above: kept
        for tag, edge in (("eq", eq), ("ulp", above)):
            parts = [edge, big[0], big[1], R, big[2], big[3]]
            if end == "trail":
                parts = parts[::-1]
            add(f"{end}-{tag}", np.concatenate(parts), 3, 2, 101, 0.0, f"{end}-{'eq-thresh' if tag == 'eq' else 'ulp-above'}")

    # ties: ADC-quantised traces, a tie group around the quantile's index, every MAD equal
    for s in range(3):
        x = np.round(_noise_chunks(rng, 30, 100, sd=2.0) * 1.0)
        add(f"adc{s}", x, 200, 10, 100, (0.0, 0.5, 0.9)[s], "adc-ties")
    for perc in (0.5, 0.45):
        ds = [5, 2, 3, 3, 3, 3, 3, 6, 4]
        add(f"tie-at-idx-{perc}", np.concatenate([mad_chunk(d, rng) for d in ds]), 2, 2, 101, perc, "tie-at-idx")
    add("all-mads-equal", np.tile(np.float32([1, 5, 2, 8, 3]), 400), 200, 10, 100, 0.3, "all-mads-equal")

    # which chunks are kept
    lo_c = lambda: mad_chunk(1.0, rng)                   # noqa: E731
    hi_c = lambda: mad_chunk(9.0, rng)                   # noqa: E731
    add("kept-only-first", np.concatenate([hi_c(), lo_c(), lo_c(), lo_c()]), 5, 5, 101, 0.0, "kept-first-0", "one-kept")
    add("kept-only-last", np.concatenate([lo_c(), lo_c(), lo_c(), hi_c()]), 5, 5, 101, 0.0, "kept-last-end", "one-kept")
    add("kept-only-middle", np.concatenate([lo_c(), lo_c(), hi_c(), lo_c()]), 5, 5, 101, 0.0, "only-middle", "one-kept")
    add("kept-all", np.concatenate([hi_c(), lo_c(), hi_c(), hi_c()]), 5, 5, 101, 0.0, "kept-first-0", "kept-last-end")
    add("kept-none", np.concatenate([lo_c(), lo_c(), lo_c()]), 5, 5, 101, 0.0, "none-kept")

    # fixed trims on a read whose kept chunks are 1 .. 3 of 5 (samples 101 .. 404)
    fx = np.concatenate([lo_c(), hi_c(), hi_c(), hi_c(), lo_c()])
    add("fixed-empty", fx, 150, 153, 101, 0.0, "fixed-start-eq-end")
    add("fixed-one-sample", fx, 150, 152, 101, 0.0, "fixed-one-sample")
    add("fixed-none", fx, 0, 0, 101, 0.0, "fixed-zero")
    add("fixed-end-below-trim-end", np.concatenate([hi_c(), lo_c(), lo_c()]), 0, 150, 101, 0.0, "end-below-trim-end")

    # sample values
    add("negative", _noise_chunks(rng, 12, 64, lo=-130, hi=-60), 10, 10, 64, 0.0, "negative")
    mixed = _noise_chunks(rng, 12, 64, lo=-5, hi=5, sd=3.0)
    mixed[::7] = 0.0
    mixed[3::11] = -0.0
    add("mixed-sign-zeros", mixed, 10, 10, 64, 0.1, "mixed-sign-zeros")
    add("huge", _f32(_noise_chunks(rng, 12, 64, sd=30.0) * np.float32(2 ** 19)), 10, 10, 64, 0.2, "magnitude>=2^24")
    fm = np.concatenate([_f32(rng.uniform(0.5, 1.0, 64 * 6)) * FLT_MAX, -_f32(rng.uniform(0.5, 1.0, 64 * 6)) * FLT_MAX])
    fm[:64] = FLT_MAX * np.float32(0.75) + _f32(rng.normal(0, 1, 64)) * np.float32(2 ** 100)    # a quiet leading chunk
    add("near-flt-max", fm, 10, 10, 64, 0.0, "near-flt-max")
    return cases


class TrimTrace:
    def __init__(self, port, c: TrimCase):
        t = port.trim_trace(c.x, c.ts, c.te, c.chunk, c.perc)
        self.__dict__.update(t)
        self.nchunk = c.x.shape[0] // c.chunk

    def ref_ok(self, c: TrimCase) -> bool:
        """whether the reference can be asked: a chunk at least, a kept chunk, and no wrap of rt.end - trim_end"""
        return self.nchunk > 0 and self.first <= self.last and (self.last + 1) * c.chunk >= c.te


def trim_edges(c: TrimCase, t: TrimTrace) -> set:
    e = set()
    n, ns, ch = t.nchunk, c.x.shape[0], c.chunk
    e.add("chunk-odd" if ch % 2 else "chunk-even")
    e.add(f"chunk={ch}")
    if ns == 0:
        e.add("ns=0")
    if ns == ch - 1:
        e.add("ns=chunk-1")
    if ns == ch:
        e.add("ns=chunk")
    if ns % ch == 0 and ns // ch >= 2:
        e.add("ns=m*chunk")
    if (ns + 1) % ch == 0 and ns // ch >= 2:
        e.add("ns=m*chunk-1")
        e.add("ns=m*chunk+chunk-1")
    for v in (1, 2, 3, 255, 256, 257, 513):
        if n == v:
            e.add(f"nchunk={v}")
    if n > 8 and n % 8 == 7:
        e.add("nchunk=8k-1")
    if n > 8 and n % 8 == 1:
        e.add("nchunk=8k+1")
    if n >= 10_000:
        e.add("nchunk>=1e4")
    if n > 0:
        idx, remf, interp = quantile_pos(c.perc, n)
        assert interp == t.interp
        if c.perc == 0.0:
            e.add("perc=0")
        if c.perc == 1.0:
            e.add("perc=1")
        if 0.0 < c.perc < 1.0 and interp and remf == 0.0 and idx > 0:
            e.add("perc-exact-index")
        if interp and remf > np.float32(0.99):
            e.add("perc-rem-near-1")
        if c.perc == float(np.nextafter(np.float32(1), np.float32(0))) and interp and remf > np.float32(0.99):
            e.add("perc-1-ulp")
        if np.float32(c.perc) == np.float32(1.4e-45):
            e.add("perc=min-float")
        m = t.mads
        if interp:
            srt = np.sort(m)
            assert _mix(remf, srt[idx], srt[idx + 1]) == t.thresh
            td = _mix(remf, srt[idx], srt[idx + 1], double_product=True)
            if td != t.thresh and ((m[0] > t.thresh) != (m[0] > td) or (m[-1] > t.thresh) != (m[-1] > td)):
                e.add("mix-product-decides")
        if n >= 2 and m[0] == t.thresh and t.first > 0:
            e.add("lead-eq-thresh")
        if n >= 2 and m[0] == _up(t.thresh) and t.first == 0:
            e.add("lead-ulp-above")
        if n >= 2 and m[-1] == t.thresh and t.last < n - 1:
            e.add("trail-eq-thresh")
        if n >= 2 and m[-1] == _up(t.thresh) and t.last == n - 1:
            e.add("trail-ulp-above")
        if np.all(c.x == np.round(c.x)) and np.unique(m).shape[0] < n:
            e.add("adc-ties")
        s = np.sort(m)
        if 1 <= idx and idx + 1 < n and s[idx - 1] == s[idx] == s[idx + 1]:
            e.add("tie-at-idx")
        if n >= 2 and np.all(m == m[0]):
            e.add("all-mads-equal")
        if t.first <= t.last:
            if t.first == 0:
                e.add("kept-first-0")
            if t.last == n - 1:
                e.add("kept-last-end")
            if t.first == t.last:
                e.add("one-kept")
                if 0 < t.first < n - 1:
                    e.add("only-middle")
            start, end = t.first * ch + c.ts, (t.last + 1) * ch
            if end < c.te:
                e.add("end-below-trim-end")
            elif start == end - c.te:
                e.add("fixed-start-eq-end")
            elif end - c.te - start == 1:
                e.add("fixed-one-sample")
            if c.ts == 0 and c.te == 0:
                e.add("fixed-zero")
        else:
            e.add("none-kept")
    if ns:
        if np.all(c.x < 0):
            e.add("negative")
        if (c.x > 0).any() and (c.x < 0).any() and (np.signbit(c.x) & (c.x == 0)).any() and (~np.signbit(c.x) & (c.x == 0)).any():
            e.add("mixed-sign-zeros")
        if np.abs(c.x).max() >= 2.0 ** 24:
            e.add("magnitude>=2^24")
        if np.abs(c.x).max() >= FLT_MAX / 4:
            e.add("near-flt-max")
    return e


TRIM_EDGES = (["chunk-odd", "chunk-even", "ns=0", "ns=chunk-1", "ns=chunk", "ns=m*chunk-1", "ns=m*chunk", "ns=m*chunk+chunk-1"]
              + [f"nchunk={v}" for v in (1, 2, 3)] + ["nchunk=8k-1", "nchunk=8k+1"] + [f"nchunk={v}" for v in (255, 256, 257, 513)]
              + ["nchunk>=1e4", "perc=0", "perc=1", "perc-exact-index", "perc-rem-near-1", "perc-1-ulp", "perc=min-float",
                 "mix-product-decides", "lead-eq-thresh", "lead-ulp-above", "trail-eq-thresh", "trail-ulp-above", "adc-ties", "tie-at-idx", "all-mads-equal",
                 "kept-first-0", "kept-last-end", "one-kept", "only-middle", "none-kept", "fixed-start-eq-end", "fixed-one-sample",
                 "fixed-zero", "end-below-trim-end", "negative", "mixed-sign-zeros", "magnitude>=2^24", "near-flt-max"])


def check_trim_edges(port, cases=None):
    """confirm every trim case's claims on the port oracle's trace; returns ({edge: [case names]}, {case: TrimTrace})"""
    cases = trim_cases() if cases is None else cases
    cover = {k: [] for k in TRIM_EDGES}
    traces = {}
    chunks = set()
    for c in cases:
        t = traces[c.name] = TrimTrace(port, c)
        e = trim_edges(c, t)
        assert c.claims <= e, f"{c.name} misses {sorted(c.claims - e)}"
        for k in e:
            if k in cover:
                cover[k].append(c.name)
            elif k.startswith("chunk="):
                chunks.add(int(k[6:]))
    assert chunks >= set(range(2, MAX_CHUNK + 1)), f"chunk sizes without a case: {sorted(set(range(2, 129)) - chunks)}"
    return cover, traces


def trim_deviations(cases, traces) -> list:
    """cases the reference is never asked about (it asserts, reads an empty array or wraps): device against port only"""
    return [c.name for c in cases if not traces[c.name].ref_ok(c)]


# ---- calibration cases ------------------------------------------------------------------------------------------------
@dataclass
class CalCase:
    name: str
    model: synth.PoreModel
    codes: np.ndarray            # base codes of the read's sequence: n_kmers + K - 1 bases
    ev_mean: np.ndarray          # f32[n_events]
    pairs: np.ndarray            # PAIR_DT[n_pairs]
    claims: set = field(default_factory=set)
    read_shift: float = 0.0      # the read's scalings before the call (kept when it is not recalibrated)
    read_scale: float = 1.0

    @property
    def ranks(self):
        return synth.kmer_ranks_from_codes(self.codes, K, 4)

    @property
    def n_kmers(self):
        return self.codes.shape[0] - K + 1

    def read(self):
        r = np.zeros(1, synth.READ_DT)
        r[0] = (0, self.ev_mean.shape[0], 0, self.read_scale, self.read_shift, 0.0, 1.0, 0.0, 0.0)
        return r

    def job(self):
        j = np.zeros(1, synth.ABEA_JOB_DT)
        j[0] = (0, 0, 0, self.n_kmers, max(self.pairs.shape[0], 1), 0)
        return j[0]

    def seq(self) -> bytes:
        return synth._CODE2DNA[self.codes].tobytes()


def cal_fingerprint(c: CalCase) -> str:
    h = hashlib.sha1(c.codes.tobytes() + _f32(c.ev_mean).tobytes() + c.pairs.tobytes())
    h.update(np.ascontiguousarray(c.model.level_mean, np.float64).tobytes() + np.ascontiguousarray(c.model.level_stdv, np.float64).tobytes())
    h.update(repr((c.read_shift, c.read_scale)).encode())
    return h.hexdigest()


def cal_hash(shift, scale, drift, var, epb, n_used, calibrated) -> str:
    return hashlib.sha1(np.float64([shift, scale, drift, var, epb]).tobytes() + repr((int(n_used), bool(calibrated))).encode()).hexdigest()


def port_cal_hash(cal, n_pairs) -> str:
    """cal_hash of an nph_calibration record (the port's or the device's), or "no-alignment" for a job without pairs"""
    if n_pairs == 0:
        return "no-alignment"
    return cal_hash(cal["shift"], cal["scale"], cal["drift"], cal["var"], cal["events_per_base"], cal["n_used"],
                    int(cal["n_used"]) >= MIN_M)


def _model(mean, sd=1.0, name="case"):
    mean = np.asarray(mean, np.float64)
    sd = np.full(mean.shape[0], sd, np.float64) if np.isscalar(sd) else np.asarray(sd, np.float64)
    return synth.PoreModel(name, K, "nucleotide", mean, sd, np.log(sd))


def _codes(rng, n_kmers, max_run=3):
    """random bases without a homopolymer run longer than max_run, so consecutive k-mers never share a rank by chance"""
    n = n_kmers + K - 1
    c = rng.integers(0, 4, n).astype(np.uint8)
    run = 1
    for i in range(1, n):
        run = run + 1 if c[i] == c[i - 1] else 1
        if run > max_run:
            c[i] = (c[i] + 1 + rng.integers(0, 3)) % 4
            run = 1
    return c


def _layout(ranks, counts, model, rng, noise=1.0):
    """k-mer ki gets counts[ki] consecutive new events; pairs in k-mer order; each event's mean is its k-mer's level plus noise"""
    pr, means = [], []
    e = 0
    for ki, cnt in enumerate(counts):
        for _ in range(int(cnt)):
            pr.append((ki, e))
            means.append(model.level_mean[ranks[ki]] + rng.normal(0.0, noise))
            e += 1
    return np.array(pr, synth.PAIR_DT), _f32(means)


NUC = None


def _nuc():
    global NUC
    if NUC is None:
        NUC = synth.load_model("nucleotide")
    return NUC


def _random_case(name, n_kmers, seed, claims=(), zero=(), model=None, max_run=3):
    rng = np.random.default_rng(seed)
    model = model or _nuc()
    codes = _codes(rng, n_kmers, max_run)
    ranks = synth.kmer_ranks_from_codes(codes, K, 4)
    counts = rng.integers(1, 4, n_kmers)
    counts[list(zero)] = 0
    pairs, ev = _layout(ranks, counts, model, rng)
    return CalCase(name, model, codes, ev, pairs, set(claims))


def _qc_case(name, levels, n_kmers, seed, epb=None, bump=False):
    """two exactly representable levels (sigma 1), one event per k-mer, events at level +- 2.5 balanced in each level group,
    so that shift 0, scale 1 and var = 2.5 come out exactly.  epb: the last k-mer gets a second event at index
    round(epb * n_kmers) (events_per_base = that / n_kmers); bump: one event one float ulp further out (var just above 2.5)."""
    rng = np.random.default_rng(seed)
    codes = _codes(rng, n_kmers)
    ranks = synth.kmer_ranks_from_codes(codes, K, 4)
    mean = np.where(np.arange(4 ** K) % 2 == 0, levels[0], levels[1]).astype(np.float64)
    model = _model(mean)
    lv = mean[ranks]
    use = np.ones(n_kmers, bool)
    for v in levels:
        idx = np.nonzero(lv == v)[0]
        if idx.shape[0] % 2:
            use[idx[-1]] = False
    use[0] = use[-1] = True
    for v in levels:                  # the first and last k-mers must keep their events; rebalance the group without them
        idx = np.nonzero((lv == v) & use)[0]
        if idx.shape[0] % 2:
            inner = [i for i in idx if 0 < i < n_kmers - 1]
            use[inner[-1]] = False
    stride = 1 if epb is None else 5
    pr = [(ki, stride * ki) for ki in np.nonzero(use)[0]]
    n_ev = stride * (n_kmers - 1) + 1
    ev = np.full(n_ev, np.float32(np.mean(levels)), np.float32)
    sign = {}
    for ki in np.nonzero(use)[0]:
        s = sign.get(lv[ki], 1.0)
        sign[lv[ki]] = -s
        ev[stride * ki] = np.float32(lv[ki] + 2.5 * s)
    if bump:
        ki = np.nonzero(use)[0][1]
        ev[stride * ki] = np.nextafter(ev[stride * ki], np.float32(np.inf) if ev[stride * ki] > lv[ki] else np.float32(-np.inf))
    if epb is not None:
        last = int(round(epb * n_kmers))
        ev = np.concatenate([ev, np.full(last + 1 - n_ev, np.float32(np.mean(levels)), np.float32)])
        pr.append((n_kmers - 1, last))
    return CalCase(name, model, codes, ev, np.array(pr, synth.PAIR_DT), set())


def lu_solve(a00, a01, a11, b0, b1, force=None):
    """full_piv_lu_solve_2x2 in Python doubles, optionally with the pivot forced: (x0, x1, (pr, pc), rank)"""
    m = [[a00, a01], [a01, a11]]
    b = [b0, b1]
    pr = pc = 0
    big = abs(m[0][0])
    for (r, cc) in ((1, 0), (0, 1), (1, 1)):
        if abs(m[r][cc]) > big:
            big, pr, pc = abs(m[r][cc]), r, cc
    if force is not None:
        pr, pc = force
        big = abs(m[pr][pc])
    if big == 0.0:
        return 0.0, 0.0, (pr, pc), 0
    if pr == 1:
        m = [m[1], m[0]]
        b = [b[1], b[0]]
    if pc == 1:
        m = [[m[0][1], m[0][0]], [m[1][1], m[1][0]]]
    l = m[1][0] / m[0][0]
    u11 = m[1][1] - l * m[0][1]
    c1 = b[1] - l * b[0]
    maxpivot = max(big, abs(u11))
    thr = 2.220446049250313e-16 * 2.0 * maxpivot
    if abs(u11) > thr:
        y1 = c1 / u11
        y0 = (b[0] - y1 * m[0][1]) / m[0][0]
        rank = 2
    else:
        y1, y0, rank = 0.0, b[0] / m[0][0], 1
    return (y1, y0, (pr, pc), rank) if pc == 1 else (y0, y1, (pr, pc), rank)


def sums_of(mu, e, sd=None):
    """the five normal-equation sums in 'M' order, as recalibrate_model and the kernel's lane 0 add them"""
    a00 = a01 = a11 = b0 = b1 = 0.0
    for i in range(len(mu)):
        s = 1.0 if sd is None else float(sd[i])
        iv = 1.0 / (s * s)
        m, x = float(mu[i]), float(e[i])
        a00 += iv
        a01 += m * iv
        a11 += m * m * iv
        b0 += x * iv
        b1 += m * x * iv
    return a00, a01, a11, b0, b1


def _equal_level_case(name, want_rank, n_kmers=230):
    """every level equal (mu), so the system is rank 1 in exact arithmetic; search mu and the events for a rounding residual
    on the wanted side of the epsilon * 2 * maxpivot threshold"""
    for seed in range(4000):
        rng = np.random.default_rng(77_000 + seed)
        mu = float(rng.choice([rng.uniform(0.3, 0.999), rng.uniform(1.001, 3.0), rng.uniform(10.0, 200.0)]))
        codes = _codes(rng, n_kmers)
        ranks = synth.kmer_ranks_from_codes(codes, K, 4)
        model = _model(np.full(4 ** K, mu))
        pairs, ev = _layout(ranks, np.ones(n_kmers, int), model, rng, noise=0.7)
        s = sums_of(np.full(n_kmers, mu), ev.astype(np.float64))
        if lu_solve(*s)[3] == want_rank:
            return CalCase(name, model, codes, ev, pairs, {"rank1" if want_rank == 1 else "rank1-levels-rank2"})
    raise AssertionError(f"no {name} case found")


def _tie_case():
    """levels +-1 (sigma 1): A00 == A11 exactly; unbalanced signs make A01 non-zero, and the events are searched until the
    first-wins pivot (0,0) and the pivot (1,1) give different bits"""
    n_kmers = 240
    for seed in range(2000):
        rng = np.random.default_rng(91_000 + seed)
        codes = _codes(rng, n_kmers)
        ranks = synth.kmer_ranks_from_codes(codes, K, 4)
        model = _model(np.where(rng.random(4 ** K) < 0.6, 1.0, -1.0))
        pairs, ev = _layout(ranks, np.ones(n_kmers, int), model, rng, noise=0.5)
        s = sums_of(model.level_mean[ranks], ev.astype(np.float64))
        a = lu_solve(*s)
        b = lu_solve(*s, force=(1, 1))
        if s[0] == s[2] and a[2] == (0, 0) and (a[0], a[1]) != (b[0], b[1]):
            return CalCase("pivot-tie", model, codes, ev, pairs, {"pivot-tie"})
    raise AssertionError("no tie case found")


def cal_cases() -> list:
    cases = []
    for nk in (1, 31, 32, 33, 63, 64, 65):
        cases.append(_random_case(f"nk{nk}", nk, 100 + nk, {f"nk={nk}"}))
    cases.append(_random_case("nk-1e5", 100_000, 7, {"nk>=1e5"}))

    # rank carry: a homopolymer run of k-mers across the tile boundary 31/32
    rng = np.random.default_rng(5)
    c = _random_case("run-across-tile", 300, 11, {"run-across-tile"})
    c.codes[26:26 + K + 9] = 2
    c.pairs, c.ev_mean = _layout(c.ranks, rng.integers(1, 3, c.n_kmers), c.model, rng)
    cases.append(c)
    # k-mers 31 and 64 share a rank and nothing in between has events: tile 1 (32 .. 63) is empty, hm == 0 keeps the carry
    c = _random_case("carry-empty-tile", 300, 12, {"carry-across-empty-tile", "first-at-lane31", "tile-lane31-only", "tile-lane0-only"})
    c.codes[64:64 + K] = c.codes[31:31 + K]
    counts = rng.integers(1, 3, c.n_kmers)
    counts[:31] = 0
    counts[32:64] = 0
    counts[65:96] = 0
    c.pairs, c.ev_mean = _layout(c.ranks, counts, c.model, rng)
    cases.append(c)
    # a same-rank pair separated by a few k-mers without events inside one tile
    c = _random_case("carry-gap", 300, 13, {"carry-across-gap"})
    c.codes[110:110 + K] = c.codes[100:100 + K]
    counts = rng.integers(1, 3, c.n_kmers)
    counts[101:110] = 0
    c.pairs, c.ev_mean = _layout(c.ranks, counts, c.model, rng)
    cases.append(c)

    # pair lists: repeated events, one event shared by consecutive k-mers, a backwards range, a non-monotone tail
    c = _random_case("odd-pairs", 320, 14, {"repeated-events", "shared-event", "backwards-range", "non-monotone-tail"})
    p = [tuple(v) for v in c.pairs.tolist()]
    q = []
    for i, (k, e) in enumerate(p):
        q.append((k, e))
        if k == 40 and (not q[:-1] or q[-2][0] != 40):
            q.append((k, e))                                   # the same pair twice
        if k == 60 and (i + 1 == len(p) or p[i + 1][0] != 60):
            q.append((61, e))                                  # k-mer 61 starts on k-mer 60's last event
    back = [i for i, (k, _) in enumerate(q) if k == 80]
    q.insert(back[-1] + 1, (80, q[back[0]][1] - 3))            # k-mer 80's last counted event precedes its first
    q += [(315, 500), (318, 480), (316, 505), (319, 470)]        # a tail that jumps back and forth
    c.pairs = np.array(q, synth.PAIR_DT)
    cases.append(c)

    # 'M' event counts around minNumEventsToRescale: n_used of a case with every k-mer distinct is its k-mers with events
    for nu in (199, 200, 201):
        cases.append(_random_case(f"n-used-{nu}", 260, 300 + nu, {f"n_used={nu}"}, zero=range(nu, 260)))

    # QC thresholds, exact arithmetic
    for lv, tag in (((80.0, 120.0), "80-120"), ((0.25, 0.75), "quarter")):
        c = _qc_case(f"var-2.5-{tag}", lv, 240, 41)
        c.claims = {"var=2.5", "pivot11" if lv[0] > 1 else "pivot00"}
        cases.append(c)
    c = _qc_case("var-above", (80.0, 120.0), 240, 42, bump=True)
    c.claims = {"var-just-above"}
    cases.append(c)
    c = _qc_case("epb-5", (80.0, 120.0), 240, 41, epb=5.0)
    c.claims = {"epb=5", "var=2.5"}
    cases.append(c)
    c = _qc_case("epb-above", (80.0, 120.0), 240, 44, epb=5.0 + 1.0 / 240)
    c.claims = {"epb-just-above"}
    cases.append(c)
    c = _qc_case("highvar-and-stays", (80.0, 120.0), 240, 45, epb=6.0, bump=True)
    c.claims = {"highvar+stays"}
    cases.append(c)
    c = _random_case("toofew-and-stays", 150, 46)
    pr = c.pairs.copy()
    pr[-1]["read_pos"] = 7 * 150
    c.ev_mean = np.concatenate([c.ev_mean, np.full(7 * 150 + 1 - c.ev_mean.shape[0], 90.0, np.float32)])
    c.pairs = pr
    c.claims = {"toofew+stays"}
    cases.append(c)

    # LU pivots
    cases.append(_tie_case())
    cases.append(_equal_level_case("rank1", 1))
    cases.append(_equal_level_case("rank1-rounded-to-2", 2))
    rngn = np.random.default_rng(8)
    neg = _model(-rngn.uniform(60.0, 120.0, 4 ** K), rngn.uniform(1.0, 3.0, 4 ** K))
    cases.append(_random_case("negative-levels", 400, 15, {"negative-A01"}, model=neg))
    c = _random_case("not-aligned", 50, 16, {"not-aligned"})
    c.pairs = c.pairs[:0]
    cases.append(c)
    return cases


class CalTrace:
    def __init__(self, port, c: CalCase):
        self.b2e, self.cal, self.sums, self.piv, self.m_kmers = port.recalibrate_trace(
            c.read(), c.ev_mean, c.model, c.ranks, c.job(), c.pairs, c.pairs.shape[0])


def cal_edges(c: CalCase, t: CalTrace) -> set:
    e = set()
    nk = c.n_kmers
    for v in (1, 31, 32, 33, 63, 64, 65):
        if nk == v:
            e.add(f"nk={v}")
    if nk >= 100_000:
        e.add("nk>=1e5")
    ranks = c.ranks
    has = (t.b2e["start"] != -1) & (t.b2e["start"] <= t.b2e["stop"])
    m = set(int(v) for v in t.m_kmers)
    hk = np.nonzero(has)[0]
    for ki in range(TILE, nk, TILE):
        if has[ki] and has[ki - 1] and ranks[ki] == ranks[ki - 1] and ki not in m:
            e.add("run-across-tile")
    for a, b in zip(hk[:-1], hk[1:]):
        if b - a > 1 and ranks[a] == ranks[b] and b not in m:
            e.add("carry-across-gap")
            t0 = (a // TILE + 1) * TILE
            if t0 + TILE <= b:
                e.add("carry-across-empty-tile")
    for t0 in range(0, nk - TILE + 1, TILE):
        tile = np.nonzero(has[t0:t0 + TILE])[0]
        if list(tile) == [0]:
            e.add("tile-lane0-only")
        if list(tile) == [TILE - 1]:
            e.add("tile-lane31-only")
    if hk.shape[0] and hk[0] == TILE - 1:
        e.add("first-at-lane31")
    rp = c.pairs["read_pos"].astype(np.int64)
    kp = c.pairs["ref_pos"].astype(np.int64)
    if rp.shape[0] > 1:
        same = rp[1:] == rp[:-1]
        if (same & (kp[1:] == kp[:-1])).any():
            e.add("repeated-events")
        if (same & (kp[1:] == kp[:-1] + 1)).any():
            e.add("shared-event")
        if (rp[1:] < rp[:-1]).any() and (kp[1:] < kp[:-1]).any():
            e.add("non-monotone-tail")
    if ((t.b2e["start"] != -1) & (t.b2e["start"] > t.b2e["stop"])).any():
        e.add("backwards-range")
    cal = t.cal
    nu, st = int(cal["n_used"]), int(cal["status"])
    for v in (199, 200, 201):
        if nu == v:
            e.add(f"n_used={v}")
    if st == 0 and cal["var"] == MAX_VAR:
        e.add("var=2.5")
    if st == 4 and MAX_VAR < cal["var"] < MAX_VAR + 1e-6:
        e.add("var-just-above")
    if st == 0 and cal["events_per_base"] == MAX_EPB:
        e.add("epb=5")
    if st == 8 and MAX_EPB < cal["events_per_base"] < MAX_EPB + 0.01:
        e.add("epb-just-above")
    if st == 4 and cal["events_per_base"] > MAX_EPB:
        e.add("highvar+stays")
    if st == 2 and cal["events_per_base"] > MAX_EPB:
        e.add("toofew+stays")
    if st == 1 and c.pairs.shape[0] == 0:
        e.add("not-aligned")
    if t.piv[2] >= 1:
        a00, a01, a11 = t.sums[:3]
        mus = c.model.level_mean[ranks[sorted(m)]]
        if tuple(t.piv[:2]) == (0, 0) and a11 < a00:
            e.add("pivot00")
        if tuple(t.piv[:2]) == (1, 1) and a11 > a00:
            e.add("pivot11")
        if a00 == a11 and tuple(t.piv[:2]) == (0, 0):
            x = lu_solve(*t.sums)
            y = lu_solve(*t.sums, force=(1, 1))
            assert (x[0], x[1]) == (cal["shift"], cal["scale"])
            if (x[0], x[1]) != (y[0], y[1]):
                e.add("pivot-tie")
        if np.all(mus == mus[0]):
            e.add("rank1" if t.piv[2] == 1 else "rank1-levels-rank2")
        if a01 < 0:
            e.add("negative-A01")
    return e


CAL_EDGES = ([f"nk={v}" for v in (1, 31, 32, 33, 63, 64, 65)] + ["nk>=1e5", "run-across-tile", "carry-across-empty-tile",
             "carry-across-gap", "tile-lane0-only", "tile-lane31-only", "first-at-lane31", "repeated-events", "shared-event",
             "backwards-range", "non-monotone-tail", "n_used=199", "n_used=200", "n_used=201", "var=2.5", "var-just-above", "epb=5",
             "epb-just-above", "highvar+stays", "toofew+stays", "pivot00", "pivot11", "pivot-tie", "rank1", "rank1-levels-rank2",
             "negative-A01", "not-aligned"])


def check_cal_edges(port, cases=None):
    cases = cal_cases() if cases is None else cases
    cover = {k: [] for k in CAL_EDGES}
    traces = {}
    for c in cases:
        t = traces[c.name] = CalTrace(port, c)
        e = cal_edges(c, t)
        assert c.claims <= e, f"{c.name} misses {sorted(c.claims - e)}"
        for k in e:
            cover.setdefault(k, []).append(c.name)
    return cover, traces


def coverage_table(cover: dict, title: str) -> str:
    rows = [f"{title}: edge".ljust(34) + "cases"]
    for k, v in cover.items():
        rows.append(k.ljust(34) + (f"{len(v):4d}  {', '.join(v[:3])}{' ...' if len(v) > 3 else ''}" if v else "MISSING"))
    return "\n".join(rows)


# ---- load_from_raw cases ----------------------------------------------------------------------------------------------
def step_read(rng, n_steps, spacing=20, last_jump=-20.0):
    """noise-free levels: a flat leading chunk (MAD 0, trimmed), a chunk with one level change at its middle (the first MAD
    above 0; the fixed 200-sample trim starts inside the next chunks), n_steps level changes spaced `spacing` apart from
    sample 300 on, and a last chunk with one change at its middle (the last MAD above 0)"""
    lv = lambda i: 100.0 + 7.0 * (i % 5) + rng.integers(0, 3)      # noqa: E731
    x = [np.full(100, 100.0), np.full(50, 100.0), np.full(150, 130.0)]
    for i in range(n_steps):
        x.append(np.full(spacing, lv(i)))
    n = sum(v.shape[0] for v in x)
    x.append(np.full((n + 99) // 100 * 100 - n + 50, x[-1][0] if n_steps else 130.0))
    x.append(np.full(50, x[-1][0] + last_jump))
    return _f32(np.concatenate(x))


def live_event_count(port, x, prm):
    ok, s, e = port.trim_raw(x, *LFR_TRIM)
    return port.detect_events(np.ascontiguousarray(x[s:e]), prm).shape[0] if ok else 0


def read_with_events(port, target: int, prm, seed: int):
    """a step read whose trimmed range has exactly `target` events under prm (searched over the step count and the noise)"""
    for s in range(max(0, target - 4), target + 4):
        for jump in (-20.0, 1e-3):
            x = step_read(np.random.default_rng(seed * 1000 + s), s, last_jump=jump)
            if live_event_count(port, x, prm) == target:
                return x
    raise AssertionError(f"no read with {target} events")
