"""Adaptive banded event alignment (ABEA) jobs built to reach named edges of the device aligner, `abea_kernel` in
nanopolish_b200/csrc/abea.cu, and of the method-of-moments kernel that prepares its input.

The kernel's geometry (checked against abea.cu's literals by test_abea_edges_oracle.py):
  * the band is BAND = 100 columns wide; column c = k + 1, c = 0 being the trim column (k-mer -1);
  * the band's columns live in a circular window of WINDOW = 128 columns, 4 register slots x 32 lanes; the last column K
    sits at lane K & 31, slot (K >> 5) & 3;
  * the backtrack reads the band trace in blocks of TRACE_BLOCK = 64 bands, blk_lo = max(0, bi - 63), reloading when the
    path's band bi = event + k-mer + 2 drops below blk_lo;
  * QC flags a job whose max_gap > 50 or whose mean emission < -5.

Every builder returns Jobs tagged with the edges they claim, and `check_edges` confirms each claim on the port oracle's
result and band history (npo_abea_bands: each band's lower-left k-mer); a builder that misses its edge fails.  Edge names:
  K<band           K < 100: the band is wider than the matrix
  E<50             fewer events than half the band
  E=1, E=2, E=3    one to three events
  past-last-event  a band whose lowest cell lies past the last event and whose other end lies outside the matrix: Suzuki's
                   rule sees both ends at -inf and moves by band parity
  E>>K             K = 1..3 against hundreds of events, a long stall on k-mer 0
  lead-trim        the first pair's event > 0 (leading events trimmed);  lead-trim-50: >= 50
  tail-trim        the last pair's event < E - 1
  end-e0           the best end cell is at event 0;  end-last: at event E - 1
  no-end-cell      the last k-mer's column is never inside the band (NPH_ABEA_NO_END_CELL).  No read with levels the device
                   takes reached it: with E << K (K up to 1000, E down to 1) the trim column keeps the band moving right, and
                   check_edges asserts that no such job carries it.  Only a NaN level, which the device refuses, reaches it on
                   the oracle, so the device's NO_END_CELL record is never compared with the oracle's.
  end-bi<63, end-bi=63, end-bi=64, end-bi=65    the end cell's band
  diag-cross-block a diagonal step from the first band of a trace block to two bands below it, skipping the block's edge
  bi=2             the path reaches band 2 (k-mer 0, event 0)
  gap=50, gap=51   the path's max_gap is exactly 50 (passes QC) / 51 (fails)
  low-emission, max-gap, low-emission+max-gap    the QC verdicts alone and together
  cap=n-1 ... cap=n+1000, cap=1    pairs_cap relative to the path length n; n - 1 and 1 overflow
  level-inf, level-nan, level-flt-max, level-2^64, level-1e30, level-max, level-above-max    one level outside the pA range
                   mid-read and one in the first 20 events, each credited on the oracle (see level_edge): the 2^64 window on
                   the path with a finite emission below -1e38; max (2048, the largest level the device takes) and the next
                   float above it with a finite emission against every k-mer; inf, -inf, NaN, FLT_MAX and 1e30 emitted as -inf (NaN)
                   by every k-mer

NOT_SPANNED is not reachable: every finite cell traces back to k-mer 0 or the trim column, so a path that passes
end-cell and capacity checks always ends at k-mer 0; check_edges asserts that no job carries it.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200 import synth

BAND = 100
WINDOW = 128
TRACE_BLOCK = 64
MAX_GAP = 50
MIN_AVG = -5.0
MAX_LEVEL = 2048.0            # NPH_ABEA_MAX_LEVEL, include/nph.h: the largest |level| the device aligner takes
K_MER = 6
ABEA_OK, LOW_EMISSION, NOT_SPANNED, MAX_GAP_BIT, NO_END_CELL, PAIRS_OVERFLOW = 0, 1, 2, 4, 8, 16

FAMILIES = ("lane-slot", "band", "E-edges", "trim", "backtrack", "qc", "capacity", "levels")


@dataclass
class Job:
    codes: np.ndarray                     # bases of the sequence (A, C, G, T = 0..3)
    nev: np.ndarray                       # events emitted from each k-mer (0: the k-mer is skipped)
    family: str
    edges: set = field(default_factory=set)
    lead: int = 0                         # noise events no k-mer fits, before the k-mers' events
    tail: int = 0                         # ... and after them
    exact: np.ndarray | None = None       # bool per k-mer: its events sit exactly on the model level
    noise: bool = False                   # every event is unrelated to the sequence
    levels: tuple = ()                    # (event index, level name[, k-mer]): "2^64" puts |x - mu'| / sigma' of that k-mer (default:
                                          # the one that emitted the event) in [2^64, 2^64.5)
    cap: tuple = ("full",)                # ("full",): n_events + n_kmers; ("n", d): path length + d; ("abs", c)
    read_of: int | None = None            # share the read of an earlier job (-1: the job before)
    seed: int = 0

    @property
    def K(self) -> int:
        return int(self.codes.shape[0]) - K_MER + 1

    @property
    def E(self) -> int:
        return self.lead + int(self.nev.sum()) + self.tail


def spread(rng, K: int, E: int) -> np.ndarray:
    """E events over K k-mers, about 1.8 per k-mer, the first and the last with at least one where E >= 2"""
    nev = np.zeros(K, np.int64)
    if K == 1 or E < 2:
        nev[0] = E
        return nev
    nev[0] += 1; nev[-1] += 1
    np.add.at(nev, rng.integers(0, K, E - 2), 1)
    return nev


def plain(rng, K, E, family, edges=(), **kw) -> Job:
    codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
    return Job(codes, spread(rng, K, E), family, set(edges), seed=int(rng.integers(1 << 30)), **kw)


# ---------------------------------------------------------------- families
def lane_slot_jobs(seed: int = 1):
    """K mod 128 takes every value (E ~ 1.8 K), plus the window's and band's named K and a few K >= 1000"""
    rng = np.random.default_rng(seed)
    Ks = [128 + r for r in range(128)]
    Ks += [1, 2, 3, 31, 32, 33, 49, 50, 51, 99, 100, 101, 127, 129, 255, 256, 257, 1000, 1151, 1407]
    return [plain(rng, K, max(1, int(1.8 * K)), "lane-slot", {"K<band"} if K < BAND else set()) for K in Ks]


def event_edge_jobs(seed: int = 2):
    """E = 1, 2, 3 and E < 50 against several K; E << K where the band walks past the last event; E >> K"""
    rng = np.random.default_rng(seed)
    out = []
    for K in (1, 2, 3, 20, 60, 120):
        for E in (1, 2, 3, 30, 49):
            edges = {"E<50"} | ({f"E={E}"} if E <= 3 else set()) | ({"K<band"} if K < BAND else set())
            out.append(plain(rng, K, E, "E-edges", edges))
    for K, E in ((150, 8), (200, 20), (260, 40), (400, 60), (300, 5)):
        out.append(plain(rng, K, E, "band", {"past-last-event"}))
    for K, E in ((1, 300), (2, 400), (3, 250)):
        j = plain(rng, K, E, "E-edges", {"E>>K"})
        out.append(j)
    # a long stall on k-mer 0's level: 300 events exactly on it, then the rest of a short sequence
    codes = rng.integers(0, 4, 3 + K_MER - 1).astype(np.uint8)
    nev = np.array([300, 2, 2], np.int64)
    exact = np.array([True, False, False])
    out.append(Job(codes, nev, "E-edges", {"E>>K"}, exact=exact))
    return out


def trim_jobs(seed: int = 3):
    """leading and trailing noise events the path trims; the best end cell at event 0 and at the last event"""
    rng = np.random.default_rng(seed)
    out = []
    for lead in (5, 20, 50, 60):
        out.append(plain(rng, 150, 270, "trim", {"lead-trim"} | ({"lead-trim-50"} if lead >= 50 else set()), lead=lead))
    for tail in (3, 30):
        out.append(plain(rng, 150, 270, "trim", {"tail-trim"}, tail=tail))
    out.append(plain(rng, 1, 1, "trim", {"end-e0", "end-last"}))
    out.append(plain(rng, 1, 1, "trim", {"end-e0", "tail-trim"}, tail=5))
    out.append(plain(rng, 80, 150, "trim", {"end-last"}))
    return out


# (K, E, seed) whose path starts at (k-mer 0, event 0), ends at the last event and passes QC (found by search)
END_BANDS = {"end-bi=63": (10, 53, 0), "end-bi=64": (10, 54, 0), "end-bi=65": (10, 55, 0)}


def backtrack_jobs(seed: int = 4):
    """end cells in bands < 63, 63, 64, 65 (band = end event + K + 1); long reads for block crossings"""
    rng = np.random.default_rng(seed)
    out = [plain(rng, 20, 30, "backtrack", {"end-bi<63", "bi=2"})]
    for edge, (K, E, s) in END_BANDS.items():
        out.append(plain(np.random.default_rng(s * 1000 + K), K, E, "backtrack", {edge, "bi=2"}))
    for K in (300, 700):
        out.append(plain(rng, K, int(1.8 * K), "backtrack", {"diag-cross-block", "bi=2"}))
    return out


# Deleting the events of a run of k-mers rarely yields that gap: mismatching the neighbours' events costs less than skipping.
# So the run is a homopolymer of G (GGGGGG, the lowest level of the model) whose events are deleted: (run length, seed)
# found by search for max_gap exactly 50 passing QC, 51 failing on the gap alone, and 51 failing on both gap and emission.
GAP_RUNS = {"gap=50": (52, 6), "gap=51": (56, 4), "low-emission+max-gap": (53, 2)}


def gap_job(L: int, s: int, edges) -> Job:
    rng = np.random.default_rng(5000 + s)
    K, a = 200, 80
    codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
    codes[a:a + L + K_MER - 1] = 2
    nev = spread(rng, K, int(1.8 * K))
    nev[a:a + L] = 0
    return Job(codes, nev, "qc", set(edges), seed=5000 + s)


def qc_jobs(seed: int = 5):
    rng = np.random.default_rng(seed)
    out = [gap_job(*GAP_RUNS["gap=50"], {"gap=50"}), gap_job(*GAP_RUNS["gap=51"], {"gap=51", "max-gap"}),
           gap_job(*GAP_RUNS["low-emission+max-gap"], {"gap=51", "low-emission+max-gap"})]
    out.append(plain(rng, 200, 360, "qc", {"low-emission"}, noise=True))
    out.append(plain(rng, 120, 2, "qc", {"low-emission+max-gap"}))
    return out


CAPS = (("n", -1), ("n", 0), ("n", 1), ("n", 31), ("n", 32), ("n", 33), ("n", 1000), ("abs", 1))


def capacity_jobs(seed: int = 6):
    """pairs_cap at and around the path length, and a job pair that shares one read"""
    rng = np.random.default_rng(seed)
    out = []
    for i, cap in enumerate(CAPS):
        K = (40, 150, 333)[i % 3]
        name = "cap=1" if cap[0] == "abs" else f"cap=n{cap[1]:+d}".replace("+0", "")
        out.append(plain(rng, K, int(1.8 * K), "capacity", {name}, cap=cap))
    # two jobs on one read: the whole sequence, and its first half
    j = plain(rng, 120, 216, "capacity", {"shared-read"})
    out.append(j)
    half = Job(j.codes[:60 + K_MER - 1].copy(), j.nev[:60].copy(), "capacity", {"shared-read"}, read_of=-1)
    out.append(half)
    return out


LEVELS = ("inf", "-inf", "nan", "flt-max", "2^64", "1e30", "max", "above-max")


# (K, E, seed, event, k-mer) of reads whose oracle path pairs `event` with `k-mer` after the event's level is set to put
# |x - mu'| / sigma' of that k-mer in [2^64, 2^64.5) (found by search): the reference's emission there is finite, below -1e38
WINDOW_JOBS = {"head": (2, 13, 43, 6, 0), "mid": (40, 72, 32, 36, 0)}


def level_jobs(seed: int = 7):
    """one out-of-range level mid-read and one in the first 20 events"""
    rng = np.random.default_rng(seed)
    out = []
    for i, lv in enumerate(LEVELS):
        for where in ("mid", "head"):
            if lv == "2^64":
                K, E, s, e, km = WINDOW_JOBS[where]
                j = plain(np.random.default_rng(s), K, E, "levels", {"level-2^64"})
                j.levels = ((e, lv, km),)
            else:
                j = plain(rng, 120, 216, "levels", {f"level-{lv.lstrip('-')}"})
                j.levels = ((108 if where == "mid" else 7 + i, lv),)
            out.append(j)
    return out


def all_jobs():
    return (lane_slot_jobs() + event_edge_jobs() + trim_jobs() + backtrack_jobs() + qc_jobs() + capacity_jobs() + level_jobs())


# ---------------------------------------------------------------- a batch as the C ABI takes it
@dataclass
class Batch:
    reads: np.ndarray            # READ_DT
    ev_mean: np.ndarray
    ev_start_time: np.ndarray
    jobs: np.ndarray             # ABEA_JOB_DT
    kmer_ranks: np.ndarray
    pairs_total: int
    seqs: list                   # per job: the sequence as the reference takes it
    spec: list


def window_level(model, rank: int) -> np.float32:
    """a level x with |x - mu'| / sigma' in [2^64, 2^64.5) for k-mer `rank` (scale 1, shift 0, var 1)"""
    mu, sd = np.float32(model.level_mean[rank]), np.float32(model.level_stdv[rank])
    return np.float32(np.float64(mu) + np.float64(sd) * 2.0 ** 64.25)


def _level(model, name, rank):
    return {"inf": np.float32(np.inf), "-inf": np.float32(-np.inf), "nan": np.float32(np.nan),
            "flt-max": np.float32(np.finfo(np.float32).max), "1e30": np.float32(1e30), "max": np.float32(MAX_LEVEL),
            "above-max": np.nextafter(np.float32(MAX_LEVEL), np.float32(np.inf))}.get(name) if name != "2^64" \
        else window_level(model, rank)


def make_batch(jobs, model, gap: int = 0, port=None) -> Batch:
    """one read per job (unless read_of), slots in job order with `gap` unused pairs between them.  Jobs with an ("n", d)
    capacity need the port oracle to learn their path length."""
    k = model.k
    n_reads = sum(j.read_of is None for j in jobs)
    reads = np.zeros(n_reads, synth.READ_DT)
    rows, ranks_l, seqs, means, times = [], [], [], [], []
    read_idx = {}
    off = 0
    r = 0
    for i, jb in enumerate(jobs):
        fr = synth.kmer_ranks_from_codes(jb.codes, k, 4)
        seqs.append(synth._CODE2DNA[jb.codes].tobytes())
        ranks_l.append(fr)
        if jb.read_of is not None:
            rows.append((read_idx[i + jb.read_of], jb.K))
            read_idx[i] = read_idx[i + jb.read_of]
            continue
        rng = np.random.default_rng(jb.seed)
        which = np.repeat(np.arange(jb.K), jb.nev)
        mu = model.level_mean[fr[which]]
        sd = model.level_stdv[fr[which]]
        z = rng.standard_normal(which.shape[0])
        if jb.exact is not None:
            z[jb.exact[which]] = 0.0
        body = mu + sd * z
        if jb.noise:
            body = rng.uniform(60.0, 130.0, which.shape[0])
        m = np.concatenate([rng.uniform(170.0, 200.0, jb.lead), body, rng.uniform(170.0, 200.0, jb.tail)]).astype(np.float32)
        for e, name, *km in jb.levels:
            m[e] = _level(model, name, int(fr[km[0] if km else which[e - jb.lead]]))
        E = m.shape[0]
        t = np.arange(E, dtype=np.float64) * 0.002 + rng.uniform(0.0, 100.0)
        reads[r] = (off, E, 0, 1.0, 0.0, 0.0, 1.0, 0.0, E / float(jb.K))
        means.append(m); times.append(t)
        read_idx[i] = r
        rows.append((r, jb.K))
        off += E
        r += 1
    jobs_arr = np.zeros(len(jobs), synth.ABEA_JOB_DT)
    roff = 0
    for i, (rd, K) in enumerate(rows):
        jobs_arr[i] = (roff, 0, rd, K, int(reads[rd]["n_events"]) + K, 0)
        roff += K
    kr = np.concatenate(ranks_l).astype(np.uint32)
    ev_mean, ev_t = np.concatenate(means), np.concatenate(times)
    for i, jb in enumerate(jobs):
        if jb.cap[0] == "n":
            assert port is not None, "a path-relative capacity needs the port oracle"
            _, res, _ = port.abea_bands(reads, ev_mean, ev_t, model, kr, jobs_arr[i])
            jobs_arr[i]["pairs_cap"] = max(1, int(res["n_aligned"]) + jb.cap[1])
        elif jb.cap[0] == "abs":
            jobs_arr[i]["pairs_cap"] = jb.cap[1]
    poff = 0
    for i in range(len(jobs)):
        jobs_arr[i]["pairs_off"] = poff
        poff += int(jobs_arr[i]["pairs_cap"]) + gap
    return Batch(reads, ev_mean, ev_t, jobs_arr, kr, poff, seqs, list(jobs))


def batch(model, port, gap: int = 0, levels: bool = True) -> Batch:
    return make_batch([j for j in all_jobs() if levels or j.family != "levels"], model, gap=gap, port=port)


def fingerprint(b: Batch, j: int) -> str:
    """the inputs of job j, under which the reference's answer is recorded"""
    jr = b.jobs[j]
    r = b.reads[int(jr["read"])]
    o, n = int(r["event_off"]), int(r["n_events"])
    h = hashlib.sha1()
    for part in (b.seqs[j], r.tobytes(), b.ev_mean[o:o + n].tobytes(), b.ev_start_time[o:o + n].tobytes()):
        h.update(part)
    return h.hexdigest()


def pairs_hash(ref_pos, read_pos) -> str:
    return hashlib.sha1(np.ascontiguousarray(ref_pos, np.int32).tobytes() + np.ascontiguousarray(read_pos, np.int32).tobytes()).hexdigest()


# ---------------------------------------------------------------- edges seen on the oracle
def oracle_run(port, b: Batch, model, full_cap: bool = False):
    """per job (pairs [n_pairs], result record, ll_k band history, walked path); full_cap runs every job with room n_events +
    n_kmers.  The walked path is the whole path in ascending order, also for a job that fails QC (empty on overflow or without
    an end cell)."""
    out = []
    for j in range(b.jobs.shape[0]):
        jr = b.jobs[j].copy()
        if full_cap:
            jr["pairs_cap"] = int(b.reads[int(jr["read"])]["n_events"]) + int(jr["n_kmers"])
        pairs, res, ll_k = port.abea_bands(b.reads, b.ev_mean, b.ev_start_time, model, b.kmer_ranks, jr)
        walked = 0 if int(res["status"]) & (NO_END_CELL | PAIRS_OVERFLOW) else int(res["n_aligned"])
        out.append((pairs[:int(res["n_pairs"])].copy(), res, ll_k, pairs[:walked].copy()))
    return out


def reference_emission(port, model, x, rank) -> float:
    """the reference's Gaussian log-density of level x under k-mer `rank` (scale 1, shift 0, var 1)"""
    f = port.lib.npo_log_normal_pdf
    return float(f(np.float32(x), np.float32(model.level_mean[rank]), np.float32(model.level_stdv[rank]),
                   np.float32(model.level_log_stdv[rank])))


def in_domain(levels) -> bool:
    """the levels the device aligner takes (include/nph.h): finite, |level| <= MAX_LEVEL"""
    return bool(np.all(np.abs(levels) <= MAX_LEVEL))


def level_edge(name: str, pair_on_path: bool, em: float, event_on_path: bool, em_all: np.ndarray) -> bool:
    """the out-of-range level reached the result as claimed, on the oracle: for 2^64 the path holds the windowed (k-mer, event)
    pair and the reference's emission there is finite and below -1e38; for max and above-max the reference's emission is
    finite against every k-mer of the job; for the others the reference's emission of the event is -inf (NaN for nan) against every k-mer of the
    job, so the path either leaves the event out (trimmed, or the path ends before it) or scores -inf (NaN) with it"""
    if name == "2^64":
        return pair_on_path and bool(np.isfinite(em) and em < -1e38)
    if name in ("max", "above-max"):
        return bool(np.isfinite(em_all).all())
    every = np.isnan(em_all).all() if name == "nan" else (em_all == -np.inf).all()
    return bool(every)


def block_crossings(pairs) -> bool:
    """walk the path backwards as the backtrack does; True if a diagonal step skips the band just below a block"""
    blk_lo = 1 << 30
    prev = None
    for i in range(pairs.shape[0] - 1, -1, -1):
        k, e = int(pairs["ref_pos"][i]), int(pairs["read_pos"][i])
        bi = e + k + 2
        if bi < blk_lo:
            if prev is not None and prev[0] - 1 == k and prev[1] - 1 == e and bi == blk_lo - 2:
                return True
            blk_lo = max(0, bi - (TRACE_BLOCK - 1))
        prev = (k, e)
    return False


def path_edges(spec: Job, jr, E: int, pairs, res, ll_k) -> set:
    got = set()
    K = int(jr["n_kmers"])
    st = int(res["status"])
    if K < BAND:
        got.add("K<band")
    if E < BAND // 2:
        got.add("E<50")
    if E <= 3:
        got.add(f"E={E}")
    if K <= 3 and pairs.shape[0] and np.bincount(pairs["ref_pos"]).max() >= TRACE_BLOCK:
        got.add("E>>K")                                        # observed: one k-mer holds more of the path's events than a trace block
    n_bands = E + K + 2
    for bi in range(2, n_bands):
        lk = int(ll_k[bi - 1])
        le = (bi - 1) - 2 - lk
        ll_out = le >= E or lk >= K
        ur_e, ur_k = le - (BAND - 1), lk + (BAND - 1)
        ur_out = ur_e < 0 or ur_k >= K or (ur_k == -1 and ur_e >= E)
        if le >= E and ll_out and ur_out and lk >= 0:
            got.add("past-last-event")
            break
    if st & NO_END_CELL:
        got.add("no-end-cell")
    low, gap = st & LOW_EMISSION, st & MAX_GAP_BIT
    if low and gap:
        got.add("low-emission+max-gap")
    elif low:
        got.add("low-emission")
    elif gap:
        got.add("max-gap")
    if not (st & (NO_END_CELL | PAIRS_OVERFLOW)):
        if int(res["max_gap"]) in (50, 51):
            got.add(f"gap={int(res['max_gap'])}")
    if pairs.shape[0]:
        e0, e1 = int(pairs["read_pos"][0]), int(pairs["read_pos"][-1])
        if e0 > 0:
            got.add("lead-trim")
        if e0 >= 50:
            got.add("lead-trim-50")
        if e1 < E - 1:
            got.add("tail-trim")
        if e1 == 0:
            got.add("end-e0")
        if e1 == E - 1:
            got.add("end-last")
        bi_end = e1 + K + 1
        got.add("end-bi<63" if bi_end < 63 else f"end-bi={bi_end}" if bi_end <= 65 else "end-bi>65")
        if int(pairs["ref_pos"][0]) == 0 and e0 == 0:
            got.add("bi=2")
        if block_crossings(pairs):
            got.add("diag-cross-block")
    return got


def check_edges(b: Batch, runs, full_runs, port, model) -> dict:
    """assert every job reached the edges it claims; returns {family: set of edges reached}.  runs: oracle_run at the jobs'
    own capacity; full_runs: at full capacity (the path the capacity edges are measured against).  Also asserts that no job
    whose levels the device takes ends without an end cell, and that none is NOT_SPANNED."""
    cover = {f: set() for f in FAMILIES}
    for j, spec in enumerate(b.spec):
        jr = b.jobs[j]
        E = int(b.reads[int(jr["read"])]["n_events"])
        pairs, res, ll_k, _ = runs[j]
        fpairs, fres, _, walked = full_runs[j]
        st = int(res["status"])
        assert not (st & NOT_SPANNED), f"job {j}: NOT_SPANNED without overflow or a missing end cell"
        o = int(b.reads[int(jr["read"])]["event_off"])
        if in_domain(b.ev_mean[o:o + E]):
            assert not (st & NO_END_CELL), f"job {j}: NO_END_CELL on levels the device takes"
        got = path_edges(spec, jr, E, fpairs, fres, ll_k)
        n, cap = int(fres["n_aligned"]), int(jr["pairs_cap"])
        for c in CAPS:
            name = "cap=1" if c[0] == "abs" else f"cap=n{c[1]:+d}".replace("+0", "")
            if (c[0] == "abs" and cap == c[1] and n > 1) or (c[0] == "n" and cap == n + c[1] and n > 1):
                got.add(name)
        if cap < n:
            assert st == PAIRS_OVERFLOW and int(res["n_pairs"]) == 0, f"job {j}: cap {cap} < path {n}, status {st}"
        if int((b.jobs["read"] == jr["read"]).sum()) > 1:
            got.add("shared-read")
        ranks = b.kmer_ranks[int(jr["rank_off"]):int(jr["rank_off"]) + int(jr["n_kmers"])]
        for e, name, *km in spec.levels:
            at = walked["ref_pos"][walked["read_pos"] == e]
            k = km[0] if km else (int(at[0]) if at.shape[0] else 0)
            em = reference_emission(port, model, b.ev_mean[o + e], int(ranks[k]))
            em_all = np.array([reference_emission(port, model, b.ev_mean[o + e], int(r)) for r in ranks])
            if level_edge(name.lstrip("-"), bool((at == k).any()), em, at.shape[0] > 0, em_all):
                got.add(f"level-{name.lstrip('-')}")
        missing = spec.edges - got
        assert not missing, f"job {j} ({spec.family}, K={int(jr['n_kmers'])}, E={E}): claims {sorted(missing)} not reached"
        cover[spec.family] |= got & (spec.edges | {"no-end-cell", "past-last-event", "diag-cross-block", "bi=2", "lead-trim", "tail-trim",
                                                    "end-e0", "end-last", "end-bi<63", "end-bi=63", "end-bi=64", "end-bi=65"})
    return cover


def coverage_table(cover: dict, kmods: set) -> str:
    lines = [f"K mod 128 values reached: {len(kmods)} of 128"]
    for f in FAMILIES:
        lines.append(f"{f:>10}: " + ", ".join(sorted(cover[f])))
    return "\n".join(lines)


# ---------------------------------------------------------------- method of moments
MOM_SIZES = (1, 31, 32, 33, 63, 64, 65)


def mom_batch(model, seed: int = 9) -> Batch:
    """every (E, K) with E and K in MOM_SIZES, and one large read: the MoM kernel's 32-wide staging at and around its edges"""
    rng = np.random.default_rng(seed)
    jobs = [plain(rng, K, E, "mom") for E in MOM_SIZES for K in MOM_SIZES]
    jobs.append(plain(rng, 12000, 21000, "mom"))
    return make_batch(jobs, model)


def scheduling_jobs(n: int, seed: int = 10):
    """n jobs mixing long and tiny reads, and runs of jobs with equal band counts E + K + 2"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = i % 4
        if kind == 0:
            K = int(rng.integers(600, 1200)); E = int(1.8 * K)
        elif kind == 1:
            K = int(rng.integers(1, 40)); E = int(rng.integers(1, 80))
        else:                                   # equal band counts: E + K = 540
            K = int(rng.integers(150, 250)); E = 540 - K
        out.append(plain(rng, K, E, "scheduling"))
    return out
