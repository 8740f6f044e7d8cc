"""Viterbi (profile_hmm_align) jobs built to reach named edges of the device aligner, csrc/hmm_viterbi.cu and
csrc/hmm_viterbi_kernel.cuh, with a restatement of the host's choices that decide which edges a job reaches.

Restated from csrc/hmm_viterbi.cu (not imported from the library, so a change there shows up as a failing test):
  * the class: C columns per lane, C in (1, 2, 3, 4, 6, 8), the cheapest steps(K, E, C) * (120 + 70 C), first C on ties;
  * the per-warp movement trace, (steps + 1) * 32C uint16 rounded up to 64 entries, sized by the batch's largest job;
  * the resident-CTA cap that keeps 16 warps' traces within 16 GiB per CTA count, and the refusal of a batch whose trace
    does not fit even one CTA.

Every builder returns jobs tagged with the edges they claim, and `check_edges` confirms each claim on the port oracle's path
(a builder that misses its edge fails; it does not skip).  Edge names:
  strip-1, strip, strip+1   K = n * 32C - 1, n * 32C, n * 32C + 1 (n = 1, 2, 3) in class C
  one-col-lane              the last lane of the last strip owns exactly one column
  short-period              several strips with E < 40: the period pads to 40 and the trace has dead rows
  skip-run                  >= 33 consecutive K (silent skip) states: the backtrack re-stages along the k-mer axis only
  stall                     >= 33 consecutive states on one k-mer: the backtrack re-stages along the row axis only
  homopolymer               the path moves between adjacent k-mers of one rank (events exactly at the model level)
  strip-cross               the path crosses a strip boundary between two states read from one staged 32 x 32 corner
  asserts                   the reference asserts (one event, or the path's last cell is -inf): zero states
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200 import synth

COLS = (1, 2, 3, 4, 6, 8)
MIN_PERIOD = 40               # NPH_MIN_PERIOD, csrc/hmm_classes.h
WARPS = 16                    # warps per CTA
TRACE_BUDGET = 16 << 30       # bytes of movement trace over all resident CTAs
TILE = 32                     # the backtrack's staged corner is TILE x TILE
K_MER = 6
PAD = 3                       # events of the read before and after each job's window

EDGES = ("strip-1", "strip", "strip+1", "one-col-lane", "short-period", "skip-run", "stall", "homopolymer", "strip-cross")
# edges a class can have.  Class 1 only ever holds K <= 32: one strip, no 33-k-mer skip.  K = n * 32C + 1 (n <= 3) is never
# chosen for classes 2 and 3.  Class 2 holds K > 64 only with E near 40, too few events to pin a 33-k-mer skip.
CLASS_EDGES = {1: set(EDGES) - {"one-col-lane", "short-period", "skip-run", "strip-cross", "strip+1"},
               2: set(EDGES) - {"strip+1", "skip-run"}, 3: set(EDGES) - {"strip+1"},
               4: set(EDGES), 6: set(EDGES), 8: set(EDGES)}


# ---------------------------------------------------------------- restatement of the host's choices
def class_steps(K: int, E: int, C: int) -> int:
    strip = 32 * C
    ns = (K + strip - 1) // strip
    P = max(E, MIN_PERIOD) if ns > 1 else E
    return (ns - 1) * P + E + (K - (ns - 1) * strip - 1) // C


def choose_class(K: int, E: int) -> tuple[int, int]:
    """(C, steps): the cheapest class, the first (fewest columns) on ties"""
    best, bc, bs = None, 0, 0
    for C in COLS:
        st = class_steps(K, E, C)
        cost = float(st) * (120.0 + 70.0 * C)
        if best is None or cost < best:
            best, bc, bs = cost, C, st
    return bc, bs


def trace_stride(shapes) -> int:
    """uint16 entries of each warp's trace for a batch of (K, E) jobs"""
    t = 1
    for K, E in shapes:
        C, st = choose_class(K, E)
        t = max(t, (st + 1) * 32 * C)
    return (t + 63) // 64 * 64


def cta_trace_bytes(shapes) -> int:
    return 2 * trace_stride(shapes) * WARPS


def max_ctas(shapes, sm_count: int) -> int:
    """resident CTAs of each launch; 0 where the batch is refused (NPH_ERR_UNSUPPORTED)"""
    per = cta_trace_bytes(shapes)
    if per > TRACE_BUDGET:
        return 0
    return min(sm_count, max(1, TRACE_BUDGET // per))


def smallest_refused_square() -> int:
    """the smallest K = E whose one-job batch is refused"""
    lo, hi = 1000, 40000
    assert cta_trace_bytes([(lo, lo)]) <= TRACE_BUDGET < cta_trace_bytes([(hi, hi)])
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if cta_trace_bytes([(mid, mid)]) > TRACE_BUDGET:
            hi = mid
        else:
            lo = mid
    return hi


def smallest_capped_square(sm_count: int) -> int:
    """the smallest K = E whose one-job batch runs with fewer resident CTAs than SMs"""
    n = 32
    while max_ctas([(n, n)], sm_count) >= sm_count:
        n += 1
    return n


# ---------------------------------------------------------------- jobs
@dataclass
class Job:
    codes: np.ndarray         # bases the events were emitted from (forward strand)
    nev: np.ndarray           # events per k-mer of `codes`
    rc: bool
    flags: int
    indel_bias: float
    edges: set = field(default_factory=set)
    exact: np.ndarray | None = None     # bool per k-mer: its events sit exactly on the model level
    outlier_last: bool = False          # the window's last row is an event no k-mer can emit (-inf everywhere)

    @property
    def K(self) -> int:
        return int(self.codes.shape[0]) - K_MER + 1

    @property
    def E(self) -> int:
        return int(self.nev.sum())


def spread(rng, K: int, E: int) -> np.ndarray:
    """E events over K k-mers, the first and the last k-mer with at least one (E >= 2)"""
    nev = np.zeros(K, np.int64)
    if K == 1:
        nev[0] = E
        return nev
    nev[0] += 1; nev[-1] += 1
    np.add.at(nev, rng.integers(0, K, E - 2), 1)
    return nev


def plain(rng, K, E, rc=False, flags=0, bias=1.0, edges=()):
    codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
    return Job(codes, spread(rng, K, E), rc, flags, bias, set(edges))


def fits(K: int, E: int, C: int) -> bool:
    return choose_class(K, E)[0] == C


def pick_E(K: int, C: int, candidates) -> int | None:
    for E in list(candidates) + list(range(2, 3000)):
        if E >= 2 and fits(K, E, C):
            return E
    return None


_E_TRIES = (2, 3, 39, 40, 41, 24, 60, 100, 160, 240, 300, 400, 520)


def strip_edge_jobs(seed: int = 1):
    """per class: K = n*32C - 1, n*32C, n*32C + 1 for n = 1, 2, 3, each with an E that keeps the job in class C"""
    rng = np.random.default_rng(seed)
    out = []
    i = 0
    for C in COLS:
        strip = 32 * C
        for n in (1, 2, 3):
            for d, name in ((-1, "strip-1"), (0, "strip"), (1, "strip+1")):
                K = n * strip + d
                E = pick_E(K, C, _E_TRIES[i % 3:] + _E_TRIES[:i % 3])
                if E is None:
                    continue
                edges = {name}
                ns = (K + strip - 1) // strip
                if C > 1 and (K - (ns - 1) * strip) % C == 1:
                    edges.add("one-col-lane")
                if ns > 1 and E < MIN_PERIOD:
                    edges.add("short-period")
                out.append(plain(rng, K, E, rc=bool(i & 1), flags=i % 4, bias=(1.0, 0.9)[(i >> 1) & 1], edges=edges))
                i += 1
    return out


def one_col_jobs(seed: int = 8):
    """per class C > 1: a K whose last lane owns one column, away from the strip edges"""
    rng = np.random.default_rng(seed)
    out = []
    for i, C in enumerate(COLS[1:]):
        strip = 32 * C
        K, E = next((K, E) for K in range(strip + 2, 4 * strip) for E in (41, 100, 300, 39, 2, 24) if (K % strip) % C == 1 and K % strip > 1
                    and fits(K, E, C))
        out.append(plain(rng, K, E, rc=bool(i & 1), flags=(i + 1) % 4, bias=(0.9, 1.0)[i & 1], edges={"one-col-lane"}))
    return out


def event_count_jobs(seed: int = 2):
    """E in {2, 3, 39, 40, 41, 97} against K of several classes; E < 40 with several strips pads the period"""
    rng = np.random.default_rng(seed)
    out = []
    i = 0
    for K in (20, 70, 100, 150, 200, 330, 520):
        for E in (2, 3, 39, 40, 41, 97):
            C, _ = choose_class(K, E)
            strip = 32 * C
            ns = (K + strip - 1) // strip
            edges = {"short-period"} if (ns > 1 and E < MIN_PERIOD) else set()
            out.append(plain(rng, K, E, rc=bool(i % 3 == 1), flags=(i * 3) % 4, bias=(1.0, 0.9)[i & 1], edges=edges))
            i += 1
    return out


def _shape_for(C: int, Kmin: int, ratio: float, Emin: int = 2):
    """a (K, E) in class C with K >= Kmin, E >= Emin and E near ratio * K"""
    strip = 32 * C
    for K in range(max(Kmin, 8), 3 * strip + 200):
        for E in (int(ratio * K), int(ratio * K) + 7, int(ratio * K) - 7, 2 * K, K // 2, 41, 60, 100, 160):
            if E >= Emin and fits(K, E, C):
                return K, E
    return None


def skip_run_jobs(seed: int = 3):
    """48 k-mers without events spliced into the middle of the window, about one event for every other k-mer: a run of K
    states longer than the staged corner"""
    rng = np.random.default_rng(seed)
    out = []
    for i, C in enumerate(COLS[2:]):
        K, E = next((K, E) for K in range(90, 3000) for E in [*range(K - 48, K + K // 4), *range((K - 48) // 2, K - 48)]
                    if fits(K, E, C))
        a = K // 2 - 24
        nev = np.zeros(K - 48, np.int64)
        nev[rng.permutation(K - 48)[:min(E, K - 48)]] = 1
        np.add.at(nev, rng.integers(0, K - 48, E - int(nev.sum())), 1)
        nev = np.concatenate([nev[:a], np.zeros(48, np.int64), nev[a:]])
        codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
        out.append(Job(codes, nev, bool(i & 1), (0, 3, 1, 2, 0)[i], (1.0, 0.9)[i % 2], {"skip-run"}))
    return out


def stall_jobs(seed: int = 4):
    """56 events exactly on the level of one k-mer (a stalled pore): more rows on one k-mer than the staged corner holds"""
    rng = np.random.default_rng(seed)
    out = []
    for i, C in enumerate(COLS):
        K, E = _shape_for(C, 8 if C == 1 else 16 * C + 17, 1.8, Emin=58)
        nev = spread(rng, K, E - 56)
        nev[K // 2] += 56
        exact = np.zeros(K, bool)
        exact[K // 2] = True
        codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
        out.append(Job(codes, nev, bool(i & 1), (1, 2, 3, 0, 1, 2)[i], (0.9, 1.0)[i % 2], {"stall"}, exact=exact))
    return out


def homopolymer_jobs(seed: int = 5):
    """a 24-base run of one base (19 adjacent k-mers of one rank) whose events sit exactly on the model level"""
    rng = np.random.default_rng(seed)
    out = []
    for i, C in enumerate(COLS):
        K, E = _shape_for(C, 26 if C == 1 else 30 * C, 1.6)
        codes = rng.integers(0, 4, K + K_MER - 1).astype(np.uint8)
        a = max(0, min(K // 3, K + K_MER - 1 - 24))
        codes[a:a + 24] = i % 4
        nev = spread(rng, K, E)
        exact = np.zeros(K, bool)
        exact[max(0, a - K_MER + 1):a + 24] = True
        out.append(Job(codes, nev, bool(i & 1), (2, 0, 3, 1, 2, 3)[i], (1.0, 0.9)[i % 2], {"homopolymer"}, exact=exact))
    return out


def strip_cross_jobs(seed: int = 6):
    """several strips per class: the path crosses each strip boundary, usually inside one staged corner"""
    rng = np.random.default_rng(seed)
    out = []
    for i, C in enumerate(COLS[1:]):
        for j, ratio in enumerate((1.7, 0.6)):
            K, E = _shape_for(C, 32 * C + 5 + 29 * j, ratio)
            out.append(plain(rng, K, E, rc=bool((i + j) & 1), flags=(i + 2 * j) % 4, bias=(1.0, 0.9)[j], edges={"strip-cross"}))
    return out


def assert_jobs(seed: int = 7):
    """jobs the reference asserts on: one event, and a last event no k-mer can emit (its row is -inf in every MATCH cell)"""
    rng = np.random.default_rng(seed)
    out = []
    for i, (K, E) in enumerate(((30, 1), (150, 1), (40, 60), (200, 90), (700, 400))):
        j = Job(rng.integers(0, 4, K + K_MER - 1).astype(np.uint8), spread(rng, K, E) if E >= 2 else np.eye(1, K, K // 2, np.int64)[0],
                bool(i & 1), i % 4, (1.0, 0.9)[i % 2], {"asserts"}, outlier_last=E >= 2)
        out.append(j)
    return out


def all_jobs():
    return (strip_edge_jobs() + one_col_jobs() + event_count_jobs() + skip_run_jobs() + stall_jobs() + homopolymer_jobs() + strip_cross_jobs()
            + assert_jobs())


# ---------------------------------------------------------------- a batch of jobs as the C ABI takes it
@dataclass
class Batch:
    reads: np.ndarray
    ev_mean: np.ndarray
    ev_start_time: np.ndarray
    jobs: np.ndarray           # HMM_JOB_DT, model_id 0
    kmer_ranks: np.ndarray
    seqs: list                 # per job: the HMM sequence as the reference takes it (reverse complement for rc jobs)
    spec: list                 # the Job of each row


def make_batch(jobs, model, seed: int = 11) -> Batch:
    """one read per job: PAD noise events, the job's events, PAD noise events; the window is the job's events"""
    k = model.k
    reads = np.zeros(len(jobs), synth.READ_DT)
    rows, ranks, seqs, means, times = [], [], [], [], []
    off = 0
    for r, jb in enumerate(jobs):
        rng = np.random.default_rng(seed * 100003 + r)
        codes = jb.codes
        fr = synth.kmer_ranks_from_codes(codes, k, 4)
        which = np.repeat(np.arange(jb.K), jb.nev)
        E = which.shape[0]
        shift, scale, var = rng.uniform(-5.0, 5.0), rng.uniform(0.9, 1.1), rng.uniform(0.9, 1.3)
        t = np.arange(E + 2 * PAD, dtype=np.float64) * 0.002 + rng.uniform(0.0, 100.0)
        mu = scale * model.level_mean[fr[which]] + shift
        sd = var * model.level_stdv[fr[which]]
        noise = rng.standard_normal(E)
        if jb.exact is not None:
            noise[jb.exact[which]] = 0.0
        m = np.concatenate([rng.uniform(70, 110, PAD), mu + sd * noise, rng.uniform(70, 110, PAD)]).astype(np.float32)
        if jb.outlier_last:
            m[PAD if jb.rc else PAD + E - 1] = np.float32(1e30)
        reads[r] = (off, E + 2 * PAD, 0, scale, shift, 0.0, var, np.log(var), max(E / float(jb.K), 0.5))
        e0, e1 = PAD, PAD + E - 1
        if not jb.rc:
            ranks.append(fr)
            seqs.append(synth._CODE2DNA[codes].tobytes())
            rows.append((r, 0, e0, e1, 0, jb.flags))
        else:
            rcs = (3 - codes[::-1]).astype(np.uint8)
            ranks.append(synth.dna_rc_kmer_ranks(rcs, k))
            seqs.append(synth._CODE2DNA[rcs].tobytes())
            rows.append((r, 0, e1, e0, 1, jb.flags))
        means.append(m); times.append(t)
        off += E + 2 * PAD
    hj = synth._finish_jobs(rows, ranks)
    return Batch(reads, np.concatenate(means), np.concatenate(times), hj.jobs, hj.kmer_ranks, seqs, list(jobs))


def batches(model) -> dict:
    """all builder jobs, one batch per indel bias (the C ABI takes one bias per call)"""
    js = all_jobs()
    return {b: make_batch([j for j in js if j.indel_bias == b], model, seed=int(b * 10)) for b in (1.0, 0.9)}


def fingerprint(b, j: int, bias: float) -> str:
    """the inputs of job j of a batch (this module's or forward_cases'), under which the reference's answer is recorded"""
    jr = b.jobs[j]
    r = b.reads[int(jr["read"])]
    o, n = int(r["event_off"]), int(r["n_events"])
    h = hashlib.sha1()
    for part in (b.seqs[j], jr.tobytes(), r.tobytes(), b.ev_mean[o:o + n].tobytes(), b.ev_start_time[o:o + n].tobytes(),
                 np.float64(bias).tobytes()):
        h.update(part)
    return h.hexdigest()


# ---------------------------------------------------------------- edges seen on a path
def staged_corners(path, e_first: int, stride: int):
    """walk the path backwards as the kernel's backtrack does; yields (state index, re-stage reason or None)"""
    row0, kmer0 = 0, -1
    for i in range(path.shape[0] - 1, -1, -1):
        row = (int(path["event_idx"][i]) - e_first) * stride + 1
        kmer = int(path["kmer_idx"][i])
        reason = None
        if kmer0 < 0:
            reason = "first"
        elif row <= row0 - TILE or kmer <= kmer0 - TILE:
            reason = "both" if (row <= row0 - TILE and kmer <= kmer0 - TILE) else ("row" if row <= row0 - TILE else "kmer")
        if reason:
            row0, kmer0 = row, kmer
        yield i, reason


def longest_run(mask: np.ndarray) -> int:
    best = cur = 0
    for v in mask:
        cur = cur + 1 if v else 0
        best = max(best, cur)
    return best


def path_edges(path, job_row, spec: Job, ranks: np.ndarray) -> set:
    """the path-shape edges this path reaches"""
    got = set()
    if path.shape[0] == 0:
        return got
    e_first, stride = int(job_row["event_start"]), int(job_row["stride"])
    C, _ = choose_class(int(job_row["n_kmers"]), spec.E)
    strip = 32 * C
    st = path["state"]
    if longest_run(st == b"K") >= TILE + 1:
        got.add("skip-run")
    km = path["kmer_idx"].astype(np.int64)
    if longest_run(np.r_[False, km[1:] == km[:-1]]) + 1 >= TILE + 1:
        got.add("stall")
    steps = np.flatnonzero(km[1:] == km[:-1] + 1)
    if any(ranks[km[s]] == ranks[km[s] + 1] for s in steps):
        got.add("homopolymer")
    reasons = dict(staged_corners(path, e_first, stride))
    for s in steps:
        if km[s + 1] % strip == 0 and reasons[s] is None:    # state s (k-mer b-1) read from the corner that held state s+1 (k-mer b)
            got.add("strip-cross")
    return got


def check_edges(batch: Batch, paths, statuses) -> dict:
    """assert every job reached the edges it claims; returns {class: set of edges reached}"""
    cover = {C: set() for C in COLS}
    for j, (spec, path, status) in enumerate(zip(batch.spec, paths, statuses)):
        jr = batch.jobs[j]
        K = int(jr["n_kmers"])
        C, _ = choose_class(K, spec.E)
        if "asserts" in spec.edges:
            assert status != 0 and path.shape[0] == 0, f"job {j}: claimed to make the reference assert, oracle status {status}"
            continue
        assert status == 0 and path.shape[0] > 0, f"job {j}: oracle status {status}"
        got = path_edges(path, jr, spec, batch.kmer_ranks[int(jr["rank_off"]):int(jr["rank_off"]) + K])
        shape_claims = spec.edges & {"skip-run", "stall", "homopolymer", "strip-cross"}
        assert shape_claims <= got, f"job {j} (K={K}, E={spec.E}, C={C}): claims {sorted(shape_claims)}, path reaches {sorted(got)}"
        strip = 32 * C
        ns = (K + strip - 1) // strip
        for e in spec.edges - shape_claims:
            if e in ("strip-1", "strip", "strip+1"):
                assert (K - {"strip-1": -1, "strip": 0, "strip+1": 1}[e]) % strip == 0, f"job {j}: {e} with K={K}, C={C}"
            elif e == "one-col-lane":
                assert C > 1 and (K - (ns - 1) * strip) % C == 1, f"job {j}: one-col-lane with K={K}, C={C}"
            elif e == "short-period":
                assert ns > 1 and spec.E < MIN_PERIOD, f"job {j}: short-period with K={K}, E={spec.E}, C={C}"
        cover[C] |= got | spec.edges
    return cover


def coverage_table(covers) -> str:
    merged = {C: set() for C in COLS}
    for cv in covers:
        for C in COLS:
            merged[C] |= cv[C]
    lines = ["class " + " ".join(f"{e:>12}" for e in EDGES)]
    for C in COLS:
        lines.append(f"C={C:<3} " + " ".join(f"{('yes' if e in merged[C] else ('-' if e not in CLASS_EDGES[C] else 'NO')):>12}" for e in EDGES))
    return "\n".join(lines), merged
