"""Forward-HMM (profile_hmm_score) jobs built to reach named edges of the device forward kernel, csrc/hmm_forward_kernel.cuh, with
a restatement of the class choice in csrc/hmm_classes.h that decides which kernel instance, strip and lane a job reaches.

Restated from csrc/hmm_classes.h (not imported, so that a change there shows up as a failing test; tests/test_forward_classes.py
pins this restatement to the header compiled on the host):
  * nph_wave_geometry and total_steps: strips of W*C columns, a period of max(E, 40) rows between chained strips, and the steps
    until the lane holding k-mer K - 1 has done row E of the last strip;
  * nph_choose_class: the cheapest of the 50 (C, W, chained) classes by steps * (46 + 67 C) * W / 32, evaluated in float32 in
    the header's loop order (width outer, C inner) with strict <, so that ties go where the header sends them;
  * nph_key_bucket: a class's schedule runs level chunk ascending, then steps descending.

A class is (C, W, chained): C columns per lane, W lanes per job (32 / W jobs share a warp), chained = the W = 32 class whose jobs
are wider than one strip.  Jobs are vc.Job records (tests/viterbi_cases.py) batched by vc.make_batch, one read per job with drift 0;
`outlier_rows` adds events no k-mer can emit (level 1e30) at rows of the window.

Edge names (each builder tags a job with the edges it claims; `job_edges` recomputes them from the restatement and the test
asserts every claim):
  strip-1, strip, strip+1   K = n*W*C - 1, n*W*C, n*W*C + 1 (n = 1 single strip; n = 1..3 chained, where K > 32C)
  end-slot-0, end-slot-last the last k-mer sits in column 0, or column C - 1, of its lane (one and the same for C = 1)
  one-col-lane              the last lane owns one column (C > 1; the same jobs as end-slot-0)
  lanes-past-K              lanes of the group whose columns lie wholly beyond K (col0 >= K) in the last strip
  E=1, E=2                  one and two rows
  E=39, E=40, E=41          (chained) the period edge: P = max(E, 40) rows between strip starts
  short-period              (chained) E < 40 over several strips: rows E + 1 .. 40 of every period are dead
  one-row-strips            (chained) E = 1 over several strips: only row 1 is live in each period
  fwd-f<k>, rc-f<k>         flags k (0..3: pre-clip 1, post-clip 2) on the forward and the reverse strand; on the chained class
                            the post-clip fold runs in the last strip from its row 1
  bias-1.0, bias-0.9        indel bias
  outlier-mid, outlier-last an event at level 1e30 mid-window, and on the window's last row
  exact-level               events exactly on the model level of their k-mer
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

from tests import viterbi_cases as vc

MIN_PERIOD = 40               # NPH_MIN_PERIOD
MAX_COLS = 10                 # NPH_MAX_COLS
NUM_WIDTHS = 5                # W = 4, 8, 16, 32 single strip; 32 chained
STEP_BUCKETS = 1024           # NPH_STEP_BUCKETS
CHUNK_BUCKETS = 8             # NPH_CHUNK_BUCKETS
LEVEL_CHUNKS = 8              # nph_ctx::kLevelChunks: the one-shot call's level chunks
PIPELINE_MIN_EVENTS = 1 << 20 # the one-shot call streams levels in chunks from this many events on (all reads with drift 0)
WARPS_PER_SM_W32 = 16         # CtaShape<C, 32>::warps
STREAM_MIN_E = 33             # a full-warp single-strip job streams with more than 32 rows and flags without clipping


# ---------------------------------------------------------------- restatement of csrc/hmm_classes.h
def class_width(wi: int) -> int:
    return 32 if wi >= 3 else 4 << wi


def class_of(index: int) -> tuple[int, int, bool]:
    """(C, W, chained) of a class index (wi * 10 + C - 1)"""
    wi = index // MAX_COLS
    return index % MAX_COLS + 1, class_width(wi), wi == 4


def class_index(C: int, W: int, chained: bool) -> int:
    wi = 4 if chained else {4: 0, 8: 1, 16: 2, 32: 3}[W]
    return wi * MAX_COLS + C - 1


@dataclass
class Geom:
    K: int
    E: int
    C: int
    strip: int
    n_strips: int
    kpad: int
    P: int

    @property
    def last_strip(self) -> int:
        return self.n_strips - 1

    @property
    def end_lane(self) -> int:
        return ((self.K - 1) - self.last_strip * self.strip) // self.C

    @property
    def end_slot(self) -> int:
        return ((self.K - 1) - self.last_strip * self.strip) % self.C

    @property
    def total_steps(self) -> int:
        return self.last_strip * self.P + self.E + self.end_lane


def wave_geometry(K: int, E: int, C: int, W: int, may_chain: bool) -> Geom:
    strip = W * C
    ns = (K + strip - 1) // strip if may_chain else 1
    kpad = ns * strip
    P = max(E, MIN_PERIOD) if kpad > strip else E
    return Geom(K, E, C, strip, ns, kpad, P)


def choose_class_np(K, E):
    """(class index, steps) arrays for arrays of K and E: nph_choose_class elementwise"""
    K = np.asarray(K, np.int64)
    E = np.asarray(E, np.int64)
    best = np.full(K.shape, 3.0e38, np.float32)
    best_cls = np.full(K.shape, class_index(MAX_COLS, 32, True), np.int64)
    best_steps = np.zeros(K.shape, np.int64)
    f32 = np.float32
    for wi in range(NUM_WIDTHS):
        W = class_width(wi)
        chained = wi == 4
        for C in range(1, MAX_COLS + 1):
            fits = K <= W * C
            take = ~fits if chained else fits
            strip = W * C
            ns = (K + strip - 1) // strip
            P = np.where(ns > 1, np.maximum(E, MIN_PERIOD), E)
            steps = (ns - 1) * P + E + ((K - 1) - (ns - 1) * strip) // C
            cost = steps.astype(np.uint32).astype(f32) * (f32(46.0) + f32(67.0) * f32(C)) * (f32(W) * (f32(1.0) / f32(32.0)))
            upd = take & (cost < best)
            best = np.where(upd, cost, best)
            best_cls = np.where(upd, wi * MAX_COLS + C - 1, best_cls)
            best_steps = np.where(upd, steps, best_steps)
    return best_cls, best_steps


def choose_class(K: int, E: int) -> tuple[tuple[int, int, bool], int]:
    """((C, W, chained), steps) of one job"""
    c, s = choose_class_np(np.array([K]), np.array([E]))
    return class_of(int(c[0])), int(s[0])


def key_bucket(steps: int, chunk: int) -> int:
    b = steps if steps < 768 else 768 + (steps - 768) // 32
    b = min(b, STEP_BUCKETS - 1)
    chunk = min(chunk, CHUNK_BUCKETS - 1)
    return chunk * STEP_BUCKETS + (STEP_BUCKETS - 1 - b)


# the classes some K < 2000 reaches (tests/test_forward_classes.py checks this against the header): every sub-warp class at W = 4,
# C = 6..10 at W = 8, 16 and 32, and the chained class at C = 2..10.  The other 16 never win: a W = 8, 16 or 32 single strip with
# C <= 5 loses to the class of half the lanes and twice the columns, and a chained strip of 32 columns to one of 64 or more.
REACHABLE = frozenset([(C, 4, False) for C in range(1, 11)] + [(C, W, False) for W in (8, 16, 32) for C in range(6, 11)]
                      + [(C, 32, True) for C in range(2, 11)])
STREAMED = frozenset((C, 32, False) for C in range(6, 11))   # hmm_forward_kernel<C, 32, false> runs its jobs through run_stream


# ---------------------------------------------------------------- edges
STRIP_EDGES = ("strip-1", "strip", "strip+1")
SHAPE_EDGES = STRIP_EDGES + ("end-slot-0", "end-slot-last", "one-col-lane", "lanes-past-K", "E=1", "E=2")
CHAIN_EDGES = ("E=39", "E=40", "E=41", "short-period", "one-row-strips")
FLAG_EDGES = tuple(f"{s}-f{f}" for s in ("fwd", "rc") for f in range(4))
BIAS_EDGES = ("bias-1.0", "bias-0.9")
EVENT_EDGES = ("outlier-mid", "outlier-last", "exact-level")
EDGES = SHAPE_EDGES + CHAIN_EDGES + FLAG_EDGES + BIAS_EDGES + EVENT_EDGES
BIASES = (1.0, 0.9)

# the (K, E) grid the builders choose from: every K up to the widest strip edge (3 * 320 + 1) with E < 1200
GRID_K, GRID_E = 3 * 32 * MAX_COLS + 2, 1199


@functools.lru_cache(maxsize=None)
def _grid():
    K, E = np.meshgrid(np.arange(1, GRID_K + 1), np.arange(1, GRID_E + 1), indexing="ij")
    K, E = K.ravel(), E.ravel()
    c, s = choose_class_np(K, E)
    return K, E, c, s


def _class_grid(cls):
    """the grid's (K, E, steps) in class cls, with at most 8 events per k-mer and 40 more, so that the jobs stay near what reads
    hold; `long_window_jobs` adds windows with up to 240 rows per k-mer"""
    K, E, c, s = _grid()
    sel = (c == class_index(*cls)) & (E <= 8 * K + 40)
    return K[sel], E[sel], s[sel]


def edge_masks(K, E, cls) -> dict:
    """{shape edge: bool array} for arrays of (K, E) that lie in class cls"""
    C, W, chained = cls
    K, E = np.asarray(K, np.int64), np.asarray(E, np.int64)
    strip = W * C
    ns = (K + strip - 1) // strip
    rest = K - 1 - (ns - 1) * strip
    end_lane, end_slot = rest // C, rest % C
    m = {}
    for d, name in zip((-1, 0, 1), STRIP_EDGES):
        n = (K - d) // strip
        m[name] = ((K - d) % strip == 0) & (n >= 1) & (n <= (3 if chained else 1))
    m["end-slot-0"] = end_slot == 0
    m["end-slot-last"] = end_slot == C - 1
    m["one-col-lane"] = (end_slot == 0) & (C > 1)
    m["lanes-past-K"] = end_lane < W - 1
    for e in (1, 2):
        m[f"E={e}"] = E == e
    for e in (39, 40, 41):
        m[f"E={e}"] = (E == e) & chained
    m["short-period"] = (E < MIN_PERIOD) & (ns > 1)
    m["one-row-strips"] = (E == 1) & (ns > 1)
    return m


def shape_edges(K: int, E: int) -> set:
    """the shape edges a (K, E) job reaches in the class the restatement gives it"""
    cls, _ = choose_class(K, E)
    return {n for n, v in edge_masks([K], [E], cls).items() if v[0]}


@functools.lru_cache(maxsize=None)
def class_edges(cls) -> frozenset:
    """the edges class cls can hold: the shape edges some (K, E) of the builders' grid reaches in it, and every strand, flag, bias and
    event edge.  What a class cannot hold follows from the cost model: the last lane owns one column only at C <= 4 for W = 4 and
    C <= 8 for W = 8, one row never reaches W = 8 and 16 at C = 6 or W = 32 at C = 6 and 7, two rows never W = 16 and 32 at C = 6;
    the chained class takes K = 32C + 1 only at C = 2, E = 39..41 only at C <= 6, and one or two rows only at C >= 6."""
    Kc, Ec, _ = _class_grid(cls)
    shape = {n for n, v in edge_masks(Kc, Ec, cls).items() if v.any()}
    return frozenset(shape | set(FLAG_EDGES) | set(BIAS_EDGES) | set(EVENT_EDGES))


# ---------------------------------------------------------------- jobs
@dataclass
class Job(vc.Job):
    outlier_rows: tuple = ()      # rows of the window (1..E) whose event sits at level 1e30


def job_edges(spec: Job) -> set:
    """every edge a job reaches (its shape from the restatement, then strand, flags, bias and events)"""
    out = shape_edges(spec.K, spec.E)
    out.add(f"{'rc' if spec.rc else 'fwd'}-f{spec.flags}")
    out.add(f"bias-{spec.indel_bias}")
    if spec.E in spec.outlier_rows:
        out.add("outlier-last")
    if any(1 < r < spec.E for r in spec.outlier_rows):
        out.add("outlier-mid")
    if spec.exact is not None and spec.exact.any():
        out.add("exact-level")
    return out


def spread(rng, K: int, E: int) -> np.ndarray:
    """vc.spread, and for E = 1 the one event on a random k-mer"""
    if E >= 2 or K == 1:
        return vc.spread(rng, K, E)
    return np.eye(1, K, int(rng.integers(0, K)), np.int64)[0]


def _pick(Kc, Ec, mask):
    """the (K, E) of mask with rows nearest to 1.6 per k-mer (within 3..400), then the smallest K"""
    idx = np.flatnonzero(mask)
    target = np.clip(Kc[idx] * 8 // 5, 3, 400)
    best = idx[np.lexsort((Kc[idx], np.abs(Ec[idx] - target)))[0]]
    return int(Kc[best]), int(Ec[best])


def class_shapes(cls) -> list:
    """(K, E, edges claimed) of class cls: every strip edge n*W*C + d the class holds, then one job for each other shape edge
    the jobs so far miss"""
    C, W, chained = cls
    Kc, Ec, _ = _class_grid(cls)
    masks = edge_masks(Kc, Ec, cls)
    out = []
    for n in (1, 2, 3) if chained else (1,):
        for d, name in zip((-1, 0, 1), STRIP_EDGES):
            m = Kc == n * W * C + d
            if m.any():
                K, E = _pick(Kc, Ec, m)
                out.append((K, E, {name}))
    have = set().union(*(shape_edges(K, E) for K, E, _ in out)) if out else set()
    for name in SHAPE_EDGES + CHAIN_EDGES:
        if name not in have and masks[name].any():
            K, E = _pick(Kc, Ec, masks[name])
            out.append((K, E, {name}))
            have |= shape_edges(K, E)
    return out


def class_jobs(cls, seed: int) -> list:
    """the edge jobs of one class: its shapes, three event-edge jobs, and random jobs of the class up to 16, with strand, flags
    and bias cycling so that each of the 16 combinations occurs"""
    rng = np.random.default_rng(seed)
    shapes = class_shapes(cls)
    Kc, Ec, _ = _class_grid(cls)
    K, E = _pick(Kc, Ec, Ec >= 3)
    shapes += [(K, E, {"outlier-mid"}), (K, E, {"outlier-last"}), (K, E, {"exact-level"})]
    small = np.flatnonzero(Kc * Ec <= 40000)
    while len(shapes) < 16:
        i = int(rng.choice(small))
        shapes.append((int(Kc[i]), int(Ec[i]), set()))
    jobs = []
    for i, (K, E, claims) in enumerate(shapes):
        flags, rc, bias = i % 4, bool((i // 4) % 2), BIASES[(i // 8) % 2]
        j = Job(rng.integers(0, 4, K + vc.K_MER - 1).astype(np.uint8), spread(rng, K, E), rc, flags, bias,
                claims | {f"{'rc' if rc else 'fwd'}-f{flags}", f"bias-{bias}"})
        if "outlier-mid" in claims:
            j.outlier_rows = (E // 2 + 1,)
        elif "outlier-last" in claims:
            j.outlier_rows = (E,)
        elif "exact-level" in claims:
            j.exact = np.ones(K, bool)
        jobs.append(j)
    return jobs


# ---------------------------------------------------------------- the warps of a sub-warp class
def schedule_keys(steps, chunks=None) -> np.ndarray:
    """the schedule key of each job in its class's slice (ascending = earlier)"""
    chunks = np.zeros(len(steps), np.int64) if chunks is None else chunks
    return np.array([key_bucket(int(s), int(c)) for s, c in zip(steps, chunks)], np.int64)


def fixed_warps(keys, G: int) -> list:
    """the warps of a class (G jobs each, in schedule order) whose set of jobs the schedule fixes whatever order it gives the
    jobs of one key: lists of positions into keys"""
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    bounds = {0, len(sk)} | {i for i in range(1, len(sk)) if sk[i] != sk[i - 1]}
    out = []
    for a in range(0, len(sk), G):
        z = min(a + G, len(sk))
        if a in bounds and z in bounds:
            out.append(sorted(order[a:z].tolist()))
    return out


def mixed_warp(specs, G: int) -> bool:
    """a fixed warp holds jobs of different step counts, and pre-clip jobs next to others (the soft fold on for every row)"""
    steps = np.array([choose_class(s.K, s.E)[1] for s in specs])
    for w in fixed_warps(schedule_keys(steps), G):
        pre = {bool(specs[i].flags & 1) for i in w}
        if pre == {False, True} and len({int(steps[i]) for i in w}) > 1:
            return True
    return False


def _mix_jobs(cls, specs, bias, rng) -> list:
    """G jobs of class cls whose steps exceed every job of specs, all different: they fill the class's first warp alone,
    pre-clip and not in turn"""
    C, W, _ = cls
    G = 32 // W
    Kc, Ec, Sc = _class_grid(cls)
    top = max(choose_class(s.K, s.E)[1] for s in specs)
    out, seen = [], set()
    for i in np.argsort(Sc, kind="stable"):
        if Sc[i] > top and int(Sc[i]) not in seen and Kc[i] * Ec[i] <= 200000:
            seen.add(int(Sc[i]))
            K, E = int(Kc[i]), int(Ec[i])
            fl = (1, 0, 3, 2)[len(out) % 4]
            out.append(Job(rng.integers(0, 4, K + vc.K_MER - 1).astype(np.uint8), spread(rng, K, E), bool(len(out) & 1), fl, bias,
                           {f"{'rc' if len(out) & 1 else 'fwd'}-f{fl}", f"bias-{bias}"}))
            if len(out) == G:
                return out
    raise AssertionError(f"class {cls}: fewer than {G} step counts above {top}")


def all_jobs() -> list:
    """every class's edge jobs; in each indel-bias batch a sub-warp class has a job count that is not a multiple of its jobs per
    warp (the last warp has empty groups) and a warp that mixes step counts and pre-clipping"""
    out = []
    for n, cls in enumerate(sorted(REACHABLE, key=lambda c: (c[2], c[1], c[0]))):
        js = class_jobs(cls, seed=1000 + n)
        C, W, _ = cls
        if W < 32:
            rng = np.random.default_rng(2000 + n)
            G = 32 // W
            for bias in BIASES:
                mine = [j for j in js if j.indel_bias == bias]
                if not mixed_warp(mine, G):
                    mine += _mix_jobs(cls, mine, bias, rng)
                if len(mine) % G == 0:
                    Kc, Ec, _ = _class_grid(cls)
                    i = int(rng.choice(np.flatnonzero(Kc * Ec <= 40000)))
                    K, E = int(Kc[i]), int(Ec[i])
                    mine.append(Job(rng.integers(0, 4, K + vc.K_MER - 1).astype(np.uint8), spread(rng, K, E), False, 0, bias,
                                    {"fwd-f0", f"bias-{bias}"}))
                js = [j for j in js if j.indel_bias != bias] + mine
        out += js
    return out


# ---------------------------------------------------------------- batches
def make_batch(jobs, model, seed: int = 11) -> vc.Batch:
    """vc.make_batch, with the outlier rows of each job set to 1e30"""
    b = vc.make_batch(jobs, model, seed)
    for r, jb in enumerate(jobs):
        off = int(b.reads[r]["event_off"])
        for row in getattr(jb, "outlier_rows", ()):
            b.ev_mean[off + vc.PAD + (jb.E - row if jb.rc else row - 1)] = np.float32(1e30)
    return b


# Rows per k-mer where a window still has a score: events_per_base (E / K in these batches) above about 286 makes p_mm_next of
# calculate_transitions negative and its log NaN, and the reference and the port oracle then index their log-sum table with NaN
# (the reference dies of SIGSEGV).
MAX_ROWS_PER_KMER = 240


def long_window_jobs(bias: float, seed: int = 5) -> list:
    """eight windows of one to four k-mers with 188 to 921 events (up to MAX_ROWS_PER_KMER per k-mer), past the grid's bound.  They
    all go to class (1, 4, False) with more steps than its other jobs, all different, so they fill its first warp alone, pre-clip
    and not in turn: its job count modulo 8 and its mixed warp stay as they were"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(8):
        K = 1 + i % 4
        E, fl, rc = MAX_ROWS_PER_KMER * K - 13 * i, (1, 0, 3, 2)[i % 4], bool(i & 1)
        assert choose_class(K, E)[0] == (1, 4, False) and 8 * K + 40 < E <= MAX_ROWS_PER_KMER * K
        out.append(Job(rng.integers(0, 4, K + vc.K_MER - 1).astype(np.uint8), spread(rng, K, E), rc, fl, bias,
                       {f"{'rc' if rc else 'fwd'}-f{fl}", f"bias-{bias}"}))
    return out


def batches(model) -> dict:
    """all builder jobs, one batch per indel bias (the C ABI takes one bias per call)"""
    js = all_jobs()
    return {b: make_batch([j for j in js if j.indel_bias == b] + long_window_jobs(b), model, seed=int(b * 10) + 3) for b in BIASES}


def code_form(b: vc.Batch):
    """(seq_codes, jobs) of the base-code form (nph_hmm_score_batch_seq): the forward-strand bases of each job, rank_off = their
    offset"""
    codes = [s.codes for s in b.spec]
    jobs = b.jobs.copy()
    jobs["rank_off"] = np.concatenate([[0], np.cumsum([c.shape[0] for c in codes])[:-1]]).astype(np.uint64)
    return np.concatenate(codes).astype(np.uint8), jobs


def classes_of(b: vc.Batch) -> list:
    c, _ = choose_class_np(b.jobs["n_kmers"], [s.E for s in b.spec])
    return [class_of(int(x)) for x in c]


# ---------------------------------------------------------------- coverage
def check_claims(b: vc.Batch) -> dict:
    """assert every job reaches the edges it claims; returns {class: edges reached}"""
    cover = {c: set() for c in REACHABLE}
    for j, s in enumerate(b.spec):
        assert int(b.jobs[j]["n_kmers"]) == s.K
        got = job_edges(s)
        assert s.edges <= got, f"job {j} (K={s.K}, E={s.E}, flags {s.flags}, rc {s.rc}): claims {sorted(s.edges - got)} it misses"
        cover[choose_class(s.K, s.E)[0]] |= got
    return cover


def coverage_table(covers) -> tuple[str, dict]:
    """yes: a job reaches the edge; -: the class cannot hold it; NO: it can and no job does"""
    merged = {c: set() for c in REACHABLE}
    for cv in covers:
        for c in REACHABLE:
            merged[c] |= cv[c]
    names = [e.replace("bias-", "b") for e in EDGES]
    lines = ["class        " + " ".join(f"{n:>6.6}" for n in names)]
    for c in sorted(REACHABLE, key=lambda c: (c[2], c[1], c[0])):
        cells = ["yes" if e in merged[c] else ("-" if e not in class_edges(c) else "NO") for e in EDGES]
        lines.append(f"C={c[0]:<2} W={c[1]:<2} {'ch' if c[2] else '  '} " + " ".join(f"{x:>6}" for x in cells))
    return "\n".join(lines), merged


# ---------------------------------------------------------------- the pipelined one-shot call
def level_chunk_events(n_events_total: int) -> int:
    """events per level chunk of the one-shot call (nph_api.cu: total / 8 rounded up to a multiple of 32)"""
    c = (n_events_total + LEVEL_CHUNKS - 1) // LEVEL_CHUNKS
    return (c + 31) // 32 * 32


def pipelined_batch(model, seed: int = 17, per_class: int = 6000, n_sub_warp: int = 700):
    """(batch, chunk of each job): per_class jobs in each streamed class (K 161..320, E > 32, flags 0 but for about every sixth job)
    and n_sub_warp jobs of the sub-warp classes, in random read order; drift 0 on every read and several times 2^20 events, so that
    the one-shot call copies the levels in chunks behind a progress word and every chunk holds jobs of every class.  With 6 000 jobs
    a streamed class has more than twice as many streamable jobs as the warps of its launch, so warps pull further jobs inside
    run_stream, through the progress check of fetch_job."""
    rng = np.random.default_rng(seed)
    shapes = []
    for cls in sorted(STREAMED):
        C = cls[0]
        got = []
        while len(got) < per_class:
            K = rng.integers(32 * (C - 1) + 1, 32 * C + 1, 4 * per_class)
            E = rng.integers(STREAM_MIN_E, 321, 4 * per_class)
            ok = choose_class_np(K, E)[0] == class_index(*cls)
            got += list(zip(K[ok].tolist(), E[ok].tolist()))
        shapes += got[:per_class]
    while len(shapes) < len(STREAMED) * per_class + n_sub_warp:
        K = rng.integers(1, 161, 4 * n_sub_warp)
        E = rng.integers(1, 8 * K + 41)
        ok = np.array([class_of(int(c))[1] < 32 for c in choose_class_np(K, E)[0]])
        shapes += list(zip(K[ok].tolist(), E[ok].tolist()))[:len(STREAMED) * per_class + n_sub_warp - len(shapes)]
    specs = []
    for i in rng.permutation(len(shapes)):
        K, E = shapes[i]
        fl = int(rng.integers(1, 4)) if rng.integers(0, 6) == 0 else 0
        specs.append(Job(rng.integers(0, 4, K + vc.K_MER - 1).astype(np.uint8), spread(rng, K, E), bool(rng.integers(0, 2)), fl, 1.0))
    b = make_batch(specs, model, seed=seed)
    ce = level_chunk_events(b.ev_mean.shape[0])
    rr = b.reads[b.jobs["read"]]
    return b, ((rr["event_off"] + rr["n_events"] - 1) // ce).astype(np.int64)


def rising_chunk_boundaries(b: vc.Batch, chunks) -> list:
    """(class, chunk) where, in the class's schedule, the jobs that end chunk c and the jobs that open chunk c + 1 all stream, and
    every one of the latter has more rows than every one of the former: a warp that streams from one to the other enters a longer
    job of a later level chunk"""
    cls_idx, steps = choose_class_np(b.jobs["n_kmers"], [s.E for s in b.spec])
    E = np.array([s.E for s in b.spec])
    streams = (E >= STREAM_MIN_E) & (np.array([s.flags for s in b.spec]) == 0)
    keys = np.array([key_bucket(int(st), int(ch)) for st, ch in zip(steps, chunks)])
    out = []
    for cls in sorted({class_of(int(c)) for c in np.unique(cls_idx)} & STREAMED):
        mine = cls_idx == class_index(*cls)
        for c in range(int(chunks[mine].min()), int(chunks[mine].max())):
            before, after = mine & (chunks == c), mine & (chunks == c + 1)
            if not before.any() or not after.any():
                continue
            a = mine & (keys == keys[before].max())      # the jobs that end chunk c in the schedule, in any order
            z = mine & (keys == keys[after].min())       # and those that open chunk c + 1
            if streams[a | z].all() and E[z].min() > E[a].max():
                out.append((cls, c))
    return out
