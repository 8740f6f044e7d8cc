"""Bound model of the full-warp forward kernels on the scorereads classes (CPU only; a model, not a measurement).

Two resources can bind `hmm_forward_kernel<C, 32, false>`, one job per warp and 16 warps per SM:

* issue: each SM sub-partition (4 per SM) issues one warp instruction per clock, so a warp step of N
  instructions costs the SM N/4 clocks of issue;
* shared memory: the SM serves one wavefront per clock.  A warp-wide LDS takes as many wavefronts as the
  largest number of distinct 32-bit words any one of the 32 banks is asked for (same-word requests broadcast).

Issue side: `cuobjdump -sass` of the compiled kernel.  The steady-state warp step is the shortest path through
the step loop's body that performs at least 7*C table look-ups (every lane live, no end-state fold, no
soft-clip fold).  Its opcode histogram for C = 9 and C = 10 gives the per-column and per-step costs.

Shared-memory side: the kernel's lockstep schedule replayed on a sample of bench.py's own scorereads jobs.
At step g lane j owns row g - j + 1 and columns j*C .. j*C + C - 1; every look-up index comes from a float32
restatement of the recurrence in the kernel's (= oracle/np_oracle.c's) operation order.  Three index forms are
replayed on the same look-ups, per site (m1..m4 the match fold, b the bad state, k1 k2 the skip fold):
  * cut:       min(floor(|a - b| * 1000), 15700), NaN -> 15700 (exact_math.cuh's lsum, 8 instructions)
  * saturated: min(floor(|a - b| * 1000), 16384), NaN -> 0      (exact_math.cuh's lsum_sat, 7 instructions)
  * ideal:     the saturated form with every look-up that leaves the sum unchanged (mx + tbl[i] == mx) sent to one
               word; a bound on what a sink word for no-op look-ups could give, not a form the kernel has.

Usage: python scripts/k1_bounds.py [--jobs N] [--object path/to/hmm_forward_w32.o]
       python scripts/k1_bounds.py --compare parent/csrc/build new/csrc/build
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "nanopolish_b200", "csrc")
LOGSUM_CUT = 15700
SAT_INDEX = 16384          # the saturated index's largest value; the table holds 16385 entries
SITES = ("m1", "m2", "m3", "m4", "b", "k1", "k2")

# Steady-state warp step of the parent revision's kernels (cuobjdump -sass, CUDA 12.9, sm_90a), with the
# 8-instruction log-sum (FMUL, FMNMX clamp to 15700) instead of the saturated 7-instruction one.  Recorded here
# because the script compiles only the current source.
BEFORE = {
    9: {"total": 712, "ops": {"FADD": 216, "FADD.RM": 63, "FMNMX": 126, "FMUL": 81, "FFMA": 45, "IMAD/LEA": 65, "LDS": 63,
                              "SHFL": 3, "SEL/MOV": 19, "SETP/LOP": 9, "IADD": 3, "LDG": 1, "BRA/BSSY": 7, "other": 11}},
    10: {"total": 786, "ops": {"FADD": 240, "FADD.RM": 70, "FMNMX": 140, "FMUL": 90, "FFMA": 50, "IMAD/LEA": 72, "LDS": 70,
                               "SHFL": 3, "SEL/MOV": 20, "SETP/LOP": 9, "IADD": 3, "LDG": 1, "BRA/BSSY": 7, "other": 11}},
}


def compile_object(out_dir: str) -> str:
    obj = os.path.join(out_dir, "hmm_forward_w32.o")
    subprocess.run(["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC",
                    "-c", os.path.join(CSRC, "hmm_forward_w32.cu"), "-o", obj], check=True)
    return obj


# ---------------------------------------------------------------------------------------------------------
# issue side
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z0-9_.]+)([^;]*);")


def sass_functions(obj: str) -> dict[str, list[tuple[int, str, str, str]]]:
    txt = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs: dict[str, list] = {}
    cur = None
    for line in txt.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            funcs[cur] = []
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            funcs[cur].append((int(m.group(1), 16), (m.group(2) or "").strip(), m.group(3), m.group(4).strip()))
    return funcs


def _target(ops: str) -> int | None:
    m = re.search(r"0x([0-9a-f]+)", ops)
    return int(m.group(1), 16) if m else None


def _loops(insns, min_lds: int):
    """(length, head, tail) instruction-index ranges of the backward branches whose body holds >= min_lds LDS"""
    addr_ix = {a: i for i, (a, _, _, _) in enumerate(insns)}
    loops = []
    for i, (a, pred, op, ops) in enumerate(insns):
        if op.startswith("BRA") and not op.startswith("BRA.DIV"):
            t = _target(ops)
            if t is not None and t <= a:
                lo = addr_ix[t]
                lds = sum(1 for x in insns[lo:i + 1] if x[2].startswith("LDS"))
                if lds >= min_lds:
                    loops.append((i - lo, lo, i))
    return loops


def steady_step(insns, min_lds: int):
    """Shortest path (in instructions) through the innermost loop holding >= min_lds LDS, taking >= min_lds LDS."""
    _, head, tail = min(_loops(insns, min_lds))
    return _loop_step(insns, head, tail, min_lds)


def window_step(insns, C: int):
    """Step of the streamed kernel's transition window: the innermost loop with the soft-fold copy of column 0 (>= 7*C + 1 LDS),
    other than the steady loop, inside the smallest loop that encloses the steady loop (the stream).  None if there is none, as in
    a kernel without streaming, where the loop enclosing the step loop is the job loop and holds no second step loop."""
    row_loops = _loops(insns, 7 * C)
    _, sh, st = min(row_loops)
    outer = [(n, h, t) for n, h, t in row_loops if h <= sh and st <= t and (h, t) != (sh, st)]
    if not outer:
        return None
    _, oh, ot = min(outer)
    inner = [(n, h, t) for n, h, t in _loops(insns, 7 * C + 1)
             if oh <= h and t <= ot and (h, t) not in ((sh, st), (oh, ot))
             and not any(h <= h2 and t2 <= t and (h2, t2) != (h, t) for _, h2, t2 in row_loops)]
    if not inner:
        return None
    _, head, tail = min(inner, key=lambda x: x[1])
    return _loop_step(insns, head, tail, 7 * C + 1)


def _loop_step(insns, head: int, tail: int, min_lds: int):
    """Shortest path (in instructions) from head to tail taking >= min_lds LDS."""
    addr_ix = {a: i for i, (a, _, _, _) in enumerate(insns)}
    # DP over (instruction, LDS taken so far): fewest instructions issued
    INF = 1 << 30
    cap = min_lds
    best = [[INF] * (cap + 1) for _ in range(tail - head + 2)]
    prev = [[None] * (cap + 1) for _ in range(tail - head + 2)]
    best[0][0] = 0
    end = None
    for k in range(tail - head + 1):
        i = head + k
        a, pred, op, ops = insns[i]
        for l in range(cap + 1):
            d = best[k][l]
            if d >= INF:
                continue
            nl = min(cap, l + (1 if op.startswith("LDS") else 0))
            nd = d + 1
            succ = []
            if i == tail:
                if nl >= cap and (end is None or nd < end[0]):
                    end = (nd, k, l)
                continue
            is_bra = op.startswith("BRA") and not op.startswith("BRA.DIV")
            if is_bra:
                t = _target(ops)
                if t is not None and t > a and addr_ix[t] <= tail:
                    succ.append(addr_ix[t] - head)
                if pred:
                    succ.append(k + 1)
            elif op == "EXIT" and not pred:
                pass
            else:
                succ.append(k + 1)
            for s in succ:
                if nd < best[s][nl]:
                    best[s][nl] = nd
                    prev[s][nl] = (k, l)
    assert end is not None, "no steady-state path through the step loop"
    path = []
    k, l = end[1], end[2]
    while True:
        path.append(head + k)
        p = prev[k][l]
        if p is None:
            break
        k, l = p
    return [insns[i] for i in reversed(path)]


CLASSES = [("FADD", lambda o: o == "FADD" or o.startswith("FADD.FTZ")), ("FADD.RM", lambda o: o.startswith("FADD.RM")),
           ("FMNMX", lambda o: o.startswith("FMNMX")), ("FMUL", lambda o: o.startswith("FMUL")),
           ("FFMA", lambda o: o.startswith("FFMA")), ("IMAD/LEA", lambda o: o.startswith(("IMAD", "LEA"))),
           ("LDS", lambda o: o.startswith("LDS")), ("SHFL", lambda o: o.startswith("SHFL")),
           ("SEL/MOV", lambda o: o.startswith(("FSEL", "SEL", "MOV", "IMAD.MOV"))),
           ("SETP/LOP", lambda o: o.startswith(("ISETP", "FSETP", "PLOP3", "LOP3", "P2R", "R2P"))),
           ("IADD", lambda o: o.startswith(("IADD", "VIADD"))),
           ("LDG", lambda o: o.startswith("LDG")), ("BRA/BSSY", lambda o: o.startswith(("BRA", "BSSY", "BSYNC", "WARPSYNC")))]


def classify(path) -> collections.Counter:
    out = collections.Counter()
    for _, _, op, _ in path:
        for name, f in CLASSES:
            if f(op):
                out[name] += 1
                break
        else:
            out["other:" + op.split(".")[0]] += 1
    return out


def issue_side(obj: str) -> dict[int, dict]:
    """Per C: the steady step and the step of the streamed jobs' transition window (window_step; every lane live, no lane entering
    or leaving a job)."""
    funcs = sass_functions(obj)
    res = {}
    for C in (9, 10):
        name = f"_ZN7nph_fwd18hmm_forward_kernelILi{C}ELi32ELb0EEEvNS_9FwdParamsE"
        path = steady_step(funcs[name], 7 * C)
        window = window_step(funcs[name], C)
        res[C] = {"total": len(path), "ops": classify(path), "window": len(window) if window else None}
    return res


_KERNEL = re.compile(r"hmm_forward_kernelILi(\d+)ELi(\d+)ELb([01])E")


def _normalised(insns):
    """instructions without register numbers, branch targets and constant-bank offsets"""
    def norm(t):
        return re.sub(r"\b(U?[RP])\d+\b", r"\1", re.sub(r"0x[0-9a-f]+", "0x", t))
    return [(norm(pred), op, norm(ops)) for _, pred, op, ops in insns]


def compare_objects(parent_dir: str, new_dir: str) -> int:
    """Every hmm_forward_kernel<C, W, CHAIN> of the hmm_forward_w*.o in two build directories: same SASS or not, and the
    steady-state step's instruction count.  Returns the number of kernels that differ in more than instruction order."""
    rows, worse = [], 0
    for name in sorted(f for f in os.listdir(new_dir) if re.fullmatch(r"hmm_forward_w\d+c?\.o", f)):
        old, new = sass_functions(os.path.join(parent_dir, name)), sass_functions(os.path.join(new_dir, name))
        for fn in sorted(new, key=lambda f: tuple(int(x) for x in _KERNEL.search(f).groups()[::-1]) if _KERNEL.search(f) else ()):
            m = _KERNEL.search(fn)
            if not m or fn not in old:
                continue
            C, W, chain = int(m.group(1)), int(m.group(2)), m.group(3) == "1"
            a, b = _normalised(old[fn]), _normalised(new[fn])
            if a == b:
                verdict = "identical"
            elif collections.Counter(x[1] for x in a) == collections.Counter(x[1] for x in b):
                verdict = "same opcode histogram"
            else:
                verdict = "differs"
            steps = [len(steady_step(f[fn], 7 * C)) for f in (old, new)]
            worse += verdict == "differs" or steps[1] > steps[0]
            rows.append((C, W, chain, verdict, len(a), len(b), steps[0], steps[1]))
    print("| C | W | chained | SASS, registers and addresses normalised | instructions parent / new | steady step parent / new |")
    print("|---|---|---|---|---|---|")
    for C, W, chain, verdict, na, nb, sa, sb in rows:
        print(f"| {C} | {W} | {'yes' if chain else 'no'} | {verdict} | {na} / {nb} | {sa} / {sb} |")
    tally = collections.Counter(r[3] for r in rows)
    print(f"{len(rows)} kernels: " + ", ".join(f"{v} {k}" for k, v in sorted(tally.items())))
    return worse


# ---------------------------------------------------------------------------------------------------------
# shared-memory side
def _lsum(a, b, tbl):
    """kernel's lsum in float32; returns (result, index per form).  Both forms give the same sum: entries 15700..16384
    of the table are 0.0f, and the NaN difference (both operands -inf) adds log 2 or 0 to -inf."""
    with np.errstate(invalid="ignore", over="ignore"):
        mx = np.maximum(a, b)
        d = np.abs(a - b) * np.float32(1000.0)
        nan = np.isnan(d)
        cut = np.floor(np.where(nan, np.float32(LOGSUM_CUT), np.minimum(d, np.float32(LOGSUM_CUT)))).astype(np.int32)
        sat = np.floor(np.where(nan, np.float32(0.0), np.minimum(d, np.float32(SAT_INDEX)))).astype(np.int32)
        r = (mx + tbl[sat]).astype(np.float32)
        ideal = np.where(r == mx, LOGSUM_CUT, sat)   # one sink word for no-op look-ups (mx = -inf included)
        return r, {"cut": cut, "saturated": sat, "ideal": ideal}


FORMS = ("cut", "saturated", "ideal")


def job_indices(rs, jobs, j, model, tbl, consts):
    """look-up indices of every cell of job j, per form: array [site, row, column] (sites: m1..m4, b, k1, k2; -1 unused)"""
    job = jobs.jobs[j]
    rd = rs.reads[job["read"]]
    ranks = jobs.kmer_ranks[job["rank_off"]:job["rank_off"] + job["n_kmers"]].astype(np.int64)
    K = int(job["n_kmers"])
    e0, e1, st = int(job["event_start"]), int(job["event_stop"]), int(job["stride"])
    E = abs(e1 - e0) + 1
    ev = np.arange(E) * st + e0
    x = levels_of(rs, job["read"])[ev]
    mu = (rd["scale"] * model.level_mean[ranks] + rd["shift"]).astype(np.float32)
    sd = (model.level_stdv[ranks] * rd["var"]).astype(np.float32)
    lsd = (model.level_log_stdv[ranks] + rd["log_var"]).astype(np.float32)
    cc = (consts["log_inv_sqrt_2pi"] - lsd).astype(np.float32)
    lp_mm_self, lp_mm_next = consts["trans"][job["read"]]
    f32 = np.float32
    NEG = f32(-np.inf)
    idx = {f: np.full((7, E, K), -1, np.int32) for f in FORMS}

    def put(site, r, ix, c=slice(None)):
        for f in FORMS:
            idx[f][site, r, c] = ix[f]

    Mp = np.full(K, NEG, f32); Bp = Mp.copy(); Kp = Mp.copy()
    for r in range(E):
        a = ((f32(x[r]) - mu) / sd).astype(f32)
        em = (cc + (f32(-0.5) * a) * a).astype(f32)
        Ml = np.concatenate(([NEG], Mp[:-1])); Bl = np.concatenate(([NEG], Bp[:-1])); Kl = np.concatenate(([NEG], Kp[:-1]))
        m = (f32(lp_mm_self) + Mp).astype(f32)
        m, ix = _lsum(m, f32(lp_mm_next) + Ml, tbl); put(0, r, ix)
        m, ix = _lsum(m, consts["lp3"] + Bp, tbl); put(1, r, ix)
        m, ix = _lsum(m, consts["lp3"] + Bl, tbl); put(2, r, ix)
        m, ix = _lsum(m, consts["lp_km"] + Kl, tbl); put(3, r, ix)
        if r == 0:
            m[:1] = _lsum(m[:1], consts["flank"][:1], tbl)[0]       # soft-clip fold, column 0 of row 1
        m = (m + em).astype(f32)
        b, ix = _lsum(consts["lp_mb"] + Mp, consts["lp_bb"] + Bp, tbl); put(4, r, ix)
        kk1, ix = _lsum(consts["lp_mk"] + np.concatenate(([NEG], m[:-1])), consts["lp3"] + np.concatenate(([NEG], b[:-1])), tbl)
        put(5, r, ix)
        kk = np.empty(K, f32)
        prev = NEG
        lp_kk = consts["lp_kk"]
        for c in range(K):
            v, ix = _lsum(kk1[c:c + 1], np.array([lp_kk + prev], f32), tbl)
            kk[c] = v[0]; put(6, r, {f: ix[f][0] for f in FORMS}, c)
            prev = kk[c]
        Mp, Bp, Kp = m, b, kk
    return idx


_LEVELS = {}


def levels_of(rs, read):
    """drift-scaled event levels of one read (nph read prologue)"""
    if read not in _LEVELS:
        rd = rs.reads[read]
        o, n = int(rd["event_off"]), int(rd["n_events"])
        t = rs.ev_start_time[o:o + n]
        time = (t - t[0]).astype(np.float32).astype(np.float64)
        _LEVELS[read] = (rs.ev_mean[o:o + n].astype(np.float64) - time * float(rd["drift"])).astype(np.float32)
    return _LEVELS[read]


def wavefronts(idx, C: int):
    """replay lane j = row g - j + 1, columns j*C..: wavefronts per site (summed over steps and slots), and the steps"""
    S, E, K = idx.shape
    lanes = np.arange(32)
    end_lane = (K - 1) // C
    steps = E + end_lane
    total = np.zeros(S, np.int64)
    g = np.arange(steps)[:, None]
    row = g - lanes[None, :]                                   # 0-based row of lane j at step g
    valid_row = (row >= 0) & (row < E)
    for c in range(C):
        col = lanes * C + c
        ok = valid_row & (col < K)[None, :]
        rr = np.clip(row, 0, E - 1)
        cc = np.clip(col, 0, K - 1)
        for s in range(S):
            v = np.where(ok, idx[s][rr, cc[None, :]], -1)          # [steps, 32]
            v = np.sort(v, axis=1)
            first = np.ones_like(v, bool)
            first[:, 1:] = v[:, 1:] != v[:, :-1]
            first &= v >= 0
            bank = np.where(first, v & 31, 32)
            counts = np.zeros((steps, 33), np.int32)
            np.add.at(counts, (np.repeat(np.arange(steps), 32), bank.ravel()), 1)
            total[s] += counts[:, :32].max(axis=1).sum()
    return total, steps


def smem_side(n_jobs: int):
    from nanopolish_b200 import synth
    nuc = synth.load_model("nucleotide")
    rs = synth.gen_reads(max(1, n_jobs // 6 + 1), 4000, nuc, seed=42)      # bench.py: gen_reads(reads, 4000, seed=42 + ...)
    jobs = synth.scorereads_jobs(rs, 500, model_id=0)
    tbl = np.array([np.float32(np.log(1. + np.exp(-i / np.float32(1000.)))) for i in range(LOGSUM_CUT)]
                   + [0.0] * (SAT_INDEX + 1 - LOGSUM_CUT), np.float32)
    f = np.float32
    p_third = f((f(1.0) - f(0.001)) / f(3))
    consts = {"lp_mk": f(np.log(f(0.0025))), "lp_mb": f(np.log(f(0.001))), "lp_bb": f(np.log(f(0.001))),
              "lp3": f(np.log(p_third)), "lp_kk": f(np.log(f(0.3))), "lp_km": f(np.log(f(1.0) - f(0.3))),
              "log_inv_sqrt_2pi": f(np.log(0.3989422804014327))}
    consts["flank"] = np.array([np.log(1 - 0.5)], f)
    trans = []
    for rd in rs.reads:
        epb = max(1.25, float(rd["events_per_base"]))          # indel bias 1
        p_stay = f(1 - 1 / epb)
        trans.append((f(np.log(p_stay)), f(np.log(f(f(f(1.0) - p_stay) - f(0.0025)) - f(0.001)))))
    consts["trans"] = trans
    out = {}
    for C in (9, 10):
        out[C] = {"wavefronts": {f: np.zeros(len(SITES), np.int64) for f in FORMS}, "steps": 0, "jobs": 0, "lookups": 0}
    for j in range(min(n_jobs, len(jobs.jobs))):
        K = int(jobs.jobs[j]["n_kmers"])
        C = 9 if K <= 288 else 10
        if K > 320:
            continue
        idx = job_indices(rs, jobs, j, nuc, tbl, consts)
        o = out[C]
        for f in FORMS:
            w, st = wavefronts(idx[f], C)
            o["wavefronts"][f] += w
        o["steps"] += st; o["jobs"] += 1; o["lookups"] += 7 * C * st
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--jobs", type=int, default=180, help="bench scorereads jobs replayed for the shared-memory side")
    ap.add_argument("--object", default=None, help="compiled hmm_forward_w32.o (default: compile the current source)")
    ap.add_argument("--compare", nargs=2, metavar=("PARENT_OBJECTS", "NEW_OBJECTS"), default=None,
                    help="two directories of hmm_forward_w*.o: compare every forward kernel's SASS and steady-state step, then exit")
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare_objects(*args.compare) else 0)
    obj = args.object
    if obj is None:
        import tempfile
        obj = compile_object(tempfile.mkdtemp(prefix="k1_bounds_"))
    after = issue_side(obj)
    print("Issue side: steady-state warp step of hmm_forward_kernel<C, 32, false> (SASS instructions)")
    for C in (9, 10):
        for tag, d in (("before", BEFORE[C]), ("after", after[C])):
            ops = collections.Counter()
            for k, v in d["ops"].items():
                ops["other" if k.startswith("other") else k] += v
            print(f"  C={C:2d} {tag:6s} {d['total']:4d}: " + ", ".join(f"{k} {v}" for k, v in sorted(ops.items())))
    per_col = {t: d[10]["total"] - d[9]["total"] for t, d in (("before", BEFORE), ("after", after))}
    per_step = {t: d[9]["total"] - 9 * per_col[t] for t, d in (("before", BEFORE), ("after", after))}
    for t in ("before", "after"):
        print(f"  {t}: {per_step[t]} per warp step + {per_col[t]} per column")
    for C in (9, 10):
        print(f"  C={C:2d} transition window step (streamed jobs, 33 per job): {after[C]['window'] or 'no window'}")

    sm = smem_side(args.jobs)
    print(f"\nShared-memory side: look-up wavefronts, lockstep replay of bench scorereads jobs (seed 42)")
    for C in (9, 10):
        o = sm[C]
        if not o["jobs"]:
            continue
        site_lookups = o["lookups"] / len(SITES)
        print(f"  <{C},32,false>: {o['jobs']} jobs, {o['steps'] / o['jobs']:.1f} steps/job, {7 * C} LDS/step; wavefronts per LDS by site:")
        print("    " + f"{'form':10s}" + "".join(f"{s:>6s}" for s in SITES) + f"{'all':>6s}{'smem clk/step':>15s}")
        for f in FORMS:
            w = o["wavefronts"][f]
            print("    " + f"{f:10s}" + "".join(f"{x / site_lookups:6.2f}" for x in w)
                  + f"{w.sum() / o['lookups']:6.2f}{w.sum() / o['steps']:15.1f}")
    print("\nBound per warp step, per SM clock (max of issue and shared memory):")
    for C in (9, 10):
        o = sm[C]
        if not o["jobs"]:
            continue
        before = (BEFORE[C]["total"] / 4, o["wavefronts"]["cut"].sum() / o["steps"])
        now = (after[C]["total"] / 4, o["wavefronts"]["saturated"].sum() / o["steps"])
        print(f"  <{C},32,false>: before issue {before[0]:.1f}, smem {before[1]:.1f} -> {max(before):.1f};"
              f"  after issue {now[0]:.1f}, smem {now[1]:.1f} -> {max(now):.1f}  ({100 * (1 - max(now) / max(before)):.1f}% fewer clocks)")
    print("(per SM: 4 sub-partitions issue one warp instruction each per clock; shared memory serves one wavefront per clock;\n"
          " the look-ups at the fill/drain edges, where fewer lanes are live, are counted at what they cost)")


if __name__ == "__main__":
    main()
