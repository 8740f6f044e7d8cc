"""Timing of nph_call_variant_groups_batch on one `variants` region: a 50 kb draft at depth 50 (reads of 2 000 bases on both strands)
whose truth differs from it by 400 substitutions.  The candidates are the truth's substitutions, a wrong substitution 2 bases after
each (the pair forms one group) and 400 wrong substitutions on their own; min_flanking_sequence 30, min_distance_between_variants 10,
max_haplotypes 1000, HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, ploidy 1 and 2.  Reports per ploidy the groups, haplotypes, jobs, DP rows,
genotype sets and set x key terms, the forward-kernel, genotype-kernel and host times and the whole call, with the card's name, power
limit and SM clock read in the same run.  Where oracle/_ref/libnpref_variants.so is built (and no GPU is needed for it), --reference
times the compiled reference's own call_haplotype_from_candidates on one CPU thread over the first 60 candidates instead.  Prints one
JSON line.

  python scripts/quick_call_variants.py [reps] [--reference]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from tests import call_cases as cc  # noqa: E402
from tests.ref_variants import RefVariants  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
reps = int(args[0]) if args else 5
model = synth.load_model("nucleotide")
draft, rs, recs, pairs, dur, deltas, first, truth = cc.suc._pileup(("snp", 50_000, 50, 2000, 77, 400), model)
rng = np.random.default_rng(77)
d = lambda p: draft[p - cc.REGION_START]
other = lambda p: "ACGT"[("ACGT".index(d(p)) + 1) % 4]
lo, hi = cc.REGION_START + 40, cc.REGION_START + len(draft) - 60
cands = []
for p, r, a in truth:
    if lo <= p < hi:
        cands += [(p, r, a), (p + 2, d(p + 2), other(p + 2))]
cands += [(int(p), d(int(p)), other(int(p))) for p in rng.integers(lo, hi, 400)]
cands.sort()
c = dict(draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, region_start=cc.REGION_START, region_end=cc.REGION_START + len(draft) - 1,
         region_ref=draft, genotype_only=0, max_haplotypes=1000, types=(), all_support=0, candidates=cands,
         names=[f"r{i}" for i in range(rs.reads.shape[0])])
row = dict(region_bases=len(draft), depth=50, reads=int(recs.shape[0]), candidates=len(cands))

if "--reference" in sys.argv:
    ref = RefVariants()
    sub = dict(c, candidates=cands[:60], ploidy=2)
    hs, _ = ref.register(sub)
    t0 = time.perf_counter()
    ref.called(sub, hs)
    secs = time.perf_counter() - t0
    row.update(ref_candidates=60, ref_groups=len(cc.cr.groups(cands[:60], cc.FLANK, cc.MIN_DISTANCE)), ref_call_s_1thread=secs,
               cpu=subprocess.run(["sh", "-c", "grep -m1 'model name' /proc/cpuinfo"], capture_output=True, text=True).stdout.strip())
    print(json.dumps(row), flush=True)
    sys.exit(0)

from nanopolish_b200.engine import Engine  # noqa: E402

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
row["gpu"] = gpu
eng = Engine(0)
eng.model_upload(model)
ref_bases = np.frombuffer(draft.encode(), np.uint8).copy()
for ploidy in (1, 2):
    c["ploidy"] = ploidy
    p, groups, haps, bases, cvars, nv, kr = cc.device_inputs(c, genotype_all=0)

    def call():
        return eng.call_variant_groups_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref_bases, deltas, first, recs, kr, p, groups, haps, bases,
                                             cvars, nv)
    g, v, cnt = call()                                                 # warm-up: module load, buffers
    call_ms, fwd, gt, host = [], [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        g, v, cnt = call()                                             # synchronous: returns with the results on the host
        call_ms.append((time.perf_counter() - t0) * 1e3)
        fwd.append(float(cnt["forward_ms"])); gt.append(float(cnt["genotype_ms"])); host.append(float(cnt["host_ms"]))
    row[f"ploidy{ploidy}"] = dict(groups=int(cnt["n_groups"]), haplotypes=int(cnt["n_haplotypes"]), pairs=int(cnt["n_pairs"]),
                                  jobs=int(cnt["n_jobs"]), dp_rows=int(cnt["n_dp_rows"]), sets=int(cnt["n_sets"]),
                                  set_terms=int(cnt["n_set_terms"]), called=int((g["status"] == synth.CALL_CALLED).sum()),
                                  forward_ms_median=float(np.median(fwd)), genotype_ms_median=float(np.median(gt)),
                                  host_ms_median=float(np.median(host)), call_ms_median=float(np.median(call_ms)),
                                  call_ms_min=float(np.min(call_ms)), call_ms_max=float(np.max(call_ms)))
print(json.dumps(row), flush=True)
eng.close()
