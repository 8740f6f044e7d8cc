"""Timing of nph_all_support_batch on a `variants --calculate-all-support` workload: the pile-up of quick_fix_homopolymers.py (a 50 kb
draft region at depth 50, reads of 2 000 bases on both strands, a truth that differs from the draft by 400 homopolymer-length
indels), min_flanking_sequence 30, HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, with the truth's seeded edits as the variants.
Reports the variants, (variant, read) pairs, jobs and DP rows, the kernel time (nph_last_kernel_ms), the host's exp and fold time
and the whole call, the card's name, power limit and SM clock read in the same run, and — where oracle/_ref/libnpref_variants.so is
built — the compiled reference's own annotate_variants_with_all_support on one CPU thread over a sub-region of the same pile-up, per
(variant, read) pair.  Prints one JSON line.

  python scripts/quick_all_support.py [reps]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from nanopolish_b200.engine import Engine  # noqa: E402
from tests import support_cases as sc  # noqa: E402
from tests.ref_variants import RefVariants  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
model = synth.load_model("nucleotide")
eng = Engine(0)
eng.model_upload(model)


def case(ref_len, n_err, seed=77):
    draft, rs, recs, pairs, dur, deltas, first, truth = sc._pileup(("hp", ref_len, 50, 2000, seed, n_err, {}), model)
    c = dict(draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first, region_start=sc.REGION_START,
             region_end=sc.REGION_START + len(draft) - 1, region_ref=draft, flank=30, flags=sc.FLAGS, variants=truth)
    c["params"] = np.zeros(1, synth.SUPPORT_PARAMS_DT)
    c["params"][0] = (sc.REGION_START, 30, sc.FLAGS, 6)
    c["ref_seqs"], c["varr"] = sc.variant_array(truth)
    return c


c = case(50_000, 400)
res, cnt = sc.device(eng, c)                                # warm-up: module load, buffers
call_ms, kern_ms, host_ms = [], [], []
for _ in range(reps):
    t0 = time.perf_counter()
    res, cnt = sc.device(eng, c)                            # synchronous: returns with the support fractions on the host
    call_ms.append((time.perf_counter() - t0) * 1e3)
    kern_ms.append(eng.last_kernel_ms()[0])
    host_ms.append(float(cnt["host_ms"]))
row = dict(region_bases=len(c["draft"]), depth=50, reads=int(c["recs"].shape[0]), gpu=gpu, variants=int(cnt["n_variants"]),
           pairs=int(cnt["n_pairs"]), jobs=int(cnt["n_jobs"]), dp_rows=int(cnt["n_dp_rows"]), launches=eng.last_kernel_ms()[1],
           kernel_ms_median=float(np.median(kern_ms)), host_ms_median=float(np.median(host_ms)),
           call_ms_median=float(np.median(call_ms)), call_ms_min=float(np.min(call_ms)), call_ms_max=float(np.max(call_ms)))
row["pairs_per_s"] = row["pairs"] / (row["call_ms_median"] / 1e3)
if RefVariants.available():
    ref = RefVariants()
    ref.set_globals(1.0, 1)                                             # annotate_variants_with_all_support has no OpenMP; one thread all the same
    sub = case(3_000, 24, seed=78)
    hs, _ = ref.register(sub)
    t0 = time.perf_counter()
    ref.infos(sub, hs)
    secs = time.perf_counter() - t0
    _, cnt_sub = sc.device(eng, sub)
    row.update(ref_subregion_bases=3000, ref_subregion_variants=len(sub["variants"]), ref_subregion_pairs=int(cnt_sub["n_pairs"]),
               ref_all_support_s_1thread=secs, ref_ms_per_pair_1thread=secs * 1e3 / max(1, int(cnt_sub["n_pairs"])))
print(json.dumps(row), flush=True)
eng.close()
