"""Timing of nph_homopolymer_likelihoods_batch on a `variants --fix-homopolymers` workload: a 50 kb draft region at depth 50 (reads
of 2 000 bases on both strands) whose truth differs from the draft by 400 homopolymer-length indels, min_flanking_sequence 30.
Reports the homopolymers, (homopolymer, read) pairs, jobs and DP rows, the kernel time (nph_last_kernel_ms), the host's log-gamma
time and the whole call, the card's name, power limit and SM clock read in the same run, and — where oracle/_ref/libnpref_variants.so
is built — the compiled reference's own fix_homopolymers on one CPU thread over a sub-region of the same pile-up, per
(homopolymer, read) pair.  Prints one JSON line.

  python scripts/quick_fix_homopolymers.py [reps]
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
from tests import hp_cases as hc  # noqa: E402
from tests import hp_restatement as hr  # noqa: E402
from tests.ref_variants import RefVariants  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
model = synth.load_model("nucleotide")
eng = Engine(0)
eng.model_upload(model)


def case(ref_len, n_err, seed=77):
    c = hc.build(("bench", (ref_len, 50, 2000, seed, n_err, 0), [], 30, 1.0, {}))
    return c


c = case(50_000, 400)
args = lambda: hc.device(eng, c)
liks, cnt = args()                                          # warm-up: module load, buffers
call_ms, kern_ms, host_ms = [], [], []
for _ in range(reps):
    t0 = time.perf_counter()
    liks, cnt = args()                                      # synchronous: returns with the vectors on the host
    call_ms.append((time.perf_counter() - t0) * 1e3)
    kern_ms.append(eng.last_kernel_ms()[0])
    host_ms.append(float(cnt["host_ms"]))
fixed = hr.fix_homopolymers(c["hap"], c["wins"], hc.vectors_of(liks))
called = len(fixed.variants)
row = dict(region_bases=len(c["draft"]), depth=50, reads=int(c["recs"].shape[0]), gpu=gpu, homopolymers=len(c["wins"]),
           pairs=int(cnt["n_pairs"]), jobs=int(cnt["n_jobs"]), dp_rows=int(cnt["n_dp_rows"]), chunks=int(cnt["n_chunks"]),
           seeded_errors=len(c["edits"]), called=called, launches=eng.last_kernel_ms()[1],
           kernel_ms_median=float(np.median(kern_ms)), host_lgamma_ms_median=float(np.median(host_ms)),
           call_ms_median=float(np.median(call_ms)), call_ms_min=float(np.min(call_ms)), call_ms_max=float(np.max(call_ms)))
row["pairs_per_s"] = row["pairs"] / (row["call_ms_median"] / 1e3)
if RefVariants.available():
    ref = RefVariants()
    ref.set_globals(1.0, 1)                                             # fix_homopolymers has no OpenMP; one thread all the same
    sub = case(3_000, 24, seed=78)
    hs, mh = ref.register(sub)
    t0 = time.perf_counter()
    ref.fixed(sub, hs)
    secs = time.perf_counter() - t0
    liks_sub, cnt_sub = hc.device(eng, sub)
    row.update(ref_subregion_bases=3000, ref_subregion_pairs=int(cnt_sub["n_pairs"]), ref_fix_homopolymers_s_1thread=secs,
               ref_ms_per_pair_1thread=secs * 1e3 / max(1, int(cnt_sub["n_pairs"])))
print(json.dumps(row), flush=True)
eng.close()
