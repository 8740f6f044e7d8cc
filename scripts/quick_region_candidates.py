"""Timing of the basecall candidate step of `nanopolish variants` (nph_region_candidates_batch, nph::get_variants_in_region) and of the
whole default-mode region call on one region: a 50 kb draft at depth 50 (reads of 2 000 bases on both strands, 30 true substitutions),
every basecall with 4 % substitutions, 3 % insertions of 1-3 bases, 3 % deletions and soft clips of up to 15 bases (tests/candidate_cases.py,
vcf_50k_p1).  Reports the device time of the candidate kernels and the whole device call, the host mirror's whole call
(nphh_variants_in_region: the records' compact form, the device call, the reference's std::map order, filter and std::sort) and its
share beyond the device call, the instances and distinct variants, and nph::call_variants_for_region + nph::write_variants_vcf at
ploidy 1 (the VCF's bytes equal the compiled reference's, tests/test_gpu_region_candidates.py), with the card's name, power limit and
SM clock read in the same run.  --reference times the compiled reference's own AlignmentDB::get_variants_in_region
(oracle/_ref/libnpref_variants.so) on one CPU thread instead.  Prints one JSON line.

  python scripts/quick_region_candidates.py [reps] [--reference]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from tests import candidate_cases as cc  # noqa: E402
from tests.ref_variants import RefVariants  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
reps = int(args[0]) if args else 5
c = cc.build_call(cc.CALL_CASES[0])
buffer = cc.CALL_FLANK + 10
cand = dict(c, start=c["region_start"] + buffer, stop=c["region_end"] - buffer)        # the window call_variants_for_region asks for
row = dict(region_bases=len(c["region_ref"]), depth=50, records=len(c["bases"]), record_bases=int(sum(len(b) for b in c["bases"])))

if "--reference" in sys.argv:
    ref = RefVariants()
    t = []
    for _ in range(max(1, min(reps, 3))):
        t0 = time.perf_counter()
        got = ref.variants_in_region(cand)
        t.append(time.perf_counter() - t0)
    row.update(ref_get_variants_in_region_s_1thread=float(np.median(t)), ref_kept=len(got),
               cpu=subprocess.run(["sh", "-c", "grep -m1 'model name' /proc/cpuinfo"], capture_output=True, text=True).stdout.strip())
    print(json.dumps(row), flush=True)
    sys.exit(0)

from nanopolish_b200.engine import Engine  # noqa: E402
from tests import host_mirror as hm  # noqa: E402

row["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip()
eng = Engine(0)
seq, deltas, recs = synth.seq_records(cand["bases"], cand["aligned"])
out, cnt = eng.region_candidates_batch(cand["region_ref"], cand["region_start"], seq, deltas, recs, cand["start"], cand["stop"])   # warm-up
kern, call = [], []
for _ in range(reps):
    t0 = time.perf_counter()
    out, cnt = eng.region_candidates_batch(cand["region_ref"], cand["region_start"], seq, deltas, recs, cand["start"], cand["stop"], cap=out.shape[0])
    call.append((time.perf_counter() - t0) * 1e3)
    kern.append(float(cnt["kernel_ms"]))
row.update(pairs=int(cnt["n_pairs"]), instances=int(cnt["n_instances"]), distinct=int(cnt["n_variants"]),
           device_kernel_ms_median=float(np.median(kern)), device_call_ms_median=float(np.median(call)))
host = hm.load()
cc.mirror(host, cand)
mir = []
for _ in range(reps):
    t0 = time.perf_counter()
    n, kept = cc.mirror(host, cand)
    mir.append((time.perf_counter() - t0) * 1e3)
    assert n >= 0, host.nphh_last_error()
row.update(kept=len(kept), mirror_call_ms_median=float(np.median(mir)),
           mirror_beyond_device_call_ms=float(np.median(mir) - np.median(call)))
region = []
for _ in range(max(1, min(reps, 3))):
    t0 = time.perf_counter()
    n, vcf = cc.call_region(host, c)
    region.append((time.perf_counter() - t0) * 1e3)
    assert n >= 0, host.nphh_last_error()
row.update(vcf_records=sum(1 for l in vcf.decode().splitlines() if not l.startswith("#")), region_call_and_vcf_with_read_registration_ms_median=float(np.median(region)))
print(json.dumps(row), flush=True)
eng.close()
