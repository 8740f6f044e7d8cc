"""Timing of nph_phase_reads_batch on the synthetic phase-reads workload: reads of 4 000 events on both strands, heterozygous SNPs
every 100-1 000 bases, at 512 and 10 000 reads; next to the compiled reference's profile_hmm_score over the same windows on one CPU
thread (the two forward scores per site that make up almost all of phase_single_read's work).  Prints one JSON line per size.

  python scripts/quick_phase_reads.py [n_events] [reps]
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
from oracle.oracle_py import RefOracle  # noqa: E402
from tests import phase_restatement as pr  # noqa: E402

n_events = int(sys.argv[1]) if len(sys.argv) > 1 else 4000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
model = synth.load_model("nucleotide")
eng = Engine(0)
eng.model_upload(model)
ref_o = RefOracle() if RefOracle.available() else None
for n_reads in (512, 10_000):
    rs = synth.gen_reads(n_reads, n_events, model, seed=2024)
    ref, pairs, recs, variants, vr = synth.phase_batch(rs, seed=1, step=(100, 1000), p_mismatch=0.0, p_non_snp=0.0, p_no_variants=0.0, p_iupac=0.0)
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    args = (rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs, variants, vr)
    eng.phase_reads_batch(*args)                                   # warm-up: module load, buffers
    call_ms, kern_ms = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        off, calls, scored = eng.phase_reads_batch(*args)          # synchronous: returns after the calls are on the host
        call_ms.append((time.perf_counter() - t0) * 1e3)
        kern_ms.append(eng.last_kernel_ms()[0])
    launches = eng.last_kernel_ms()[1]
    row = dict(n_reads=n_reads, n_events=n_events, gpu=gpu, sites=int(calls.shape[0]), jobs=2 * int(calls.shape[0]), scored_events=scored,
               kernel_ms_median=float(np.median(kern_ms)), launches=launches, call_ms_median=float(np.median(call_ms)),
               call_ms_min=float(np.min(call_ms)), call_ms_max=float(np.max(call_ms)))
    t = row["call_ms_median"] / 1e3
    row.update(sites_per_s=row["sites"] / t, jobs_per_s=row["jobs"] / t, scored_events_per_s=scored / t)
    if ref_o is not None and n_reads == 512:
        sites, jobs, _, windows = pr.enumerate_batch(ref, pairs, recs, variants, vr, model.k)
        mh = ref_o.builtin_model()
        rh = ref_o.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, mh)
        _, secs = ref_o.score_batch(rh, jobs, windows, [mh], threads=1)
        ref_o.clear_reads()
        row.update(ref_profile_hmm_score_ms_per_read_1thread=secs * 1e3 / n_reads)
    print(json.dumps(row), flush=True)
eng.close()
