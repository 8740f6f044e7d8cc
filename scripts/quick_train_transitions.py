"""Timing of nph_train_transitions_batch (scorereads --train-transitions) at the benchmark's scorereads shape: 10 000 reads of 4 000
events, 500-event segments, every other read on the reverse strand, the strand as the group.  Reports the jobs, the forward kernel
time (nph_last_kernel_ms of the same batch through nph_hmm_score_batch_seq), the Viterbi time (K3 and its state-offset kernel) and
the observation kernel time (nph_tt_params' viterbi_ms_out and observe_ms_out), the whole training call and the same call without training, each the
median of several calls after a warm-up; the card's name, power limit and SM clock read in the same run; and — where
oracle/_ref/libnpref_scorereads.so is built — the compiled reference's model_score with training on one CPU thread over a few
reads, per segment.  Prints one JSON line.

  python scripts/quick_train_transitions.py [reps] [n_reads]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from nanopolish_b200.engine import Engine  # noqa: E402
from tests import tt_cases as tc  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
n_reads = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
model = synth.load_model("nucleotide")
rs = synth.gen_reads(n_reads, 4000, model, seed=5)
jb = synth.scorereads_jobs(rs, 500, rc_every=2)
groups = (jb.code_jobs["rc"] != 0).astype(np.uint8)
eng = Engine(0)
eng.model_upload(model)
train = lambda: eng.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jb.seq_codes, jb.code_jobs, groups)
plain = lambda: eng.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, jb.seq_codes, jb.code_jobs)
s_train, counts, chunks = train()                                # warm-up: module load, buffers
s_plain = plain()
assert np.array_equal(s_train.view(np.uint32), s_plain.view(np.uint32))
t_train, t_plain, k_train, k_fwd, k_vit, k_obs = [], [], [], [], [], []
for _ in range(reps):
    t0 = time.perf_counter(); train(); t_train.append((time.perf_counter() - t0) * 1e3); k_train.append(eng.last_kernel_ms()[0])
    k_vit.append(eng.last_tt_ms[0]); k_obs.append(eng.last_tt_ms[1])
    t0 = time.perf_counter(); plain(); t_plain.append((time.perf_counter() - t0) * 1e3); k_fwd.append(eng.last_kernel_ms()[0])
med = lambda v: float(np.median(v))
row = dict(reads=n_reads, events_per_read=4000, jobs=int(jb.code_jobs.shape[0]), dp_rows=int(jb.scored_events), chunks=chunks, gpu=gpu,
           forward_kernel_ms_median=med(k_fwd), viterbi_ms_median=med(k_vit), observe_ms_median=med(k_obs),
           train_kernel_ms_median=med(k_train), train_call_ms_median=med(t_train), score_call_ms_median=med(t_plain),
           train_call_ms_min=float(np.min(t_train)), train_call_ms_max=float(np.max(t_train)),
           skip_observations=[int(counts[g]["skip_total"].sum()) for g in range(2)])
if tc.RefTT.available():
    ref = tc.RefTT()
    ref.lib.npref_set_globals(C.c_double(1.0), 1)
    segs, secs = 0, 0.0
    for seed in range(3):
        c = tc.build(("bench", 4000, 500, 100 + seed, 0, False, None, False, "truth"))
        t0 = time.perf_counter()
        ref.model_score(c)
        secs += time.perf_counter() - t0
        segs += len(tc.jobs_of(c)[2])
    row.update(ref_segments=segs, ref_model_score_train_ms_per_segment_1thread=secs * 1e3 / segs)
print(json.dumps(row), flush=True)
eng.close()
