"""Timing of the per-site methylation frequency table on the device (nph_methfreq_add / nph_methfreq_tsv) at the bench's
call-methylation shape: synthetic reads aligned to their own sequence, cpg, k = 6, n_reads per batch, several batches on one contig
whose reads start at the same position so keys repeat.  Per batch: the device ms of nph_methylation_run and of the fold after it
(CUDA events on the context's stream); then the ms of the table, its keys and bytes; the table is checked once against
tests/meth_frequency.py (the restatement of calculate_methylation_frequency.py) over the batches' own nph_methylation_tsv rows.
Prints one JSON line (development aid).

  python scripts/quick_methylation_frequency.py [n_batches] [n_reads] [n_events]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from nanopolish_b200.engine import Engine  # noqa: E402
from tests import meth_frequency as mf  # noqa: E402

K = 6
n_batches = int(sys.argv[1]) if len(sys.argv) > 1 else 4
n_reads = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
n_events = int(sys.argv[3]) if len(sys.argv) > 3 else 4000

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
params = synth.meth_params("cpg", K)
eng = Engine(0, stream=torch.cuda.current_stream().cuda_stream)
eng.model_upload(nuc); eng.model_upload(cpg)
batches = []
for b in range(n_batches):
    rs = synth.gen_reads(n_reads, n_events, nuc, seed=31_000 + 1_000_003 * b, cpg_keep=0.3)
    ref, pairs, recs = synth.methylation_records(rs, model_id=1, rc_every=2)
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    batches.append((rs, ref, deltas, first, recs))
names = ["read_%d" % i for i in range(n_reads)]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def load(b):
    rs, ref, deltas, first, recs = batches[b]
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.methylation_load_compact(ref, deltas, first, recs, params)


# warm-up: every kernel and the sort once
load(0); eng.methylation_run(); eng.methylation_frequency_add(0); eng.methylation_frequency_tsv(["chr1"])
eng.methylation_frequency_reset()
run_ms, add_ms, sites, texts = [], [], [], []
for b in range(n_batches):
    load(b)
    run_ms.append(timed(eng.methylation_run))
    add_ms.append(timed(lambda: eng.methylation_frequency_add(0)))
    sites.append(eng.methylation_counts()[0])
    texts.append(mf.CALLS_HEADER + eng.methylation_tsv("chr1", names, batches[b][4]["rc"]).decode())
n_keys, n_calls, n_ambiguous = eng.methylation_frequency_counts()
out = {}
tsv_ms = [timed(lambda: out.setdefault("t", eng.methylation_frequency_tsv(["chr1"]))) for _ in range(3)]
table = out["t"]
t0 = time.perf_counter()
want = mf.frequency_table(texts, 2.0, False)
restatement_s = time.perf_counter() - t0
assert table.decode() == want, "device table differs from the restatement"
eng.close()
print(json.dumps(dict(workload="per-site methylation frequency (calculate_methylation_frequency.py, -c 2.0) folded on the device",
                      card=card, batches=n_batches, reads_per_batch=n_reads, events_per_read=n_events, sites_per_batch=sites,
                      methylation_run_ms=run_ms, methfreq_add_ms=add_ms, methfreq_tsv_ms=tsv_ms, n_keys=n_keys, n_calls=n_calls,
                      n_ambiguous=n_ambiguous, table_bytes=len(table), calls_tsv_bytes=sum(len(t) for t in texts),
                      equals_restatement=True, restatement_python_s=restatement_s)))
