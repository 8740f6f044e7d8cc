"""Timing of call-methylation through the C++ host's object API (MethylationCaller: stage host buffers -> one device call
(enumeration + scoring) -> TSV); caller_ms excludes the test shim's marshalling of the flat test arrays into EventAlignedRead objects
next to the compiled reference scoring the same windows on the host cores (development aid; prints one JSON line).

  python scripts/quick_methylation.py [n_reads] [n_events]
"""
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from tests import host_mirror as hm  # noqa: E402

K = 6
n_reads = int(sys.argv[1]) if len(sys.argv) > 1 else 512
n_events = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
host = hm.load()
nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
rs = synth.gen_reads(n_reads, n_events, nuc, seed=2024, cpg_keep=0.3)
mh, ch = hm.register_model(host, nuc), hm.register_model(host, cpg)
rh = hm.register_reads(host, rs, mh)
for r in rh:
    host.nphh_read_add_model(r, b"cpg", ch)
refs_s, pairs_l = [], []
for i in range(n_reads):
    codes = rs.seq_codes[i]
    nk = codes.shape[0] - K + 1
    kfe = np.minimum(rs.kmer_first_event[i], int(rs.reads[i]["n_events"]) - 1)
    refs_s.append(synth._CODE2DNA[codes].tobytes())
    pairs_l.append(np.stack([10_000 + np.arange(K, nk - K), kfe[K:nk - K]], 1).astype(np.int32))
flat = np.concatenate(pairs_l).reshape(-1)
off = np.zeros(n_reads + 1, np.uint64); off[1:] = np.cumsum([p.shape[0] for p in pairs_l])
names = (C.c_char_p * n_reads)(*[f"read_{i}".encode() for i in range(n_reads)])
refs = (C.c_char_p * n_reads)(*refs_s)
p = hm.p
z = np.zeros(n_reads, np.uint8)
cap = 400 * 45 * n_reads
buf = C.create_string_buffer(cap)
best, stages, nj = None, None, C.c_uint64()
for it in range(4):
    secs3 = np.zeros(4)
    t0 = time.perf_counter()
    n = host.nphh_call_methylation_timed(n_reads, p(np.array(rh, np.int32)), names, p(z), p(z), p(np.full(n_reads, 10_000, np.int32)), refs,
                                         p(flat), p(off), b"chr1", C.c_double(1.0), buf, C.c_size_t(cap), C.byref(nj), p(secs3))
    dt = time.perf_counter() - t0
    assert n >= 0, host.nphh_last_error()
    print(f"run {it}: {dt * 1e3:.1f} ms  shim marshalling {secs3[3] * 1e3:.1f}  stage {secs3[0] * 1e3:.1f}  flatten+device {secs3[1] * 1e3:.1f}  tsv {secs3[2] * 1e3:.1f}", file=sys.stderr)
    if it and (best is None or dt < best):
        best, stages = dt, secs3.copy()
rows = buf.value.count(b"\n")
# the scored-event count of exactly this batch: the same reference / event alignments through the C ABI (nph_methylation_batch), whose
# enumeration is pinned to the compiled calculate_methylation_for_read; its job count must equal the C++ host's
from nanopolish_b200.engine import Engine
recs = np.zeros(n_reads, synth.METH_RECORD_DT)
ref_all = np.frombuffer(b"".join(refs_s), np.uint8)
ro_ = po_ = 0
for i in range(n_reads):
    recs[i]["ref_off"], recs[i]["pair_off"], recs[i]["read"], recs[i]["model_id"] = ro_, po_, i, 1
    recs[i]["ref_len"], recs[i]["n_pairs"], recs[i]["ref_start_pos"] = len(refs_s[i]), pairs_l[i].shape[0], 10_000
    ro_ += len(refs_s[i]); po_ += pairs_l[i].shape[0]
pairs_all = np.zeros(po_, synth.PAIR_DT)
pairs_all["ref_pos"] = flat.reshape(-1, 2)[:, 0]; pairs_all["read_pos"] = flat.reshape(-1, 2)[:, 1]
eng = Engine(0); eng.model_upload(nuc); eng.model_upload(cpg)
_, sites_dev, scored_exact = eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref_all, pairs_all, recs, synth.meth_params("cpg", K))
eng.close()
assert 2 * sites_dev.shape[0] == int(nj.value) and sites_dev.shape[0] == rows, (sites_dev.shape[0], int(nj.value), rows)
jobs = synth.methylation_jobs(rs, model_id=1, keep_seqs=True)   # windows of the same shape for the CPU arm's sample (a rate, not this job list)
ref = None
try:
    from oracle.oracle_py import RefOracle
    if RefOracle.available():
        ro = RefOracle()
        mhs = [ro.builtin_model("nucleotide"), ro.builtin_model("cpg")]
        nsub = min(n_reads, 256)
        rhr = ro.register_reads(rs.reads[:nsub], rs.ev_mean, rs.ev_start_time, mhs[0])
        sel = np.flatnonzero(jobs.jobs["read"] < nsub)[:40000]
        sub = np.ascontiguousarray(jobs.jobs[sel])
        seqs = [jobs.seqs[j] for j in sel] if jobs.seqs else None
        if seqs is not None:
            cores = os.cpu_count() or 1
            _, secs = ro.score_batch(rhr, sub, seqs, mhs, threads=cores)
            E = np.abs(sub["event_stop"].astype(np.int64) - sub["event_start"].astype(np.int64)) + 1
            ref = dict(jobs=int(sel.shape[0]), seconds=secs, threads=cores, events_per_sec=float(E.sum() / secs))
except OSError as e:
    ref = dict(error=str(e))
print(json.dumps(dict(workload="call-methylation through the C++ host", reads=n_reads, jobs=int(nj.value), tsv_rows=rows,
                      scored_events=int(scored_exact), best_ms=best * 1e3, events_per_sec=scored_exact / best,
                      reads_per_sec=n_reads / best,
                      caller_ms=float((stages[0] + stages[1] + stages[2]) * 1e3), events_per_sec_caller=scored_exact / float(stages[0] + stages[1] + stages[2]),
                      stage_ms=dict(stage_host_buffers=stages[0] * 1e3, flatten_and_device=stages[1] * 1e3, tsv=stages[2] * 1e3,
                                    test_shim_marshalling=stages[3] * 1e3, unaccounted=(best - stages.sum()) * 1e3),
                      jobs_equal_device_enumeration=True, reference=ref)))
