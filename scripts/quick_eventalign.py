"""Timing of eventalign's segment chaining through the C++ host (EventAligner::run: one Viterbi launch per round)
next to the compiled reference's align_read_to_ref on the host cores (development aid; prints one JSON line).

  python scripts/quick_eventalign.py [n_reads] [n_events] [n_reference_reads]
"""
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from oracle import eventalign_py as EP  # noqa: E402
from tests import eventalign_cases as EC  # noqa: E402
from tests import host_mirror as hm  # noqa: E402

n_reads = int(sys.argv[1]) if len(sys.argv) > 1 else 256
n_events = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
n_ref = int(sys.argv[3]) if len(sys.argv) > 3 else 32

model, rs, cases = EC.build_cases(n_reads, n_events, seed=91)
cases = cases[:n_reads]                                   # without the unmapped / windowed extras
host = hm.load()
p = hm.p
mh = hm.register_model(host, model)
rh = hm.register_reads(host, rs, mh)


def setup():
    host.nphh_ea_begin()
    for c in cases:
        r = c["read"]
        slot = EC.read_slot(c, rs.n_reads)
        a, b = np.ascontiguousarray(r.b2e_start, np.int32), np.ascontiguousarray(c["b2e_stop"], np.int32)
        host.nphh_read_set_eventalign(rh[slot], r.name.encode(), r.read_sequence.encode(), p(a), p(b), C.c_size_t(a.shape[0]),
                                      p(np.ascontiguousarray(r.stdv)), p(np.ascontiguousarray(r.duration)))
        assert host.nphh_ea_add_read(rh[slot], c["contig_name"].encode(), c["ref_pos"], c["flag"], c["mapq"], p(c["cigar"]),
                                     int(c["cigar"].shape[0]), c["fetched"].encode(), c["read_idx"], -1, -1) == c["read_idx"]


total_events = int(rs.reads["n_events"].sum())
best = {}
rounds = {}
for mode, fn in (("chain", host.nphh_ea_run), ("host_rounds", host.nphh_ea_run_rounds)):
    for it in range(3):
        setup()
        t0 = time.perf_counter()
        r = fn(C.c_double(1.0))
        dt = time.perf_counter() - t0
        assert r >= 0, host.nphh_last_error()
        rounds[mode] = int(r)
        best[mode] = dt if mode not in best else min(best[mode], dt)
        print(f"{mode} run {it}: {r} batches, {dt * 1e3:.1f} ms, {total_events / dt:.3e} events/s, {n_reads / dt:.0f} reads/s", file=sys.stderr)
setup()
host.nphh_ea_run(C.c_double(1.0))
t0 = time.perf_counter()
n = host.nphh_ea_tsv_all(None, C.c_size_t(0))               # every read's rows, formatted in parallel (size only)
t_tsv = time.perf_counter() - t0
assert n >= 0, host.nphh_last_error()
buf = C.create_string_buffer(1 << 24)
texts = []
rows = 0
for c in cases[:n_ref]:
    m = host.nphh_ea_text(c["read_idx"], 0, buf, C.c_size_t(1 << 24))
    texts.append(buf.raw[:m].decode()); rows += texts[-1].count("\n")
segs = sum(host.nphh_ea_num_segments(c["read_idx"]) for c in cases)

# the compiled reference on the host cores (single thread per read, as its OpenMP loop runs them), a bounded sample
ref = None
try:
    from oracle.oracle_py import RefOracle
    if RefOracle.available():
        ro = RefOracle()
        mhr = ro.builtin_model("nucleotide")
        rhr = ro.register_reads(rs.reads[:n_ref], rs.ev_mean, rs.ev_start_time, mhr)
        t_ref, same = 0.0, True
        for c in cases[:n_ref]:
            r, slot = c["read"], EC.read_slot(c, rs.n_reads)
            ro.read_set_eventalign(rhr[slot], r.name, r.read_sequence, r.b2e_start, c["b2e_stop"], r.stdv, r.duration)
            t0 = time.perf_counter()
            tsv, _, _ = ro.eventalign(rhr[slot], c["contig_name"], c["contig"], c["ref_pos"], c["flag"], c["cigar"], c["read_idx"],
                                      want_cigar=False)
            t_ref += time.perf_counter() - t0
            same = same and tsv == texts[c["read_idx"]]
        ev_ref = int(rs.reads["n_events"][:n_ref].sum())
        ref = dict(reads=n_ref, seconds=t_ref, events_per_sec_1_thread=ev_ref / t_ref, tsv_identical=bool(same))
except OSError as e:
    ref = dict(error=str(e))
print(json.dumps(dict(workload="eventalign chaining", reads=n_reads, events=total_events, windows=int(segs),
                      chain=dict(batches=rounds["chain"], best_ms=best["chain"] * 1e3, events_per_sec=total_events / best["chain"],
                                 reads_per_sec=n_reads / best["chain"]),
                      host_rounds=dict(rounds=rounds["host_rounds"], best_ms=best["host_rounds"] * 1e3,
                                       events_per_sec=total_events / best["host_rounds"]),
                      tsv_bytes=int(n), tsv_format_ms=t_tsv * 1e3, reference=ref)))
