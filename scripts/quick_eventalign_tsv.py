"""eventalign.tsv: rows formatted on the host against rows written on the device, on one GPU.

Two arms per batch shape and switch set, alternated, after a warm-up of each:
  (a) EventAligner::run (nph_eventalign_chain, records back, scatter) + tsv_batch (the OpenMP host writer);
  (b) EventAligner::run_tsv (nph_eventalign_chain_run + nph_eventalign_tsv into page-locked staging).
Both build the same chains on the host and end in a synchronise; the bytes of the two arms are compared before anything is timed.
Then, through the C ABI alone, the device time of the chain kernel and of the writer's passes (nph_last_kernel_ms), the rows and
bytes written, the writer's bytes per second, and the device-to-host copy of the text.  Fails without a GPU.

    python scripts/quick_eventalign_tsv.py [--shapes 10000x4000,512x4000] [--repeats 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nanopolish_b200 import synth                                  # noqa: E402
from nanopolish_b200.engine import Engine                          # noqa: E402
from tests import host_mirror as hm                                # noqa: E402

SWITCH_SETS = [("none", 0), ("--signal-index --scale-events", 2 | 4), ("--samples", 8)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def spread(xs):
    return {"median_ms": float(np.median(xs)), "min_ms": float(np.min(xs)), "max_ms": float(np.max(xs))}


def host_arms(host, model, rs, inp, switches, repeats):
    """wall time of the two EventAligner paths; returns (a, b, bytes)"""
    host.nphh_clear()
    rh = hm.register_reads(host, rs, hm.register_model(host, model))
    seqs = []
    for i, (r, h) in enumerate(zip(rs.reads, rh)):
        o, n = int(r["event_off"]), int(r["n_events"])
        seq = synth._CODE2DNA[rs.seq_codes[i]].tobytes()
        nk = len(seq) - model.k + 1
        start, stop, _ = synth.closest_event_map(rs.ev_kmer[i], nk)
        a, b = np.ascontiguousarray(start, np.int32), np.ascontiguousarray(stop, np.int32)
        tr = inp["reads"][i]
        stdv, dur = np.ascontiguousarray(inp["ev_stdv"][o:o + n]), np.ascontiguousarray(inp["ev_duration"][o:o + n])
        assert host.nphh_read_set_eventalign(h, f"read_{i}".encode(), seq, hm.p(a), hm.p(b), C.c_size_t(nk), hm.p(stdv), hm.p(dur)) == 0
        if inp["samples"] is not None:
            # the host mirror's sample clock starts at 0: shift the read's samples to where its events index them
            first = int(tr["sample_start_time"])
            smp = np.zeros(first + int(tr["n_samples"]), np.float32)
            smp[first:] = inp["samples"][int(tr["sample_off"]):int(tr["sample_off"]) + int(tr["n_samples"])]
            assert host.nphh_read_set_samples(h, hm.p(smp), C.c_size_t(smp.shape[0]), C.c_double(4000.0)) == 0
        elif switches & 4:
            one = np.zeros(1, np.float32)                            # --signal-index wants samples on the read and reads none
            assert host.nphh_read_set_samples(h, hm.p(one), C.c_size_t(1), C.c_double(4000.0)) == 0
        seqs.append(seq)

    def queue():
        host.nphh_ea_begin()
        for i, seq in enumerate(seqs):
            cigar = np.array([(len(seq) << 4) | 0], np.uint32)
            assert host.nphh_ea_add_read(rh[i], b"chr_synth", 0, 0, 60, hm.p(cigar), 1, seq, i, -1, -1) == i, host.nphh_last_error()

    def arm_a(out=None, cap=0):
        queue()
        t0 = time.perf_counter()
        assert host.nphh_ea_run(C.c_double(1.0)) >= 0, host.nphh_last_error()
        n = host.nphh_ea_tsv_all_opt(switches, out, C.c_size_t(cap), None)
        dt = time.perf_counter() - t0
        assert n >= 0, host.nphh_last_error()
        return dt * 1e3, n

    def arm_b(out=None, cap=0):
        queue()
        t0 = time.perf_counter()
        n = host.nphh_ea_run_tsv(C.c_double(1.0), switches, out, C.c_size_t(cap), None, None, None)
        dt = time.perf_counter() - t0
        assert n >= 0, host.nphh_last_error()
        return dt * 1e3, n

    # equal bytes first (this is also each arm's warm-up)
    _, n = arm_a()
    ba, bb = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    assert arm_a(hm.p(ba), n)[1] == n and arm_b(hm.p(bb), n)[1] == n
    assert np.array_equal(ba, bb), "the device's bytes differ from the host writer's"
    del ba, bb
    ta, tb = [], []
    for _ in range(repeats):
        ta.append(arm_a()[0]); tb.append(arm_b()[0])
    host.nphh_ea_begin()
    return spread(ta), spread(tb), int(n)


def abi_numbers(eng, model, rs, inp, switches, repeats):
    """device time of the chain kernel and of the writer, bytes, copy time, through the C ABI"""
    mid = eng.model_upload(model)
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    pairs, maps, rf, rr, chains = synth.eventalign_chains(rs, mid)
    kw = dict(scale_events=bool(switches & 2), signal_index=bool(switches & 4), samples=bool(switches & 8))
    results = eng.eventalign_chain_run(pairs, maps, rf, rr, chains)
    chain_ms = [eng.last_kernel_ms()[0]]
    text, read_off, refused, _ = eng.eventalign_tsv(inp, **kw)
    assert not refused.any()
    nbytes, rows = len(text), int(results["n_records"].sum())
    del text
    out = np.empty(nbytes, np.uint8)          # pageable here; run_tsv (arm b) copies into the engine's page-locked staging
    writer_ms, call_ms = [], []
    for _ in range(repeats):
        eng.eventalign_chain_run(pairs, maps, rf, rr, chains)
        chain_ms.append(eng.last_kernel_ms()[0])
        t0 = time.perf_counter()
        eng.eventalign_tsv(inp, out=out, **kw)
        call_ms.append((time.perf_counter() - t0) * 1e3)
        writer_ms.append(eng.last_kernel_ms()[0])
    w = float(np.median(writer_ms))
    return {"rows": rows, "bytes": nbytes, "chain_kernel": spread(chain_ms[1:]), "writer_passes": spread(writer_ms),
            "writer_call_incl_uploads_and_copy": spread(call_ms), "writer_GB_per_s_of_text": nbytes / (w * 1e-3) / 1e9,
            "copy_and_upload_ms_median": float(np.median(call_ms)) - w}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="10000x4000,512x4000")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-host-arms", action="store_true", help="only the C ABI numbers")
    args = ap.parse_args()
    eng = Engine(0)                                                  # raises without a GPU
    print(json.dumps({"card_and_power_limit": card()}))
    host = hm.load()
    model = synth.load_model("nucleotide")
    for shape in args.shapes.split(","):
        n_reads, n_events = (int(v) for v in shape.split("x"))
        rs = synth.gen_reads(n_reads, n_events, model, seed=5, drift=True)
        for name, switches in SWITCH_SETS:
            inp = synth.eventalign_tsv_inputs(rs, seed=6, with_samples=bool(switches & 8))
            res = {"shape": shape, "switches": name}
            res.update(abi_numbers(eng, model, rs, inp, switches, args.repeats))
            if switches & 8 and n_reads > 1024:
                # the host mirror indexes a read's samples from the start of its file: ten thousand such reads do not fit host memory
                res["host_arms"] = "not run at this shape"
            elif not args.skip_host_arms:
                a, b, n = host_arms(host, model, rs, inp, switches, args.repeats)
                res.update({"arm_a_run_plus_tsv_batch": a, "arm_b_run_tsv": b, "arm_bytes": n})
            print(json.dumps(res), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
