"""Timing of nph_polya_batch, or with --polyi of nph_detect_polyi_batch (development aid): samples/s and ms per batch at 512 and
10 000 direct-RNA-like reads, and the compiled reference's per-read work on one CPU thread for the same kind of reads
(segment_squiggle + read rate; with --polyi the segmentation + read rate + Bernoulli stage).  With --polyi the reads have
poly(I)/poly(A) tails, and nph_polya_batch runs on the same batches in the same run, alternating with it: the polya kernel is
the other instantiation of the same template and its time should not move.

Reads are ~10^5 samples (a 1.5 kb RNA read), log-uniform in [4*10^4, 2.5*10^5].  Signals are generated for a pool of 64
reads (numpy generation is the slow part) and each batch copies its picks into a raw array of the batch's full size, so the
call time includes uploading every sample of the batch."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from nanopolish_b200.engine import Engine
from tests import polya_cases as pc
from tests import polyi_cases as qc


def batch(pool_raw, pool_jobs, n, rng):
    """n reads drawn from the pool, each with its own copy of its samples in one raw array"""
    js = pool_jobs[rng.integers(0, pool_jobs.shape[0], n)].copy()
    lens = js["n_samples"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    raw = np.empty(int(lens.sum()), np.float32)
    for o, j in zip(off, js):
        raw[o:o + int(j["n_samples"])] = pool_raw[int(j["sample_off"]):int(j["sample_off"]) + int(j["n_samples"])]
    js["sample_off"] = off
    return raw, js


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--polyi", action="store_true", help="time nph_detect_polyi_batch, alternating with nph_polya_batch")
    polyi = ap.parse_args().polyi
    rng = np.random.default_rng(5)
    lens = np.exp(rng.uniform(np.log(4e4), np.log(2.5e5), 64)).astype(np.int64)
    synth_read = qc.synth_polyi_read if polyi else pc.synth_read
    pool = [synth_read(rng, f"p{i}", int(n), n_kmers=int(n) // 70) for i, n in enumerate(lens)]
    raw, jobs, dur, b2e = pc.pack(pool)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        gpu = "unknown"
    print(f"gpu: {gpu}")
    eng = Engine(0)
    calls = {"detect-polyi": eng.detect_polyi_batch, "polya": eng.polya_batch} if polyi else {"polya": eng.polya_batch}
    for n in (512, 10000):
        braw, js = batch(raw, jobs, n, rng)
        n_samples = int(js["n_samples"].astype(np.int64).sum())
        assert braw.shape[0] == n_samples
        ks = {k: [] for k in calls}
        es = {k: [] for k in calls}
        for f in calls.values():
            f(braw, js, dur, b2e)                                # warm-up
        for _ in range(5 if polyi else 3):
            for name, f in calls.items():
                t = time.perf_counter()
                f(braw, js, dur, b2e)
                es[name].append((time.perf_counter() - t) * 1e3)
                ks[name].append(eng.last_kernel_ms()[0])
        for name in calls:
            k = float(np.median(ks[name])); e = float(np.median(es[name]))
            print(f"{name} {n} reads, {n_samples:.3e} samples: kernel {k:.2f} ms ({n_samples / k * 1e3:.3e} samples/s), "
                  f"call {e:.2f} ms (uploading all {braw.nbytes / 1e9:.2f} GB of samples from pageable memory), "
                  f"kernel runs {['%.2f' % x for x in ks[name]]}")
    eng.close()
    path, ref_class, work = ((qc.REF_POLYI, qc.RefPolyi, "segmentation + read rate + Bernoulli stage") if polyi else
                             (pc.REF_POLYA, pc.RefPolya, "segment_squiggle + read rate"))
    if os.path.exists(path):
        ref = ref_class()
        t = [ref.time(r) for r in pool[:16]]
        s = sum(int(r.samples.shape[0]) for r in pool[:16])
        print(f"reference {work}, one CPU thread: {np.mean(t) * 1e3:.2f} ms per read "
              f"(mean {s / 16:.0f} samples), {s / sum(t):.3e} samples/s")
    else:
        print(f"reference: {os.path.relpath(path, pc.ROOT)} not built")


if __name__ == "__main__":
    main()
