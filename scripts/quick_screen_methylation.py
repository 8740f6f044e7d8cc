#!/usr/bin/env python
"""Methylation-aware candidate screening (`variants -q ...`) on one GPU at the bench's variants shape: 200 000 positions, 50x coverage by
2 300-base reads, on a draft with planted recognition sites (synth.gen_pileup_methylated).  Three arms over the same pile-up: no
types, -q cpg, -q dam,dcm.  Per arm: ms per nph_screen_run (CUDA events, after warm-up, several runs), rounds, jobs, DP rows, the
reference-unit rows per second, and the jobs added relative to the no-types arm.  A sample of positions per arm is checked against
the compiled reference's score_variant_thresholded (oracle/_ref/libnpref_types.so, when built), with the reference's CPU time for that sample.
Prints the card's name and power limit.  Usage: python scripts/quick_screen_methylation.py [--positions N] [--runs R]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nanopolish_b200 import synth  # noqa: E402
from nanopolish_b200.engine import Engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--positions", type=int, default=200_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sample", type=int, default=8)
    a = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {smi.splitlines()[0] if smi else torch.cuda.get_device_name(0)}")
    region = 1_000_000
    nuc = synth.load_model("nucleotide")
    tm = {t: synth.load_model(t) for t in ("cpg", "dam", "dcm")}
    t0 = time.time()
    ref, rs, recs, pairs = synth.gen_pileup_methylated(a.positions + 1, 50, 2300, nuc, ["cpg", "dam", "dcm"], tm, seed=424_243, region_start=region,
                                                       n_true_variants=max(1, a.positions // 2000), methylated_fraction=0.5, site_spacing=40)
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    ref_chars = synth._CODE2DNA[ref]
    params = synth.screen_params(region, 6, 10, 100, 3, 8)
    print(f"pile-up: {a.positions} positions, {recs.shape[0]} reads, {rs.total_events} events (generated in {time.time() - t0:.0f} s)")
    eng = Engine(0, stream=torch.cuda.current_stream().cuda_stream)
    ids = {"nucleotide": eng.model_upload(nuc)}
    for t, m in tm.items():
        ids[t] = eng.model_upload(m)
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    ref_live = None
    try:
        from tests.ref_types import RefTypesOracle
        if RefTypesOracle.available():
            ref_live = RefTypesOracle()
            rh = ref_live.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time)
    except OSError:
        ref_live = None
    base_jobs = None
    lists = None
    for types in ([], ["cpg"], ["dam", "dcm"]):
        meth = (synth.screen_methylation(types), np.array([[ids[t] for t in types]] * recs.shape[0], np.uint32).reshape(recs.shape[0], len(types)))
        eng.screen_load(ref_chars, deltas, first, recs, params, 0.9, methylation=meth)
        for _ in range(2):
            eng.screen_run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.screen_run()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        q, nr = eng.screen_fetch()
        c = eng.screen_counts()
        base_jobs = c["jobs"] if base_jobs is None else base_jobs
        med = float(np.median(ms))
        name = ",".join(types) or "none"
        print(f"-q {name:8s}: {med:9.2f} ms per nph_screen_run (median of {a.runs}, min {min(ms):.2f}), rounds {c['rounds']}, jobs {c['jobs']} "
              f"({100.0 * (c['jobs'] / base_jobs - 1):+.1f}% vs no types), DP rows {c['scored_events']}, reference rows {c['reference_events']} "
              f"= {c['reference_events'] / (med * 1e-3):.3e} rows/s, jobs without early exit {c['jobs_without_exit']}")
        if ref_live is None:
            print("   compiled reference: not built here, sample not checked")
            continue
        ref_s = ref_chars.tobytes().decode()
        from tests import var_restatement as vr
        lists = lists if lists is not None else vr.pair_lists(recs, pairs)
        rng = np.random.default_rng(len(types))
        sample = sorted(rng.choice(np.arange(20, a.positions - 20), a.sample, replace=False).tolist())
        cpu_s, bad = 0.0, 0
        for pi in sample:
            i = region + pi
            cs, ce = i - 10, i + 11
            seqs = vr.event_sequences(recs, pairs, cs, ce, lists)
            cands = vr.candidates(ref_s, pi)
            t1 = time.perf_counter()
            v = ref_live.score_variants_thresholded([rh[r] for r, _, _ in seqs], [(e1, e2) for _, e1, e2 in seqs],
                                                          np.array([recs[r]["rc"] for r, _, _ in seqs], np.uint8), ref_s[cs - region:ce - region + 1], cs,
                                                          [(region + off, rs_, as_) for _, off, rs_, as_ in cands], 3, 100, types, indel_bias=0.9)
            cpu_s += time.perf_counter() - t1
            bad += sum(np.float64(q[pi, slot]).tobytes() != np.float64(x).tobytes() for (slot, _, _, _), x in zip(cands, v))
        print(f"   compiled reference on {len(sample)} sampled positions: {bad} qualities differ, {cpu_s * 1e3:.1f} ms single-thread CPU")
    eng.close()


if __name__ == "__main__":
    main()
