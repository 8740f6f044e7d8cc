"""Parity of the CUDA adaptive-banded event aligner (through the C ABI) with the oracle and with the
compiled reference's recorded output: identical AlignedPair lists and identical QC verdicts."""
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.golden_cases import make_abea_cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


def _compare(rs, jobs, pairs_g, res_g, pairs_o, res_o):
    """every field of every record (avg_log_emission by its bits: same FP64 summation order), and the pairs"""
    assert [int(x) for x in res_g["n_pairs"]] == [int(x) for x in res_o["n_pairs"]]
    for i in range(jobs.shape[0]):
        for f in ("status", "max_gap", "n_aligned"):
            assert int(res_g[i][f]) == int(res_o[i][f]), f"read {i}: {f} {int(res_g[i][f])} vs {int(res_o[i][f])}"
        assert res_g[i:i + 1]["avg_log_emission"].tobytes() == res_o[i:i + 1]["avg_log_emission"].tobytes(), f"read {i}: avg_log_emission"
        n = int(res_o[i]["n_pairs"])
        o = int(jobs[i]["pairs_off"])
        assert np.array_equal(pairs_g[o:o + n], pairs_o[o:o + n]), f"read {i}: paths differ"


@pytest.mark.parametrize("name", ["reads_2k", "reads_short"])
def test_golden_alignments(engine, nuc, port_oracle, name):
    model, mid = nuc
    rs = make_abea_cases()[name]["rs"]
    jobs, ranks, total = synth.abea_jobs(rs)
    pairs, res = engine.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, mid, total)
    z = np.load(os.path.join(GOLD, "abea_golden.npz"))
    gp, gn = z[name + "_pairs"], z[name + "_npairs"]
    assert [int(x) for x in gn] == [int(x) for x in res["n_pairs"]]
    o = 0
    for i in range(rs.n_reads):
        n = int(gn[i])
        b = pairs[int(jobs[i]["pairs_off"]):int(jobs[i]["pairs_off"]) + n]
        assert np.array_equal(gp[o:o + n, 0], b["ref_pos"]) and np.array_equal(gp[o:o + n, 1], b["read_pos"])
        o += n
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, jobs, total)
    _compare(rs, jobs, pairs, res, po, ro)


@pytest.mark.parametrize("n_events,n_reads,scaled", [(60, 12, False), (900, 10, True), (4000, 6, False), (8000, 3, True)])
def test_random_reads_identical_paths(engine, nuc, port_oracle, n_events, n_reads, scaled):
    model, mid = nuc
    rs = synth.gen_reads(n_reads, n_events, model, seed=7000 + n_events, rng_scalings=scaled)
    jobs, ranks, total = synth.abea_jobs(rs)
    pairs, res = engine.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, mid, total)
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, jobs, total, threads=8)
    assert (res["n_pairs"] > 0).all()
    _compare(rs, jobs, pairs, res, po, ro)


def test_qc_failures_and_mixed_batch(engine, nuc, port_oracle):
    """Unrelated events fail QC (empty result); reads of very different length share one batch."""
    model, mid = nuc
    rs = synth.gen_reads(6, 500, model, seed=99, rng_scalings=False)
    rng = np.random.default_rng(1)
    o, n = int(rs.reads[1]["event_off"]), int(rs.reads[1]["n_events"])
    rs.ev_mean[o:o + n] = rng.uniform(60, 120, n).astype(np.float32)          # read 1: noise
    o, n = int(rs.reads[4]["event_off"]), int(rs.reads[4]["n_events"])
    rs.ev_mean[o + 100:o + 300] = rs.ev_mean[o + 100]                          # read 4: a long stall
    jobs, ranks, total = synth.abea_jobs(rs)
    pairs, res = engine.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, mid, total)
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, jobs, total)
    assert int(ro[1]["n_pairs"]) == 0
    _compare(rs, jobs, pairs, res, po, ro)


def test_truncated_sequence_and_event_ranges(engine, nuc, port_oracle):
    """Sequence shorter / longer than the events imply (band hits the matrix edges)."""
    model, mid = nuc
    rs = synth.gen_reads(4, 700, model, seed=123, rng_scalings=False)
    jobs, ranks, total = synth.abea_jobs(rs)
    jobs = jobs.copy()
    jobs[0]["n_kmers"] = jobs[0]["n_kmers"] // 2          # half the sequence
    jobs[1]["n_kmers"] = 3                                 # tiny
    pairs, res = engine.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, mid, total)
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, jobs, total)
    _compare(rs, jobs, pairs, res, po, ro)


def test_mom_scalings(engine, nuc, port_oracle):
    model, mid = nuc
    rs = synth.gen_reads(5, 1500, model, seed=77)
    jobs, ranks, _ = synth.abea_jobs(rs)
    got = engine.mom_batch(rs.reads, rs.ev_mean, ranks, jobs, mid)
    for i in range(rs.n_reads):
        sh, sc = port_oracle.mom(rs.reads, rs.ev_mean, model, ranks, jobs[i])
        assert got[i, 0] == sh and got[i, 1] == sc


def test_staged_abea_timing(engine, nuc):
    model, mid = nuc
    rs = synth.gen_reads(64, 2000, model, seed=5150, rng_scalings=False)
    jobs, ranks, total = synth.abea_jobs(rs)
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    engine.abea_jobs_load(ranks, jobs, mid, total)
    engine.abea_run()
    pairs, res = engine.abea_fetch()
    assert (res["n_pairs"] > 1900).all()
    ms, launches = engine.last_kernel_ms()
    assert ms > 0 and launches == 1


def test_full_size_properties(engine, nuc, port_oracle):
    """BASELINE config 4 shape (8 000-event reads) on a few thousand reads: every read aligns, pairs are sorted
    and in range, a random sample equals the oracle's path exactly, and a second run is identical."""
    model, mid = nuc
    rs = synth.gen_reads(2400, 8000, model, seed=31337, rng_scalings=False)
    jobs, ranks, total = synth.abea_jobs(rs)
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    engine.abea_jobs_load(ranks, jobs, mid, total)
    engine.abea_run(); p1, r1 = engine.abea_fetch()
    engine.abea_run(); p2, r2 = engine.abea_fetch()
    assert np.array_equal(r1["n_pairs"], r2["n_pairs"]) and (r1["n_pairs"] >= 8000).all()
    for i in range(0, rs.n_reads, 97):
        o, n = int(jobs[i]["pairs_off"]), int(r1[i]["n_pairs"])
        a = p1[o:o + n]
        assert np.array_equal(a, p2[o:o + n])
        assert a["ref_pos"][0] == 0 and a["ref_pos"][-1] == int(jobs[i]["n_kmers"]) - 1
        assert (np.diff(a["ref_pos"]) >= 0).all() and (np.diff(a["read_pos"]) >= 0).all()
        assert (np.diff(a["ref_pos"]) + np.diff(a["read_pos"]) >= 1).all()
    sample = np.array([0, 5, 777, 1234, 2399])
    sj = jobs[sample].copy()
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, sj, total, threads=8)
    for t, i in enumerate(sample):
        o, n = int(jobs[i]["pairs_off"]), int(ro[t]["n_pairs"])
        assert n == int(r1[i]["n_pairs"]) and np.array_equal(p1[o:o + n], po[o:o + n])
