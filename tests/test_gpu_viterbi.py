"""Parity of the CUDA Viterbi aligner (profile_hmm_align through the C ABI) with the oracle, which
tests/test_oracle_vs_ref.py pins to the compiled reference: identical state paths, bit-identical l_fm."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.random_cases import random_hmm_jobs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


def _compare(got, want_list):
    for j, (g, (w, status)) in enumerate(zip(got, want_list)):
        if status != 0:
            assert g.shape[0] == 0, f"job {j}: reference asserts, GPU returned {g.shape[0]} states"
            continue
        assert g.shape[0] == w.shape[0], f"job {j}: {g.shape[0]} vs {w.shape[0]} states"
        assert np.array_equal(g["event_idx"], w["event_idx"]) and np.array_equal(g["kmer_idx"], w["kmer_idx"]), f"job {j}: path"
        assert g["state"].tobytes() == w["state"].tobytes(), f"job {j}: states"
        assert np.array_equal(g["l_fm"].view(np.uint32), w["l_fm"].view(np.uint32)), f"job {j}: l_fm"


def test_eventalign_segments(engine, nuc, port_oracle):
    model, mid = nuc
    rs = synth.gen_reads(5, 1400, model, seed=808, drift=True)
    jobs = synth.scorereads_jobs(rs, 170, model_id=mid, rc_every=2)      # ~100-base segments like eventalign.cpp:668
    for flags in (0, 3):
        jj = jobs.jobs.copy(); jj["flags"] = flags
        got, scores = engine.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jj)
        oj = jj.copy(); oj["model_id"] = 0
        want = [port_oracle.hmm_align(rs.reads, rs.ev_mean, rs.ev_start_time, [model], jobs.kmer_ranks, oj[j]) for j in range(jj.shape[0])]
        _compare(got, want)
        assert all(g.shape[0] > 0 for g in got)
        for g, s in zip(got, scores):
            assert np.float32(g["l_fm"][-1]).view(np.uint32) == np.float32(s).view(np.uint32)


@pytest.mark.parametrize("shape", [
    dict(kmin=1, kmax=30, emin=2, emax=50, n=200),
    dict(kmin=20, kmax=120, emin=30, emax=260, n=120),
    dict(kmin=260, kmax=420, emin=300, emax=700, n=16),       # several chained strips
    dict(kmin=300, kmax=500, emin=5, emax=30, n=24),          # fewer events than k-mers: skips and -inf paths
])
def test_random_shapes(engine, nuc, port_oracle, shape):
    model, mid = nuc
    rs = synth.gen_reads(6, 2200, model, seed=300 + shape["kmin"])
    rng = np.random.default_rng(shape["kmax"])
    jobs = random_hmm_jobs(rs, rng, shape["n"], shape["kmin"], shape["kmax"], shape["emin"], shape["emax"], [0, 1, 2, 3])
    dj = jobs.jobs.copy(); dj["model_id"] = mid
    got, _ = engine.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dj, indel_bias=0.9)
    want = [port_oracle.hmm_align(rs.reads, rs.ev_mean, rs.ev_start_time, [model], jobs.kmer_ranks, jobs.jobs[j], indel_bias=0.9)
            for j in range(dj.shape[0])]
    _compare(got, want)


def test_single_event_job_returns_nothing(engine, nuc):
    model, mid = nuc
    rs = synth.gen_reads(1, 600, model, seed=4)
    jobs = synth.scorereads_jobs(rs, 100, model_id=mid)
    assert jobs.jobs.shape[0] >= 2
    jj = jobs.jobs.copy()
    jj[0]["event_stop"] = jj[0]["event_start"]      # n_events == 1: the reference asserts n_events >= 2
    got, _ = engine.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jj)
    assert got[0].shape[0] == 0 and got[1].shape[0] > 0
