"""The forward kernel's saturated log-sum index (lsum_sat, exact_math.cuh): the primitive on its own, and the kernel on jobs that
push it to its edges, bit for bit against the oracle.

A narrow level spread (small sigma') and outlier events make the state values very large in magnitude and put many
log-sum differences in and past [15.7, 16.384), the range the saturated index maps onto the zero entries 15700..16384.
Rows with every state at -inf (both operands -inf, a NaN difference) occur at the fill edges of every job."""
import os
import subprocess

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.random_cases import random_hmm_jobs

pytestmark = pytest.mark.gpu


def _reads(nuc, seed, var_scale, outlier_frac):
    rs = synth.gen_reads(6, 2600, nuc, seed=seed)
    rs.reads["var"] *= var_scale                      # sigma' = stdv * var: tight Gaussians, cc = log(1/sqrt(2pi)) - log(sigma') near 0
    rs.reads["log_var"] = np.log(rs.reads["var"])
    rng = np.random.default_rng(seed)
    n = rs.ev_mean.shape[0]
    pick = rng.choice(n, int(n * outlier_frac), replace=False)
    rs.ev_mean[pick] += rng.choice([-1.0, 1.0], pick.size) * rng.uniform(20.0, 400.0, pick.size)
    return rs


@pytest.fixture(scope="module")
def nuc(engine):
    model = synth.load_model("nucleotide")
    return model, engine.model_upload(model)


def _check(got, want):
    mism = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert mism.size == 0, f"{mism.size} of {got.size} scores differ, first {mism[:5]}: {got[mism[:5]]} vs {want[mism[:5]]}"


def test_saturated_logsum_primitive_on_device():
    """lsum_sat == p7_FLogsum and == the clamped lsum, bit for bit (5e8 pairs), edges of the saturated index included"""
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_lsum_saturated")
    r = subprocess.run([exe, "500"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches against the reference, 0 mismatches against the clamped form" in r.stdout


@pytest.mark.parametrize("var_scale, outlier_frac", [(0.2, 0.0), (0.35, 0.02), (1.0, 0.1)])
def test_scorereads_shaped_jobs(engine, port_oracle, nuc, var_scale, outlier_frac):
    nuc, mid = nuc
    rs = _reads(nuc, 70 + int(var_scale * 100), var_scale, outlier_frac)
    jobs = synth.scorereads_jobs(rs, 500, rc_every=2)
    assert jobs.jobs.shape[0] >= 24
    dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = mid
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, jobs.jobs, threads=8)
    assert np.all(np.isfinite(want))
    _check(got, want)


def test_clipped_and_short_jobs(engine, port_oracle, nuc):
    """soft-clip flags, sub-warp classes and chained strips on the same tight, outlier-laden reads"""
    nuc, mid = nuc
    rs = _reads(nuc, 91, 0.25, 0.05)
    rng = np.random.default_rng(91)
    jobs = random_hmm_jobs(rs, rng, 48, 4, 400, 2, 700, [0, 1, 2, 3])
    dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = mid
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs, indel_bias=0.9)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, jobs.jobs,
                                          indel_bias=0.9, threads=8)
    _check(got, want)
