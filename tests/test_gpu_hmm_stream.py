"""The streamed full-warp single-strip classes (hmm_forward_kernel<C, 32, false>, C = 6..10): a warp runs its jobs back to back through
one wavefront while they have more than 32 rows and no clipping, and hands the first job that does not to the general loop.  Scores are
compared bit for bit with the oracle on batches large enough that most warps stream more than one job."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import forward_cases as fc
from tests.random_cases import random_hmm_jobs

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def models(engine):
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    return [(nuc, engine.model_upload(nuc)), (cpg, engine.model_upload(cpg))]


# Each K range is one strip of a streamed class (K = 32C fills it, K = 32(C - 1) + 1 leaves lanes beyond K), and E starts where the
# class model sends every K of the range there: windows of 3 to about 140 rows go to the chained classes at these K, so the only
# short windows a streamed class ever holds have one or two rows.  Job counts are prime and well above twice the warps of a launch
# (16 per SM), so warps stream runs of several jobs and the last warps of a class take fewer.  Flags 1..3 (pre- or post-clipping) and
# windows of one or two rows end a stream wherever the longest-first order puts them.
# C8-two-models hands each job to the nucleotide or the cpg model at random, so a stream forms its next job's Gaussians from another
# model than the job it leaves.  The k-mer ranks are the nucleotide ones (base 4); they index the cpg table validly and the device
# and the oracle read them alike, but these are not cpg windows: the case only mixes model ids within a stream.
@pytest.mark.parametrize("kmin, kmax, n_jobs, emin, emax, flags, n_models, streamed", [
    pytest.param(161, 192, 6007, 145, 260, [0], 1, {6}, id="C6"),
    pytest.param(193, 224, 7001, 83, 200, [0] * 12 + [1, 2, 3], 1, {7}, id="C7-clipped"),
    pytest.param(225, 256, 6007, 191, 300, [0], 1, {8}, id="C8"),
    pytest.param(225, 256, 7001, 191, 300, [0] * 12 + [1, 2, 3], 2, {8}, id="C8-two-models"),
    pytest.param(257, 320, 12011, 237, 320, [0], 1, {9, 10}, id="C9-C10"),
    pytest.param(257, 320, 20011, 143, 400, [0] * 12 + [1, 2, 3], 1, {9, 10}, id="C9-C10-clipped"),
    pytest.param(289, 320, 26003, 1, 300, [0] * 6 + [3], 1, {10}, id="C10-short-windows"),
])
def test_streamed_classes_bit_exact(engine, models, port_oracle, kmin, kmax, n_jobs, emin, emax, flags, n_models, streamed):
    rs = synth.gen_reads(16, 2000, models[0][0], seed=7000 + n_jobs, drift=True)
    rng = np.random.default_rng(n_jobs)
    jobs = random_hmm_jobs(rs, rng, n_jobs, kmin, kmax, emin, emax, flags)
    jobs.jobs["model_id"] = rng.integers(0, n_models, n_jobs)
    E = np.abs(jobs.jobs["event_stop"].astype(np.int64) - jobs.jobs["event_start"]) + 1
    K = jobs.jobs["n_kmers"].astype(np.int64)
    assert {kmin, kmax} <= set(K.tolist())
    cls, _ = fc.choose_class_np(K, E)
    cls = np.array([fc.class_of(int(c)) in fc.STREAMED and fc.class_of(int(c))[0] for c in cls])
    assert set(cls[cls > 0].tolist()) == streamed
    # each class launches at most 16 warps per SM: with more than twice as many streamable jobs, warps stream runs of several jobs
    import torch
    warps = fc.WARPS_PER_SM_W32 * torch.cuda.get_device_properties(0).multi_processor_count
    streamable = (E >= fc.STREAM_MIN_E) & (jobs.jobs["flags"] == 0)
    for C in streamed:
        assert (streamable & (cls == C)).sum() > 2 * warps, f"class ({C}, 32): {(streamable & (cls == C)).sum()} streamable jobs"
        if flags != [0]:
            assert (~streamable & (cls == C)).any()
    if n_models == 2:
        assert set(jobs.jobs["model_id"][cls > 0].tolist()) == {0, 1}
    dev_jobs = jobs.jobs.copy()
    dev_jobs["model_id"] = np.array([m[1] for m in models], np.uint32)[jobs.jobs["model_id"]]
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs, indel_bias=0.9)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [m[0] for m in models[:n_models]], jobs.kmer_ranks,
                                          jobs.jobs, indel_bias=0.9, threads=8)
    mism = np.flatnonzero(_bits(got) != _bits(want))
    assert mism.size == 0, (f"{mism.size} of {got.size} scores differ in bits, first {mism[:5]}: {got[mism[:5]]} vs {want[mism[:5]]}; "
                            f"E {E[mism[:5]]}, K {K[mism[:5]]}, flags {jobs.jobs['flags'][mism[:5]]}, class C {cls[mism[:5]]}")
