"""The streamed full-warp single-strip classes (hmm_forward_kernel<C, 32, false>): a warp runs its jobs back to back through one
wavefront while they have more than 32 rows and no clipping, and hands the first job that does not to the general loop.  Scores are
compared bit for bit with the oracle on batches large enough that most warps stream more than one job."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.random_cases import random_hmm_jobs

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


# K over 257..320 puts every job in the C = 9 (K <= 288) or C = 10 single-strip class, K = 288 and 320 fill the strip, and K = 257
# leaves three lanes beyond K.  Job counts are well above the warps of a launch (16 per SM) and prime, so the last warps of a class
# take fewer jobs than the others.  Flags 1..3 (pre- or post-clipping) and windows of <= 32 events end a stream wherever the
# longest-first order puts them.
@pytest.mark.parametrize("n_jobs, emin, emax, flags", [
    (12011, 33, 70, [0]),                                # every job streams; E, K and the strand vary from job to job
    (15013, 20, 160, [0] * 12 + [1, 2, 3]),              # clipped jobs between streamed ones, short windows at the tail
    (16001, 30, 40, [0] * 6 + [3]),                      # E around the 33-row threshold, several jobs per warp
])
def test_streamed_classes_bit_exact(engine, nuc, port_oracle, n_jobs, emin, emax, flags):
    model, mid = nuc
    rs = synth.gen_reads(16, 2000, model, seed=7000 + n_jobs, drift=True)
    rng = np.random.default_rng(n_jobs)
    jobs = random_hmm_jobs(rs, rng, n_jobs, 257, 320, emin, emax, flags)
    E = np.abs(jobs.jobs["event_stop"].astype(np.int64) - jobs.jobs["event_start"]) + 1
    K = jobs.jobs["n_kmers"]
    assert {288, 320} <= set(K.tolist()) and K.min() <= 260
    assert (E > 32).any() and (flags == [0] or (E <= 32).any() or (jobs.jobs["flags"] != 0).any())
    # each class launches at most 16 warps per SM: with more than twice as many streamable jobs, warps stream runs of several jobs
    import torch
    warps = 16 * torch.cuda.get_device_properties(0).multi_processor_count
    streamable = (E > 32) & (jobs.jobs["flags"] == 0)
    assert (streamable & (K <= 288)).sum() > 2 * warps and (streamable & (K > 288)).sum() > 2 * warps
    dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = mid
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs, indel_bias=0.9)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [model], jobs.kmer_ranks, jobs.jobs,
                                          indel_bias=0.9, threads=8)
    mism = np.flatnonzero(_bits(got) != _bits(want))
    assert mism.size == 0, (f"{mism.size} of {got.size} scores differ in bits, first {mism[:5]}: {got[mism[:5]]} vs {want[mism[:5]]}; "
                            f"E {E[mism[:5]]}, K {K[mism[:5]]}, flags {jobs.jobs['flags'][mism[:5]]}")
