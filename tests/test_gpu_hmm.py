"""Parity of the CUDA forward kernel (through the C ABI) with the oracle: bit-exact floats.
north_star's bar is 1e-4 relative; we hold the stronger one because the kernel reproduces the
reference's operation order, quantised logsum and IEEE roundings exactly."""
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.golden_cases import make_hmm_cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REL_TOL = 1e-4   # north_star tolerance (we additionally assert bit equality)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check(got, want):
    assert got.shape == want.shape
    rel = np.abs(got - want) / np.maximum(1e-30, np.abs(want))
    assert np.nanmax(rel) <= REL_TOL, f"max rel err {np.nanmax(rel)}"
    mism = np.flatnonzero(_bits(got) != _bits(want))
    assert mism.size == 0, f"{mism.size} of {got.size} scores differ in bits, first {mism[:5]}: {got[mism[:5]]} vs {want[mism[:5]]}"


@pytest.fixture(scope="module")
def models(engine):
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    return {"nucleotide": (nuc, engine.model_upload(nuc)), "cpg": (cpg, engine.model_upload(cpg))}


@pytest.mark.parametrize("name", ["segments", "short_bias08", "methylation"])
def test_golden_cases(engine, models, port_oracle, name):
    case = make_hmm_cases()[name]
    rs, jobs = case["rs"], case["jobs"]
    mlist = [models[a][0] for a in case["alphabets"]]
    # golden_cases numbers models 0 (nucleotide) / 1 (cpg); map to the ids this context handed out
    dev_jobs = jobs.jobs.copy()
    dev_jobs["model_id"] = np.array([models[a][1] for a in case["alphabets"]], np.uint32)[jobs.jobs["model_id"]]
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs,
                                 indel_bias=case["indel_bias"])
    gold = np.load(os.path.join(GOLD, "hmm_golden.npz"))[name]
    _check(got, gold)                          # the compiled reference's recorded output
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, mlist, jobs.kmer_ranks,
                                          jobs.jobs, indel_bias=case["indel_bias"])
    _check(got, want)


from tests.random_cases import HMM_SHAPES, random_hmm_jobs as _random_jobs


@pytest.mark.parametrize("shape", HMM_SHAPES)
def test_random_shapes_bit_exact(engine, models, port_oracle, shape):
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(8, 2600, nuc, seed=900 + shape["kmin"], drift=True)
    rng = np.random.default_rng(shape["kmin"] * 7 + 1)
    jobs = _random_jobs(rs, rng, shape["n"], shape["kmin"], shape["kmax"], shape["emin"], shape["emax"], [0, 1, 2, 3])
    dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = models["nucleotide"][1]
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs, indel_bias=0.9)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, jobs.jobs,
                                          indel_bias=0.9, threads=8)
    _check(got, want)


def test_methylation_calls_identical(engine, models, port_oracle):
    """LLR = ll_m - ll_u per site, call rule abs(LLR) >= 2.0*n_motif (scripts/calculate_methylation_frequency.py:26,45,49)."""
    nuc, cpg = models["nucleotide"][0], models["cpg"][0]
    rs = synth.gen_reads(30, 3000, nuc, seed=4242, cpg_keep=0.3)
    jobs = synth.methylation_jobs(rs, model_id=1)
    dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = models["cpg"][1]
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, dev_jobs)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc, cpg], jobs.kmer_ranks, jobs.jobs, threads=8)
    _check(got, want)
    llr_g = got[1::2].astype(np.float64) - got[0::2]
    llr_w = want[1::2].astype(np.float64) - want[0::2]
    assert np.array_equal(np.round(llr_g, 2), np.round(llr_w, 2))
    assert np.array_equal(np.abs(llr_g) >= 2.0, np.abs(llr_w) >= 2.0)


def test_staged_api_and_rescoring(engine, models, port_oracle):
    """reads stay resident; new job lists (and a new indel bias) are scored against them."""
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(5, 1500, nuc, seed=31)
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    for seg, bias in [(200, 1.0), (120, 0.8)]:
        jobs = synth.scorereads_jobs(rs, seg, rc_every=2)
        dev_jobs = jobs.jobs.copy(); dev_jobs["model_id"] = models["nucleotide"][1]
        engine.hmm_jobs_load(jobs.kmer_ranks, dev_jobs, bias)
        engine.hmm_score()
        got = engine.hmm_scores_fetch()
        want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, jobs.jobs, indel_bias=bias, threads=8)
        _check(got, want)
        ms, launches = engine.last_kernel_ms()
        assert ms > 0 and launches >= 1


def test_invalid_jobs_are_rejected(engine, models):
    from nanopolish_b200._lib import NphError
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(1, 300, nuc, seed=5)
    jobs = synth.scorereads_jobs(rs, 100, model_id=models["nucleotide"][1])
    bad = jobs.jobs.copy()
    bad[0]["event_stop"] = 10_000            # beyond the read: the reference would read out of bounds
    with pytest.raises(NphError):
        engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, bad)
    bad = jobs.jobs.copy()
    bad[0]["stride"] = -1                    # stride must follow the event order (assert in profile_hmm_r9.inl:275)
    with pytest.raises(NphError):
        engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, bad)


def test_exact_math_primitives_on_device():
    """div_by_cached_rcp == __fdiv_rn and the 8-instruction logsum == p7_FLogsum, bit for bit (2e8 pairs each)."""
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_exact_math")
    r = subprocess.run([exe, "200"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches" in r.stdout


def test_rank_outside_model_is_rejected(engine, models):
    from nanopolish_b200._lib import NphError
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(1, 400, nuc, seed=6)
    jobs = synth.scorereads_jobs(rs, 100, model_id=models["nucleotide"][1])
    bad = jobs.kmer_ranks.copy()
    bad[7] = 4096                        # 4^6 states: ranks are 0..4095
    with pytest.raises(NphError):
        engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, bad, jobs.jobs)


def test_empty_batch_is_ok(engine, models):
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(1, 300, nuc, seed=6)
    out = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.zeros(0, np.uint32), np.zeros(0, synth.HMM_JOB_DT))
    assert out.shape == (0,)


def test_full_size_properties(engine, models, port_oracle):
    """BASELINE configs[1] at full size (10 000 reads x 4 000 events, 60 000 jobs) through size-independent
    properties: (a) a random sample of jobs equals the oracle bit for bit; (b) scoring a permuted job list
    permutes the scores (scheduling does not leak into results); (c) a second run is bit-identical."""
    nuc, mid = models["nucleotide"]
    rs = synth.gen_reads(10000, 4000, nuc, seed=42)
    jobs = synth.scorereads_jobs(rs, 500, model_id=mid)
    assert jobs.jobs.shape[0] == 60000
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    engine.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
    engine.hmm_score(); a = engine.hmm_scores_fetch()
    engine.hmm_score(); b = engine.hmm_scores_fetch()
    assert np.array_equal(_bits(a), _bits(b)) and np.isfinite(a).all()
    rng = np.random.default_rng(0)
    perm = rng.permutation(jobs.jobs.shape[0])
    engine.hmm_jobs_load(jobs.kmer_ranks, np.ascontiguousarray(jobs.jobs[perm]))
    engine.hmm_score(); c = engine.hmm_scores_fetch()
    assert np.array_equal(_bits(c), _bits(a[perm]))
    sample = np.sort(rng.choice(jobs.jobs.shape[0], 160, replace=False))
    oj = np.ascontiguousarray(jobs.jobs[sample]); oj["model_id"] = 0
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, oj, threads=64)
    _check(a[sample], want)
    # mean log-likelihood per scored event of the whole batch sits where the generator puts it
    assert abs(a.astype(np.float64).sum() / jobs.scored_events + 2.88) < 0.05


def test_two_contexts_from_two_threads(models, port_oracle):
    """The reference calls profile_hmm_score concurrently from OpenMP workers (bam_processor.cpp:99): one context per
    thread must work side by side on the same device and give the same bits."""
    import threading
    from nanopolish_b200.engine import Engine
    nuc = models["nucleotide"][0]
    results, errors = {}, []

    def work(tid):
        try:
            eng = Engine(0)
            mid = eng.model_upload(nuc)
            rs = synth.gen_reads(40, 1800, nuc, seed=700 + tid)
            jobs = synth.scorereads_jobs(rs, 300, model_id=mid, rc_every=2)
            outs = [eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs).copy() for _ in range(6)]
            results[tid] = (rs, jobs, outs)
            eng.close()
        except Exception as ex:      # surfaced below
            errors.append(ex)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for tid, (rs, jobs, outs) in results.items():
        oj = jobs.jobs.copy(); oj["model_id"] = 0
        want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, oj, threads=8)
        for o in outs:
            _check(o, want)


def test_streamed_inputs_one_shot_call(engine, models, port_oracle):
    """Batches above 2^20 events take the pipelined one-shot path: levels and k-mer ranks stream in behind progress
    words while the forward kernels already run; scores must not change, and a bad rank is still rejected."""
    from nanopolish_b200._lib import NphError
    nuc, mid = models["nucleotide"]
    rs = synth.gen_reads(320, 3600, nuc, seed=909)
    assert rs.total_events > (1 << 20)
    jobs = synth.scorereads_jobs(rs, 400, model_id=mid, rc_every=2)
    got = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs)
    # same batch through the staged (fully resident) calls
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    engine.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
    engine.hmm_score()
    resident = engine.hmm_scores_fetch()
    assert np.array_equal(_bits(got), _bits(resident))
    sample = np.arange(0, jobs.jobs.shape[0], 37)
    oj = np.ascontiguousarray(jobs.jobs[sample]); oj["model_id"] = 0
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, oj, threads=16)
    _check(got[sample], want)
    bad = jobs.kmer_ranks.copy()
    bad[-5] = 5000
    with pytest.raises(NphError):
        engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, bad, jobs.jobs)
    again = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs)   # context still usable
    assert np.array_equal(_bits(again), _bits(got))


@pytest.mark.parametrize("shape", HMM_SHAPES[:4])
def test_base_code_form_equals_rank_form(engine, models, shape):
    """nph_hmm_score_batch_seq (one byte per base, ranks formed in the kernel prologue, both strands) returns the bits of the rank form;
    the staged form likewise; a code outside the alphabet is refused."""
    nuc = models["nucleotide"][0]
    rs = synth.gen_reads(8, 2600, nuc, seed=900 + shape["kmin"], drift=True)
    rng = np.random.default_rng(shape["kmin"] * 7 + 1)
    jobs = _random_jobs(rs, rng, shape["n"], shape["kmin"], shape["kmax"], shape["emin"], shape["emax"], [0, 1, 2, 3])
    rj = jobs.jobs.copy(); rj["model_id"] = models["nucleotide"][1]
    cj = jobs.code_jobs.copy(); cj["model_id"] = models["nucleotide"][1]
    a = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, rj, indel_bias=0.9)
    b = engine.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.seq_codes, cj, indel_bias=0.9)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and (rj["rc"] == 1).any()
    engine.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    engine.hmm_jobs_load_seq(jobs.seq_codes, cj, indel_bias=0.9)
    engine.hmm_score()
    assert np.array_equal(engine.hmm_scores_fetch().view(np.uint32), a.view(np.uint32))
    bad = jobs.seq_codes.copy(); bad[int(cj[0]["rank_off"]) + 1] = 4
    from nanopolish_b200._lib import NphError
    with pytest.raises(NphError):
        engine.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, bad, cj, indel_bias=0.9)


def test_base_code_form_cpg_alphabet(engine, models, port_oracle):
    """methylated windows over the cpg alphabet (codes 0..4) through the base-code form"""
    case = make_hmm_cases()["methylation"]
    rs, jobs = case["rs"], case["jobs"]
    ids = np.array([models[a][1] for a in case["alphabets"]], np.uint32)
    rj = jobs.jobs.copy(); rj["model_id"] = ids[jobs.jobs["model_id"]]
    cj = jobs.code_jobs.copy(); cj["model_id"] = ids[jobs.jobs["model_id"]]
    a = engine.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, rj, indel_bias=case["indel_bias"])
    b = engine.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.seq_codes, cj, indel_bias=case["indel_bias"])
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and (jobs.seq_codes == 3).any()
