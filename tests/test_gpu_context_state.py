"""Call-sequence rules of one context (include/nph.h): what a new read batch invalidates, what each call leaves resident,
which timing nph_last_kernel_ms reports, and that jobs a kernel of ours wrote do not lend their trust to jobs from the
host.  Every check runs on its own contexts, so no other test's leftovers decide the outcome."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine

pytestmark = pytest.mark.gpu
K = 6
NPH_ERR_INVALID = -3        # include/nph.h: bad argument
NPH_ERR_STATE = -5          # include/nph.h: call sequence error


def _status(fn, *args, **kw):
    try:
        fn(*args, **kw)
    except NphError as e:
        return e.status
    return 0


@pytest.fixture
def ctx():
    """a fresh context with the nucleotide model (id 0) and the cpg model (id 1)"""
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    e.model_upload(synth.load_model("cpg"))
    yield e
    e.close()


def _fresh():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    e.model_upload(synth.load_model("cpg"))
    return e


def _reads(n_reads=4, n_events=2000, seed=3, **kw):
    return synth.gen_reads(n_reads, n_events, synth.load_model("nucleotide"), seed=seed, **kw)


def test_jobs_before_reads_are_refused(ctx):
    rs = _reads()
    jobs = synth.scorereads_jobs(rs, 300)
    assert _status(ctx.hmm_jobs_load, jobs.kmer_ranks, jobs.jobs) == NPH_ERR_STATE


def test_new_read_batch_drops_the_resident_jobs(ctx):
    rs = _reads()
    jobs = synth.scorereads_jobs(rs, 300)
    ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    ctx.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
    ctx.hmm_score()
    first = ctx.hmm_scores_fetch()
    ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    assert _status(ctx.hmm_score) == NPH_ERR_STATE
    assert _status(ctx.hmm_scores_fetch) == NPH_ERR_STATE
    ctx.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
    ctx.hmm_score()
    assert ctx.hmm_scores_fetch().tobytes() == first.tobytes()


def _raw_batch(model, seed):
    raw, rr, seqs = synth.gen_raw(2, 12000, model, seed=seed, return_seqs=True)
    jobs = np.zeros(len(seqs), synth.RAW_JOB_DT)
    ranks = []
    roff = 0
    for i, (r, c) in enumerate(zip(rr, seqs)):
        rk = synth.kmer_ranks_from_codes(c, model.k, 4)
        jobs[i] = (int(r["sample_off"]), roff, int(r["n_samples"]), rk.shape[0], 4000.0)
        ranks.append(rk)
        roff += rk.shape[0]
    return raw, np.concatenate(ranks).astype(np.uint32), jobs


def _between(ctx, rs, which, abea_out):
    if which == "hmm_align":
        jobs = synth.scorereads_jobs(rs, 300)
        ctx.hmm_align(jobs.kmer_ranks, jobs.jobs)
    elif which == "eventalign_chain":
        pairs, emap, rf, rr, chains = synth.eventalign_chains(rs)
        ctx.eventalign_chain(pairs, emap, rf, rr, chains)
    elif which == "mom_batch":
        jobs, ranks, _ = synth.abea_jobs(rs)
        ctx.mom_batch(rs.reads, rs.ev_mean, ranks, jobs, 0)
    elif which == "reads_load":
        ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    elif which == "load_from_raw_batch":
        raw, ranks, jobs = _raw_batch(synth.load_model("nucleotide"), 21)
        ctx.load_from_raw_batch(raw, ranks, jobs, 0, synth.event_params(False))
    elif which == "trim_raw_batch":
        raw, rr = synth.gen_raw(2, 12000, synth.load_model("nucleotide"), seed=21)
        ctx.trim_raw_batch(raw, rr)
    elif which == "detect_events_batch":
        raw, rr = synth.gen_raw(2, 12000, synth.load_model("nucleotide"), seed=21)
        ctx.detect_events_batch(raw, rr, synth.event_params(False))
    elif which == "recalibrate_batch":
        jobs, ranks, _ = synth.abea_jobs(rs)
        ctx.recalibrate_batch(rs.reads, rs.ev_mean, ranks, jobs, 0, *abea_out)


@pytest.mark.parametrize("which", [None, "hmm_align", "eventalign_chain", "mom_batch", "reads_load", "load_from_raw_batch",
                                   "trim_raw_batch", "detect_events_batch", "recalibrate_batch"])
def test_staged_abea_is_dropped_by_calls_that_reuse_its_buffers(ctx, which):
    rs = _reads(3, 1500, seed=8)
    jobs, ranks, total = synth.abea_jobs(rs)
    want_pairs, want_res = ctx.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, 0, total)
    ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    ctx.abea_jobs_load(ranks, jobs, 0, total)
    ctx.abea_run()
    if which is None:
        pairs, res = ctx.abea_fetch()
        assert pairs.tobytes() == want_pairs.tobytes() and res.tobytes() == want_res.tobytes()
        assert (res["n_pairs"] > 0).all()
        return
    _between(ctx, rs, which, (want_pairs, want_res))
    assert _status(ctx.abea_run) == NPH_ERR_STATE
    assert _status(ctx.abea_fetch) == NPH_ERR_STATE


def _prologue_outputs(e, rs, abea, raw_batch):
    """every output of the ABEA-shaped calls on one good batch: one-shot and staged ABEA, MoM, calibration, load_from_raw"""
    jobs, ranks, total = abea
    pairs, res = e.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, 0, total)
    e.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    e.abea_jobs_load(ranks, jobs, 0, total)
    e.abea_run()
    staged = e.abea_fetch()
    mom = e.mom_batch(rs.reads, rs.ev_mean, ranks, jobs, 0)
    b2e, cal = e.recalibrate_batch(rs.reads, rs.ev_mean, ranks, jobs, 0, pairs, res)
    raw, raw_ranks, raw_jobs = raw_batch
    return [pairs, res, *staged, mom, b2e, cal, *e.load_from_raw_batch(raw, raw_ranks, raw_jobs, 0, synth.event_params(False))]


def test_bad_ranks_and_wrapping_offsets_are_refused(ctx):
    """A rank outside the model (4096 of a 6-mer model's 4^6 states) and a job slice whose offset is 2^64 - 1 are refused
    with NPH_ERR_INVALID by every ABEA-shaped call; afterwards the context computes a good batch exactly as a fresh one."""
    rs = _reads(3, 1500, seed=8)
    abea = jobs, ranks, total = synth.abea_jobs(rs)
    raw_batch = raw, raw_ranks, raw_jobs = _raw_batch(synth.load_model("nucleotide"), 21)
    fresh = _fresh()
    try:
        want = _prologue_outputs(fresh, rs, abea, raw_batch)
    finally:
        fresh.close()
    pairs, res = want[0], want[1]
    bad_ranks = ranks.copy()
    bad_ranks[int(jobs[1]["rank_off"]) + 5] = 4096
    wrapped = jobs.copy()
    wrapped[1]["rank_off"] = 2**64 - 1
    calls = [lambda r, j: ctx.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, r, j, 0, total),
             lambda r, j: (ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time), ctx.abea_jobs_load(r, j, 0, total)),
             lambda r, j: ctx.mom_batch(rs.reads, rs.ev_mean, r, j, 0),
             lambda r, j: ctx.recalibrate_batch(rs.reads, rs.ev_mean, r, j, 0, pairs, res)]
    for call in calls:
        assert _status(call, bad_ranks, jobs) == NPH_ERR_INVALID
        assert _status(call, ranks, wrapped) == NPH_ERR_INVALID
    bad_raw_ranks = raw_ranks.copy()
    bad_raw_ranks[-1] = 4096
    prm = synth.event_params(False)
    assert _status(ctx.load_from_raw_batch, raw, bad_raw_ranks, raw_jobs, 0, prm) == NPH_ERR_INVALID
    for field in ("sample_off", "rank_off"):
        wrapped_raw = raw_jobs.copy()
        wrapped_raw[0][field] = 2**64 - 1
        assert _status(ctx.load_from_raw_batch, raw, raw_ranks, wrapped_raw, 0, prm) == NPH_ERR_INVALID
    got = _prologue_outputs(ctx, rs, abea, raw_batch)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    assert (want[1]["n_pairs"] > 0).all() and (want[-1]["status"] == 0).any()


def _meth_inputs(rs):
    ref, pairs, recs = synth.methylation_records(rs, model_id=1, rc_every=4)
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    return ref, deltas, first, recs, synth.meth_params("cpg", K)


def test_pipelined_one_shot_leaves_a_clean_context(ctx):
    """drift 0 and >= 2^20 events: the one-shot score streams its levels behind progress words; what runs on the same
    context afterwards (a staged score on the batch it left resident, a call-methylation batch) sees none of that."""
    rs = _reads(300, 4000, seed=999, cpg_keep=0.3)
    assert rs.ev_mean.shape[0] >= 1 << 20 and not rs.reads["drift"].any()
    jobs = synth.scorereads_jobs(rs, 500, rc_every=3)
    meth = _meth_inputs(rs)
    one_shot = ctx.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs)
    ctx.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
    ctx.hmm_score()
    staged = ctx.hmm_scores_fetch()
    off, sites, scored = ctx.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, *meth)
    fresh = _fresh()
    try:
        want = fresh.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs)
        fresh.close()
        fresh = _fresh()
        fresh.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
        fresh.hmm_jobs_load(jobs.kmer_ranks, jobs.jobs)
        fresh.hmm_score()
        want_staged = fresh.hmm_scores_fetch()
        fresh.close()
        fresh = _fresh()
        want_off, want_sites, want_scored = fresh.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, *meth)
    finally:
        fresh.close()
    assert one_shot.tobytes() == want.tobytes()
    assert staged.tobytes() == want_staged.tobytes() == want.tobytes()
    assert off.tobytes() == want_off.tobytes() and sites.tobytes() == want_sites.tobytes() and scored == want_scored
    assert sites.shape[0] > 1000


def _screen_inputs(seed=11):
    ref, rs, recs, pairs = synth.gen_pileup(150, 14, 110, synth.load_model("nucleotide"), seed=seed, region_start=5000, n_true_variants=3)
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    return rs, synth._CODE2DNA[ref], deltas, first, recs, synth.screen_params(5000, K, 10, 30, 0, 4)


def test_kernel_time_needs_a_timed_call(ctx):
    assert _status(ctx.last_kernel_ms) == NPH_ERR_STATE
    rs, ref_chars, deltas, first, recs, params = _screen_inputs()
    ctx.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    ctx.screen_load(ref_chars, deltas, first, recs, params)
    ctx.screen_run()
    ms, launches = ctx.last_kernel_ms()
    assert launches >= 1 and ms > 0.0 and ctx.screen_counts()["rounds"] >= 1
    raw, ranks, jobs = _raw_batch(synth.load_model("nucleotide"), 33)
    ctx.load_from_raw_batch(raw, ranks, jobs, 0, synth.event_params(False))
    ms, launches = ctx.last_kernel_ms()
    assert launches >= 1 and ms > 0.0


@pytest.mark.parametrize("device_jobs", ["methylation", "screening"])
def test_device_written_jobs_do_not_vouch_for_host_jobs(ctx, device_jobs):
    if device_jobs == "methylation":
        rs = _reads(6, 2000, seed=44, cpg_keep=0.3)
        off, sites, _ = ctx.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, *_meth_inputs(rs))
        assert sites.shape[0] > 0
    else:
        rs, ref_chars, deltas, first, recs, params = _screen_inputs(12)
        ctx.screen_edits_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref_chars, deltas, first, recs, params)
        assert ctx.screen_counts()["jobs"] > 0
    rs = _reads(2, 1500, seed=5)                         # host jobs on a batch of their own
    jobs = synth.scorereads_jobs(rs, 100)
    assert jobs.jobs.shape[0] > 8
    bad_ranks = jobs.kmer_ranks.copy()
    bad_ranks[7] = 4096                                  # 4^6 states: ranks are 0..4095
    with pytest.raises(NphError):
        ctx.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, bad_ranks, jobs.jobs)
    bad_codes = jobs.seq_codes.copy()
    bad_codes[int(jobs.code_jobs[0]["rank_off"]) + 1] = 4     # the nucleotide alphabet has codes 0..3
    with pytest.raises(NphError):
        ctx.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, bad_codes, jobs.code_jobs)
    ok = ctx.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jobs.kmer_ranks, jobs.jobs)
    assert np.isfinite(ok).all()
