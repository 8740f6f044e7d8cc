"""nph_train_transitions_batch (scorereads --train-transitions on the device) against the compiled reference's recorded answers
(tests/golden/ref_transitions_edges.pkl.xz), against the restatement over nph_hmm_align_batch's paths on a scorereads-shaped
batch, across chunk sizes, on an empty batch and at every refusal."""
import copy

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from tests import transition_restatement as tr
from tests import tt_cases as tc
from tests.ref_calls import case_answers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    yield e
    e.close()


def _flat(counts):
    return np.frombuffer(np.ascontiguousarray(counts).tobytes(), np.uint64)


@pytest.mark.parametrize("spec", tc.CASES, ids=[s[0] for s in tc.CASES])
def test_counts_equal_reference(eng, spec):
    c = tc.build(spec)
    score, counts, probs, text, prior = case_answers("ref_transitions_edges.pkl.xz", spec[0])[tc.fingerprint(c)]
    jobs, codes, segs = tc.jobs_of(c)
    rs = c["rs"]
    got, cnt, _ = eng.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, codes, jobs, n_groups=1)
    assert np.array_equal(_flat(cnt[0]), counts)
    if jobs.shape[0]:
        want = eng.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, codes, jobs)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    nev = sum(abs(e0 - e1) + 1 for e0, e1, _ in segs)
    total = 0.0
    for v in got:
        total += float(v)
    assert (total / nev if nev else 1.0) == score
    assert tr.train(_flat(cnt[0]), prior if prior.shape[0] else None) == list(probs)


def _batch(n_reads=200, seed=3):
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(n_reads, 2100, model, seed=seed, drift=True)
    jb = synth.scorereads_jobs(rs, 500, rc_every=2)
    groups = (jb.jobs["read"] % 2).astype(np.uint8) + 2 * ((jb.jobs["read"] // 2) % 2).astype(np.uint8)   # strand x two groups
    return model, rs, jb, groups


def test_scorereads_batch_equals_restatement(eng):
    model, rs, jb, groups = _batch()
    codes, cj = jb.seq_codes, jb.code_jobs
    scores, cnt, chunks = eng.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, codes, cj, groups, n_groups=4)
    paths, _ = eng.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jb.kmer_ranks, jb.jobs)
    want = np.zeros((4, tr.WORDS), np.uint64)
    for j, p in enumerate(paths):
        jo = jb.jobs[j]
        r = rs.reads[int(jo["read"])]
        ranks = jb.kmer_ranks[int(jo["rank_off"]):int(jo["rank_off"]) + int(jo["n_kmers"])]
        path = [(int(s["event_idx"]), int(s["kmer_idx"]), s["state"].decode()) for s in p]
        tr.add_training(want[groups[j]], path, ranks, lambda rk, r=r: tr.scaled_mean(float(model.level_mean[rk]), float(r["scale"]), float(r["shift"])))
    for g in range(4):
        assert np.array_equal(_flat(cnt[g]), want[g]), g
    assert want[:, tr.SKIPS].min() > 0
    for cap in (1, 7):
        s2, c2, n2 = eng.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, codes, cj, groups, n_groups=4, max_chunk_jobs=cap)
        assert np.array_equal(s2.view(np.uint32), scores.view(np.uint32)) and c2.tobytes() == cnt.tobytes()
        assert n2 == (cj.shape[0] + cap - 1) // cap
    assert chunks == 1


def test_empty_batch(eng):
    z = np.zeros(0, synth.HMM_JOB_DT)
    rs = synth.gen_reads(1, 600, synth.load_model("nucleotide"), seed=1)
    s, c, n = eng.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.zeros(1, np.uint8), z)
    assert s.shape == (0,) and c.tobytes() == bytes(c.nbytes) and n == 0


def _refused(fn, text):
    with pytest.raises(NphError) as e:
        fn()
    assert text in str(e.value), str(e.value)


def test_refusals(eng):
    model, rs, jb, groups = _batch(8, seed=11)
    codes, cj = jb.seq_codes, jb.code_jobs
    call = lambda **kw: lambda: eng.train_transitions_batch(kw.pop("reads", rs.reads), rs.ev_mean, rs.ev_start_time, codes, kw.pop("jobs", cj), **kw)
    _refused(call(groups=groups, n_groups=3), "group 3 >= n_groups")
    _refused(call(n_groups=0), "n_groups outside 1..256")
    one = cj[:1].copy()
    one["event_stop"][0] = one["event_start"][0]            # a single event: profile_hmm_align asserts, K3 finds no path
    _refused(call(jobs=one), "found no path")
    # a non-finite mean behind a path: the k-mer of one rank gets a mean that overflows float, so every path skips it (its match
    # cells are -inf) and the skip after a match observes it (to = from + 1)
    j0 = cj[:1].copy()
    ranks = jb.kmer_ranks[int(jb.jobs[0]["rank_off"]):int(jb.jobs[0]["rank_off"]) + int(jb.jobs[0]["n_kmers"])]
    q = next(q for q in range(len(ranks) // 2, len(ranks) - 20) if np.count_nonzero(ranks == ranks[q]) == 1)
    bad = copy.copy(synth.load_model("nucleotide"))
    bad.level_mean = bad.level_mean.copy()
    bad.level_mean[ranks[q]] = 1e39
    e2 = Engine(0)
    try:
        e2.model_upload(bad)
        _refused(lambda: e2.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, codes, j0), "not finite")
    finally:
        e2.close()


def test_bin_edges_equal_restatement(eng):
    """a model whose means are multiples of 0.5 pA, some moved one float ulp up or down, and reads with scale 1 and shift 0: level
    differences fall exactly on bin edges (d = 0.5 n) and one or two ulps either side"""
    model = copy.copy(synth.load_model("nucleotide"))
    r = np.arange(model.level_mean.shape[0])
    m = (np.float32(80.0) + np.float32(0.5) * (r % 41)).astype(np.float32)
    m = np.where((r // 41) % 3 == 1, np.nextafter(m, np.float32(np.inf)), np.where((r // 41) % 3 == 2, np.nextafter(m, np.float32(0)), m))
    model.level_mean = m.astype(np.float64)
    rs = synth.gen_reads(40, 2100, model, seed=21, rng_scalings=False)
    jb = synth.scorereads_jobs(rs, 500, rc_every=2)
    e2 = Engine(0)
    try:
        e2.model_upload(model)
        _, cnt, _ = e2.train_transitions_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jb.seq_codes, jb.code_jobs, n_groups=1)
        paths, _ = e2.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, jb.kmer_ranks, jb.jobs)
    finally:
        e2.close()
    want = np.zeros(tr.WORDS, np.uint64)
    trace = []
    for j, p in enumerate(paths):
        jo = jb.jobs[j]
        ranks = jb.kmer_ranks[int(jo["rank_off"]):int(jo["rank_off"]) + int(jo["n_kmers"])]
        path = [(int(s["event_idx"]), int(s["kmer_idx"]), s["state"].decode()) for s in p]
        tr.add_training(want, path, ranks, lambda rk: tr.scaled_mean(float(model.level_mean[rk]), 1.0, 0.0), trace=trace)
    assert np.array_equal(_flat(cnt[0]), want)
    frac = [(2 * t[7]) % 1.0 for t in trace if t[0] == "obs" and t[7] > 0]
    assert any(f == 0.0 for f in frac)                        # exactly on an edge
    assert any(0 < f < 1e-3 for f in frac)                    # just above one
    assert any(f > 1 - 1e-3 for f in frac)                    # just below one
