"""The device Viterbi aligner (csrc/hmm_viterbi.cu) at its edges, against the port oracle bit for bit (the oracle is pinned to
the compiled reference on the same jobs by tests/test_viterbi_edges_oracle.py):
  * every job of tests/viterbi_cases.py: every class at K = n*32C - 1, n*32C, n*32C + 1, one-column last lanes, E < 40 over
    several strips, skip runs and stalls longer than the backtrack's staged corner, homopolymer runs, strip boundaries crossed
    inside a staged corner, both strands, flags 0-3, indel bias 1.0 and 0.9, and jobs the reference asserts on;
  * the room each job gets in states_out: exactly the path, one less, none, caller-owned bytes around the slices, refused
    non-monotone offsets, and the staged nph_hmm_align against the batch call;
  * the resident-CTA cap (one long window among small ones) and the refusal of a window whose trace exceeds the budget."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from tests import viterbi_cases as vc

pytestmark = pytest.mark.gpu

NPH_ERR_INVALID, NPH_ERR_UNSUPPORTED = -3, -6
SENTINEL = 0xA5


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


@pytest.fixture(scope="module")
def cases(port_oracle):
    """{bias: (batch, oracle paths, oracle statuses)}"""
    model = synth.load_model("nucleotide")
    out = {}
    for bias, b in vc.batches(model).items():
        res = [port_oracle.hmm_align(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs[j], indel_bias=bias)
               for j in range(b.jobs.shape[0])]
        out[bias] = (b, [r[0] for r in res], [r[1] for r in res])
    return out


def _device_jobs(b, mid, rows=None):
    dj = (b.jobs if rows is None else b.jobs[rows]).copy()
    dj["model_id"] = mid
    return dj


def _compare(got, want, statuses, scores, what=""):
    for j, (g, w, st) in enumerate(zip(got, want, statuses)):
        if st != 0:
            assert g.shape[0] == 0 and np.isneginf(scores[j]), f"{what} job {j}: oracle status {st}, device {g.shape[0]} states"
            continue
        assert g.shape[0] == w.shape[0] > 0, f"{what} job {j}: {g.shape[0]} vs {w.shape[0]} states"
        assert np.array_equal(g["event_idx"], w["event_idx"]) and np.array_equal(g["kmer_idx"], w["kmer_idx"]), f"{what} job {j}: path"
        assert g["state"].tobytes() == w["state"].tobytes(), f"{what} job {j}: states"
        assert np.array_equal(g["l_fm"].view(np.uint32), w["l_fm"].view(np.uint32)), f"{what} job {j}: l_fm"
        assert np.float32(scores[j]).view(np.uint32) == g["l_fm"][-1].view(np.uint32), f"{what} job {j}: score"


def _oracle(port_oracle, b, bias=1.0):
    res = [port_oracle.hmm_align(b.reads, b.ev_mean, b.ev_start_time, [synth.load_model("nucleotide")], b.kmer_ranks, b.jobs[j],
                                 indel_bias=bias) for j in range(b.jobs.shape[0])]
    return [r[0] for r in res], [r[1] for r in res]


def _classes(b, rows=None):
    idx = range(b.jobs.shape[0]) if rows is None else rows
    return {vc.choose_class(int(b.jobs[j]["n_kmers"]), b.spec[j].E)[0] for j in idx}


@pytest.mark.parametrize("bias", [1.0, 0.9])
def test_every_edge_bit_exact(engine, nuc, cases, bias):
    _, mid = nuc
    b, want, statuses = cases[bias]
    got, scores = engine.hmm_align_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, _device_jobs(b, mid), indel_bias=bias)
    _compare(got, want, statuses, scores)
    _, launches = engine.last_kernel_ms()
    assert launches == len(_classes(b)) >= 5


def test_single_class_batch_is_one_launch(engine, nuc, cases, port_oracle):
    model, mid = nuc
    specs = [s for b, _, _ in cases.values() for s in b.spec]
    for C in (1, 4, 8):
        sub = vc.make_batch([s for s in specs if vc.choose_class(s.K, s.E)[0] == C], model, seed=12)
        assert sub.jobs.shape[0] >= 2 and _classes(sub) == {C}
        want, statuses = _oracle(port_oracle, sub)
        got, scores = engine.hmm_align_batch(sub.reads, sub.ev_mean, sub.ev_start_time, sub.kmer_ranks, _device_jobs(sub, mid))
        _compare(got, want, statuses, scores, f"class {C}")
        assert engine.last_kernel_ms()[1] == 1


def _align_with_offsets(engine, b, jobs, off, bias, staged=False, tail=0):
    """nph_hmm_align[_batch] with caller-chosen states offsets into a sentinel-filled buffer of off[-1] + tail states"""
    n = jobs.shape[0]
    buf = np.zeros(int(off[-1]) + tail, synth.ALIGN_STATE_DT)
    buf.view(np.uint8)[:] = SENTINEL
    counts = np.full(n, 0xFFFFFFFF, np.uint32)
    scores = np.zeros(n, np.float32)
    if staged:
        engine.reads_load(b.reads, b.ev_mean, b.ev_start_time)
        engine._check(engine.lib.nph_hmm_align(engine.ctx, _p(b.kmer_ranks), b.kmer_ranks.shape[0], _p(jobs), n, bias,
                                               _p(buf), _p(off), _p(counts), _p(scores)), "nph_hmm_align")
    else:
        engine._check(engine.lib.nph_hmm_align_batch(engine.ctx, _p(b.reads), b.reads.shape[0], _p(b.ev_mean), _p(b.ev_start_time),
                                                     b.ev_mean.shape[0], _p(b.kmer_ranks), b.kmer_ranks.shape[0], _p(jobs), n, bias,
                                                     _p(buf), _p(off), _p(counts), _p(scores)), "nph_hmm_align_batch")
    return buf, counts, scores


def test_room(engine, nuc, cases):
    _, mid = nuc
    b, want, statuses = cases[0.9]
    rows = [j for j in range(b.jobs.shape[0]) if statuses[j] == 0][:40]
    jobs = _device_jobs(b, mid, rows)
    L = np.array([want[j].shape[0] for j in rows], np.int64)
    full = np.array([b.spec[j].E + int(b.jobs[j]["n_kmers"]) + 2 for j in rows], np.int64)
    kind = np.arange(len(rows)) % 4            # 0: room == path, 1: one less, 2: none, 3: the usual E + K + 2
    room = np.where(kind == 0, L, np.where(kind == 1, L - 1, np.where(kind == 2, 0, full)))
    lead, tail = 7, 5
    off = np.zeros(len(rows) + 1, np.uint64)
    off[0] = lead
    off[1:] = lead + np.cumsum(room)
    results = [_align_with_offsets(engine, b, jobs, off, 0.9, tail=tail),
               _align_with_offsets(engine, b, jobs, off, 0.9, staged=True, tail=tail)]
    for buf, counts, scores in results:
        raw = buf.view(np.uint8).reshape(buf.shape[0], -1)
        assert (raw[:lead] == SENTINEL).all() and (raw[int(off[-1]):] == SENTINEL).all(), "bytes outside every job's slice changed"
        for i, j in enumerate(rows):
            g = buf[int(off[i]):int(off[i]) + int(counts[i])]
            if kind[i] in (1, 2):
                assert counts[i] == 0 and np.isneginf(scores[i]), f"job {j}: room {room[i]} for a {L[i]}-state path"
                continue
            _compare([g], [want[j]], [0], scores[i:i + 1], f"room {room[i]}")
    (b0, c0, s0), (b1, c1, s1) = results
    assert np.array_equal(c0, c1) and np.array_equal(s0.view(np.uint32), s1.view(np.uint32))
    for i in range(len(rows)):
        a, z = int(off[i]), int(off[i]) + int(c0[i])
        assert b0[a:z].tobytes() == b1[a:z].tobytes()
    bad = off.copy()
    bad[3] = bad[2] - 1
    with pytest.raises(NphError) as ei:
        _align_with_offsets(engine, b, jobs, bad, 0.9)
    assert ei.value.status == NPH_ERR_INVALID


def test_cta_cap_long_window_among_small_jobs(port_oracle):
    """one K = E = 2 100 window with 200 small jobs: the trace arena caps the resident CTAs below the SM count"""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    model = synth.load_model("nucleotide")
    rng = np.random.default_rng(31)
    jobs = [vc.plain(rng, 2100, 2100, rc=False, flags=0)]
    jobs += [vc.plain(rng, int(rng.integers(8, 90)), int(rng.integers(2, 150)), rc=bool(i & 1), flags=i % 4) for i in range(200)]
    b = vc.make_batch(jobs, model, seed=31)
    shapes = [(int(b.jobs[j]["n_kmers"]), s.E) for j, s in enumerate(b.spec)]
    assert 0 < vc.max_ctas(shapes, sm) < sm
    want, statuses = _oracle(port_oracle, b)
    eng = Engine(0)
    try:
        mid = eng.model_upload(model)
        got, scores = eng.hmm_align_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, _device_jobs(b, mid))
    finally:
        eng.close()
    _compare(got, want, statuses, scores, "cta cap")
    assert got[0].shape[0] > 2100


def test_trace_budget_refusal(engine, nuc, cases, port_oracle):
    """the smallest K = E window the restatement refuses raises NPH_ERR_UNSUPPORTED; the context then aligns as before"""
    model, mid = nuc
    n = vc.smallest_refused_square()
    assert vc.max_ctas([(n, n)], 132) == 0 and vc.max_ctas([(n - 1, n - 1)], 132) > 0
    big = vc.make_batch([vc.plain(np.random.default_rng(5), n, n)], model, seed=5)
    with pytest.raises(NphError) as ei:
        engine.hmm_align_batch(big.reads, big.ev_mean, big.ev_start_time, big.kmer_ranks, _device_jobs(big, mid))
    assert ei.value.status == NPH_ERR_UNSUPPORTED
    sub = vc.make_batch(cases[1.0][0].spec[:12], model, seed=13)
    want, statuses = _oracle(port_oracle, sub)
    got, scores = engine.hmm_align_batch(sub.reads, sub.ev_mean, sub.ev_start_time, sub.kmer_ranks, _device_jobs(sub, mid))
    _compare(got, want, statuses, scores, "after refusal")
