"""The device forward kernel (csrc/hmm_forward_kernel.cuh) at its class edges, against the port oracle bit for bit (the oracle is
pinned to the compiled reference on the same jobs by tests/test_forward_edges_oracle.py):
  * every job of tests/forward_cases.py: each of the 34 reachable (C, W, chained) classes at K = n*W*C - 1, n*W*C, n*W*C + 1,
    with the last k-mer in column 0 and C - 1 of its lane, lanes wholly past K, one and two rows, the chained period edge
    E = 39..41 and E < 40 (and E = 1) over several strips, flags 0..3 on both strands, indel bias 1.0 and 0.9, outlier events
    mid-window and on the last row, events exactly on the model level, and windows of one to four k-mers with up to 240 rows
    per k-mer; sub-warp warps that mix step counts and pre-clipping
    and leave empty groups; one launch per class the restatement assigns, and the base-code form giving the same bits;
  * the pipelined one-shot call (drift 0, at least 2^20 events: levels are copied in chunks behind a progress word) with jobs of
    the streamed and the sub-warp classes in every chunk, more than twice as many streamable jobs per streamed class as warps,
    against the staged resident call, the base-code forms and the oracle."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import forward_cases as fc

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


@pytest.fixture(scope="module")
def cases(port_oracle):
    """{bias: (batch, oracle scores)}"""
    model = synth.load_model("nucleotide")
    out = {}
    for bias, b in fc.batches(model).items():
        want, _ = port_oracle.hmm_score_batch(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs, indel_bias=bias,
                                              threads=8)
        out[bias] = (b, want)
    return out


def _device_jobs(jobs, mid):
    dj = jobs.copy()
    dj["model_id"] = mid
    return dj


def _compare(b, got, want, what=""):
    bad = np.flatnonzero(_bits(got) != _bits(want))
    if bad.size:
        j = int(bad[0])
        s = b.spec[j]
        cls, steps = fc.choose_class(s.K, s.E)
        g = fc.wave_geometry(s.K, s.E, cls[0], cls[1], True)
        raise AssertionError(f"{what}: {bad.size} of {got.size} scores differ; first job {j}: class {cls}, K {s.K}, E {s.E}, flags "
                             f"{s.flags}, rc {s.rc}, strips {g.n_strips}, end lane {g.end_lane}, end slot {g.end_slot}, steps {steps}, "
                             f"edges {sorted(s.edges)}: {got[j]} vs {want[j]}")


@pytest.mark.parametrize("bias", fc.BIASES)
def test_every_edge_bit_exact(engine, nuc, cases, bias):
    _, mid = nuc
    b, want = cases[bias]
    got = engine.hmm_score_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, _device_jobs(b.jobs, mid), indel_bias=bias)
    _compare(b, got, want, f"bias {bias}")
    classes = set(fc.classes_of(b))
    assert classes == fc.REACHABLE
    assert engine.last_kernel_ms()[1] == len(classes) == 34


@pytest.mark.parametrize("bias", fc.BIASES)
def test_base_code_form_same_bits(engine, nuc, cases, bias):
    _, mid = nuc
    b, want = cases[bias]
    codes, cj = fc.code_form(b)
    got = engine.hmm_score_batch_seq(b.reads, b.ev_mean, b.ev_start_time, codes, _device_jobs(cj, mid), indel_bias=bias)
    _compare(b, got, want, f"base codes, bias {bias}")


@pytest.mark.parametrize("cls", [(4, 4, False), (8, 8, False), (8, 16, False), (9, 32, False), (4, 32, True)])
def test_single_class_batch_is_one_launch(engine, nuc, cases, port_oracle, cls):
    model, mid = nuc
    specs = [s for b, _ in cases.values() for s in b.spec if fc.choose_class(s.K, s.E)[0] == cls]
    sub = fc.make_batch(specs, model, seed=12)
    assert sub.jobs.shape[0] >= 16 and set(fc.classes_of(sub)) == {cls}
    want, _ = port_oracle.hmm_score_batch(sub.reads, sub.ev_mean, sub.ev_start_time, [model], sub.kmer_ranks, sub.jobs, indel_bias=0.9,
                                          threads=8)
    got = engine.hmm_score_batch(sub.reads, sub.ev_mean, sub.ev_start_time, sub.kmer_ranks, _device_jobs(sub.jobs, mid), indel_bias=0.9)
    _compare(sub, got, want, f"class {cls}")
    assert engine.last_kernel_ms()[1] == 1


def test_pipelined_one_shot_streamed_and_sub_warp_classes(engine, nuc, port_oracle):
    """the one-shot call copies the levels in chunks behind a progress word, and every job a warp fetches, inside a stream too,
    first checks that its read's chunk has landed.  Each streamed class has more than twice as many streamable jobs as the warps
    of its launch, so warps pull further jobs inside run_stream, and its schedule runs chunk by chunk, so a warp can stream from
    the last job of one chunk into a longer job of the next.  Whether a chunk is still in flight when a warp reaches it depends
    on the copy's timing and is not measured here.  Scores equal the staged resident call's, the base-code forms' and the
    oracle's."""
    model, mid = nuc
    b, chunks = fc.pipelined_batch(model)
    # the chunked-upload conditions of the one-shot call: drift 0 on every read and at least 2^20 events
    assert (b.reads["drift"] == 0).all() and b.ev_mean.shape[0] >= fc.PIPELINE_MIN_EVENTS
    classes = fc.classes_of(b)
    assert set(chunks.tolist()) == set(range(fc.LEVEL_CHUNKS))
    for c in range(fc.LEVEL_CHUNKS):
        here = {cl for cl, ch in zip(classes, chunks) if ch == c}
        assert len(here & fc.STREAMED) == 5 and {4, 8, 16} <= {cl[1] for cl in here}, f"chunk {c} holds {sorted(here)}"
    assert fc.rising_chunk_boundaries(b, chunks), "no streamed class enters a longer job at a chunk boundary"
    import torch
    warps = fc.WARPS_PER_SM_W32 * torch.cuda.get_device_properties(0).multi_processor_count
    streamable = np.array([s.E >= fc.STREAM_MIN_E and s.flags == 0 for s in b.spec])
    for cls in fc.STREAMED:
        n = int((streamable & np.array([c == cls for c in classes])).sum())
        assert n > 2 * warps, f"class {cls}: {n} streamable jobs for {warps} warps"
    dj = _device_jobs(b.jobs, mid)
    got = engine.hmm_score_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, dj)
    assert engine.last_kernel_ms()[1] == len(set(classes))
    engine.reads_load(b.reads, b.ev_mean, b.ev_start_time)
    engine.hmm_jobs_load(b.kmer_ranks, dj)
    engine.hmm_score()
    resident = engine.hmm_scores_fetch()
    _compare(b, got, resident, "one-shot vs resident")
    codes, cj = fc.code_form(b)
    cj = _device_jobs(cj, mid)
    _compare(b, engine.hmm_score_batch_seq(b.reads, b.ev_mean, b.ev_start_time, codes, cj), got, "base-code one-shot")
    engine.reads_load(b.reads, b.ev_mean, b.ev_start_time)
    engine.hmm_jobs_load_seq(codes, cj)
    engine.hmm_score()
    _compare(b, engine.hmm_scores_fetch(), got, "base-code resident")
    rng = np.random.default_rng(3)
    sample = np.sort(rng.choice(b.jobs.shape[0], 600, replace=False))
    want, _ = port_oracle.hmm_score_batch(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, np.ascontiguousarray(b.jobs[sample]),
                                          threads=16)
    sb = fc.vc.Batch(b.reads, b.ev_mean, b.ev_start_time, b.jobs[sample], b.kmer_ranks, None, [b.spec[j] for j in sample])
    _compare(sb, got[sample], want, "one-shot vs oracle")
