"""nph_polya_batch and nph_detect_polyi_batch on every edge case of tests/tail_cases.py, bit for bit against the port oracle
(npo_polya_trace) and against the compiled reference's recorded answers (tests/golden/ref_tail_edges.pkl.xz, looked up by
fingerprint): every case in one call and again in reverse order, reads of equal length, failed loads first, last and
consecutive, and more reads than the device holds at once.  Also the refusals: no k-mer, bad map entries, fewer than 2 samples,
a NaN duration in a mapped span, and a poly(I) job of 2^31 samples (given through the count only)."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import _lib
from nanopolish_b200.synth import POLYI_RES_DT
from tests import polya_cases as pc
from tests import ref_calls
from tests import tail_cases as tc

pytestmark = pytest.mark.gpu
NPH_ERR_INVALID = -3


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def cases(port_oracle):
    return tc.all_cases(port_oracle)


def _run(eng, mode, cs):
    raw, jobs, dur, b2e = pc.pack([c.read for c in cs])
    return (eng.polya_batch if mode == "polya" else eng.detect_polyi_batch)(raw, jobs, dur, b2e)


def _compare(eng, port, mode, cs, want=None):
    got = _run(eng, mode, cs)
    bad = []
    for c, g in zip(cs, got):
        mine = tc.result_answer(c, g)
        if mine != tc.port_answer(port, c) or (want is not None and mine != want[tc.fingerprint(c)]):
            bad.append((c.name, mine, tc.port_answer(port, c)))
    assert not bad, f"{mode}: {len(bad)} of {len(cs)} reads differ, first: {bad[:2]}"


@pytest.mark.parametrize("mode", tc.MODES)
def test_every_case_in_one_call(eng, port_oracle, cases, mode):
    """the device against the port and the recorded reference on every case, in one call and again in reverse order"""
    cs = [c for c in cases if c.mode == mode]
    want = ref_calls.case_answers(tc.GOLDEN, mode)
    assert {tc.fingerprint(c) for c in cs} <= set(want)
    _compare(eng, port_oracle, mode, cs, want)
    _compare(eng, port_oracle, mode, cs[::-1], want)


@pytest.mark.parametrize("mode", tc.MODES)
def test_each_case_alone(eng, port_oracle, cases, mode):
    """one read per call: the CTA's tiles and selection do not lean on the longest-first order of a batch"""
    for c in [c for c in cases if c.mode == mode and c.read.samples.shape[0] < 20000][:60]:
        _compare(eng, port_oracle, mode, [c])


@pytest.mark.parametrize("mode", tc.MODES)
def test_equal_lengths_and_failed_loads(eng, port_oracle, mode):
    """64 reads of one length (longest-first ties) with failed loads first, last and three in a row"""
    rng = np.random.default_rng(41)
    reads = [pc.synth_read(rng, f"{mode}-eq{i}", 3000, pos=i) for i in range(64)]
    for i in (0, 20, 21, 22, 63):
        reads[i].loaded = False
    _compare(eng, port_oracle, mode, [tc.TailCase(r.name, mode, r) for r in reads])


@pytest.mark.parametrize("mode", tc.MODES)
def test_more_reads_than_resident(eng, port_oracle, mode):
    """6 000 short reads: one CTA per read, so the grid runs in several waves on a 132-SM device"""
    rng = np.random.default_rng(42)
    reads = [pc.synth_read(rng, f"{mode}-w{i}", int(rng.integers(2, 700)), n_kmers=int(rng.integers(1, 20))) for i in range(6000)]
    _compare(eng, port_oracle, mode, [tc.TailCase(r.name, mode, r) for r in reads])


@pytest.mark.parametrize("mode", tc.MODES)
def test_refusals(eng, mode):
    rng = np.random.default_rng(43)
    call = eng.polya_batch if mode == "polya" else eng.detect_polyi_batch

    def refused(r):
        raw, jobs, dur, b2e = pc.pack([r])
        with pytest.raises(_lib.NphError):
            call(raw, jobs, dur, b2e)

    r = pc.synth_read(rng, "no-kmer", 500)
    r.map_start, r.map_stop = r.map_start[:0], r.map_stop[:0]
    refused(r)
    for s, e in ((2, 1), (-2, 0), (0, None)):
        r = pc.synth_read(rng, "bad-map", 500)
        r.map_start[3], r.map_stop[3] = s, r.duration.shape[0] if e is None else e
        refused(r)
    for n in (0, 1):
        r = pc.synth_read(rng, f"n{n}", 2, n_kmers=3)
        r.samples = r.samples[:n]
        refused(r)
    # a NaN duration in a mapped span is refused; in an unmapped one it is never read, and +inf is a defined order
    r = pc.synth_read(rng, "nan-dur", 500)
    k = int(np.nonzero(r.map_start != -1)[0][0])
    r.duration[r.map_start[k]] = np.float32(np.nan)
    refused(r)
    r = pc.synth_read(rng, "inf-dur", 500)
    r.duration[r.map_start[k]] = np.float32(np.inf)
    raw, jobs, dur, b2e = pc.pack([r])
    call(raw, jobs, dur, b2e)
    r.duration = np.concatenate([r.duration, np.float32([np.nan])])
    raw, jobs, dur, b2e = pc.pack([r])
    call(raw, jobs, dur, b2e)


def test_refuses_two_to_the_31_samples(eng):
    """detect-polyi refuses a job of 2^31 samples before anything is copied.  The call is given a buffer that really spans
    2^31 samples, so that a call which wrongly accepted the job would read only memory it owns and fail this test on its
    return code instead of reading past a small buffer: np.zeros maps the 8 GiB lazily, and a refused call touches none of it."""
    r = pc.synth_read(np.random.default_rng(44), "huge", 4096)
    _, jobs, dur, b2e = pc.pack([r])
    jobs["n_samples"] = 1 << 31
    raw = np.zeros(1 << 31, np.float32)
    out = np.zeros(1, POLYI_RES_DT)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = eng.lib.nph_detect_polyi_batch(eng.ctx, p(raw), raw.shape[0], p(jobs), 1, p(dur), dur.shape[0], p(b2e), b2e.shape[0], p(out))
    assert rc == NPH_ERR_INVALID
