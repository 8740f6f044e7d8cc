"""nph_detect_polyi_batch on the device against the reference's own detect-polyi code (oracle/_ref/libnpref_polyi.so): identical
segmentations, read rates, lengths, QC, poly(I)/poly(A) switch indices and detection tags, byte-identical TSV rows."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from nanopolish_b200 import _lib, detect_polyi
from nanopolish_b200.synth import POLYI_RES_DT
from tests import polya_cases as pc
from tests import polyi_cases as qc

pytestmark = pytest.mark.gpu
NPH_ERR_INVALID = -3


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def ref():
    assert os.path.exists(qc.REF_POLYI), "oracle/_ref/libnpref_polyi.so is missing: build() makes it where the reference is"
    return qc.RefPolyi()


def _compare(eng, ref, reads):
    raw, jobs, dur, b2e = pc.pack(reads)
    got = eng.detect_polyi_batch(raw, jobs, dur, b2e)
    with ThreadPoolExecutor(max_workers=max(1, min(16, os.cpu_count() or 1))) as ex:
        want = list(ex.map(ref.read, reads))
    bad = []
    for r, g, (seg, rl, q, bern, det, row) in zip(reads, got, want):
        got_row = detect_polyi.row(r.name, r.contig, r.pos, g)
        if got_row != row:
            bad.append((r.name, r.samples.shape[0], got_row, row))
            continue
        s = g["seg"]
        if seg is None:
            assert (int(g["polyi_last"]), int(g["polya_first"]), int(g["detected"])) == (-1, -1, -1), r.name
            continue
        assert [int(s[k]) for k in ("start", "leader", "adapter", "polya", "cliffs")] == [int(v) for v in seg], r.name
        assert np.float64(s["read_rate"]).tobytes() == np.float64(rl[0]).tobytes(), r.name
        assert np.float64(s["polya_length"]).tobytes() == np.float64(rl[1]).tobytes(), r.name
        assert int(s["qc"]) == q, r.name
        assert (int(g["polyi_last"]), int(g["polya_first"]), int(g["detected"])) == (bern[0], bern[1], det), r.name
    assert not bad, f"{len(bad)} of {len(reads)} rows differ, first: {bad[:3]}"
    return got


def test_edge_reads(eng, ref):
    got = _compare(eng, ref, qc.edge_reads(np.random.default_rng(11), ref))
    assert set(int(v) for v in got["detected"]) == {-1, 0, 1, 2, 3}


def test_synthetic_polyi_reads(eng, ref):
    rng = np.random.default_rng(12)
    reads = [qc.synth_polyi_read(rng, f"syn_{i}", int(rng.integers(1000, 40000)), pos=i) for i in range(200)]
    got = _compare(eng, ref, reads)
    assert len(set(int(v) for v in got["detected"])) >= 3


def test_batch_of_long_and_short_reads(eng, ref):
    """2 000 reads of 10^3 .. 3*10^5 samples (log-uniform) in one call, launched longest first.  On the same batch the polya
    kernel segments at least one read differently: the poly(I) instantiation's mixture POLYA emission runs."""
    rng = np.random.default_rng(13)
    lens = np.exp(rng.uniform(np.log(1e3), np.log(3e5), 2000)).astype(np.int64)
    reads = [qc.synth_polyi_read(rng, f"b_{i}", int(n), cliffs=0.001) for i, n in enumerate(lens)]
    got = _compare(eng, ref, reads)
    raw, jobs, dur, b2e = pc.pack(reads)
    polya = eng.polya_batch(raw, jobs, dur, b2e)
    fields = ("start", "leader", "adapter", "polya", "cliffs")
    differ = sum(any(int(g["seg"][k]) != int(p[k]) for k in fields) for g, p in zip(got, polya))
    assert differ >= 1


def test_failed_loads_in_one_batch(eng, ref):
    """reads missing from the index (loaded = 0) and reads whose events load_from_raw cleared (n_events = 0) give the
    10-column READ_FAILED_LOAD row between computed ones"""
    rng = np.random.default_rng(14)
    reads = [qc.synth_polyi_read(rng, f"m_{i}", 5000) for i in range(12)]
    for r in reads[1::4]:
        r.loaded = False
    _compare(eng, ref, reads)
    for r in reads[2::4]:
        r.duration = np.zeros(0, np.float32)
        r.map_start[:] = -1; r.map_stop[:] = -1
    raw, jobs, dur, b2e = pc.pack(reads)
    got = eng.detect_polyi_batch(raw, jobs, dur, b2e)
    for r, g in zip(reads, got):
        failed = (not r.loaded) or r.duration.shape[0] == 0
        assert (int(g["seg"]["qc"]) == detect_polyi.READ_FAILED_LOAD) == failed, r.name
        if failed:
            assert detect_polyi.row(r.name, r.contig, r.pos, g).count("\t") == 9


def test_refused_inputs(eng):
    rng = np.random.default_rng(15)
    for name, edit in (("one_sample", None), ("bad_map", (2, 1)), ("map_past_events", (0, None))):
        r = pc.synth_read(rng, name, 1 if edit is None else 500)
        if edit is not None:
            r.map_start[3], r.map_stop[3] = edit[0], r.duration.shape[0] if edit[1] is None else edit[1]
        raw, jobs, dur, b2e = pc.pack([r])
        with pytest.raises(_lib.NphError):
            eng.detect_polyi_batch(raw, jobs, dur, b2e)
    # a read that failed to load is not computed, so it is not checked either
    r = pc.synth_read(rng, "unloaded_one_sample", 1)
    r.loaded = False
    raw, jobs, dur, b2e = pc.pack([r])
    assert int(eng.detect_polyi_batch(raw, jobs, dur, b2e)[0]["seg"]["qc"]) == detect_polyi.READ_FAILED_LOAD


def test_refuses_two_to_the_31_samples(eng):
    """A job claiming 2^31 samples is refused before anything is copied: the call is given a 4 096-sample buffer and told it
    holds 2^31 samples, so a copy would read far past it.  2^31 - 1 is the largest count BernoulliHMM's int bounds hold."""
    rng = np.random.default_rng(16)
    r = pc.synth_read(rng, "huge", 4096)
    raw, jobs, dur, b2e = pc.pack([r])
    jobs["n_samples"] = 1 << 31
    out = np.zeros(1, POLYI_RES_DT)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = eng.lib.nph_detect_polyi_batch(eng.ctx, p(raw), 1 << 31, p(jobs), 1, p(dur), dur.shape[0], p(b2e), b2e.shape[0], p(out))
    assert rc == NPH_ERR_INVALID
