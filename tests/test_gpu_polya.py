"""nph_polya_batch on the device against the reference's own poly(A) code (oracle/_ref/libnpref_polya.so): identical
segmentations, read rates, lengths and QC, byte-identical TSV rows; and the device expf / logf against this machine's libm."""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from nanopolish_b200 import _lib, polya
from tests import polya_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def ref():
    assert os.path.exists(pc.REF_POLYA), "oracle/_ref/libnpref_polya.so is missing: build() makes it where the reference is"
    return pc.RefPolya()


def _compare(eng, ref, reads):
    raw, jobs, dur, b2e = pc.pack(reads)
    got = eng.polya_batch(raw, jobs, dur, b2e)
    with ThreadPoolExecutor(max_workers=max(1, min(16, os.cpu_count() or 1))) as ex:
        want = list(ex.map(ref.read, reads))
    bad = []
    for r, g, (seg, rl, qc, row) in zip(reads, got, want):
        got_row = polya.row(r.name, r.contig, r.pos, g)
        if got_row != row:
            bad.append((r.name, r.samples.shape[0], got_row, row))
            continue
        if seg is not None:
            assert [int(g[k]) for k in ("start", "leader", "adapter", "polya", "cliffs")] == [int(v) for v in seg], r.name
            assert np.float64(g["read_rate"]).tobytes() == np.float64(rl[0]).tobytes(), r.name
            assert np.float64(g["polya_length"]).tobytes() == np.float64(rl[1]).tobytes(), r.name
            assert int(g["qc"]) == qc, r.name
    assert not bad, f"{len(bad)} of {len(reads)} rows differ, first: {bad[:3]}"
    return got


def test_edge_reads(eng, ref):
    rng = np.random.default_rng(11)
    _compare(eng, ref, pc.edge_reads(rng))


def test_synthetic_direct_rna_reads(eng, ref):
    rng = np.random.default_rng(12)
    reads = [pc.synth_read(rng, f"syn_{i}", int(rng.integers(1000, 40000)), pos=i) for i in range(200)]
    got = _compare(eng, ref, reads)
    assert (got["qc"] == polya.QC_TAGS.index("PASS")).sum() > 0


def test_batch_of_long_and_short_reads(eng, ref):
    """2 000 reads of 10^3 .. 3*10^5 samples (log-uniform) in one call, launched longest first"""
    rng = np.random.default_rng(13)
    lens = np.exp(rng.uniform(np.log(1e3), np.log(3e5), 2000)).astype(np.int64)
    reads = [pc.synth_read(rng, f"b_{i}", int(n), cliffs=0.001) for i, n in enumerate(lens)]
    _compare(eng, ref, reads)


def test_failed_loads_in_one_batch(eng, ref):
    """reads missing from the index (loaded = 0) and reads whose events load_from_raw cleared (n_events = 0) give
    READ_FAILED_LOAD rows between computed ones"""
    rng = np.random.default_rng(14)
    reads = [pc.synth_read(rng, f"m_{i}", 5000) for i in range(12)]
    for r in reads[1::4]:
        r.loaded = False
    _compare(eng, ref, reads)
    cleared = reads[2::4]
    for r in cleared:
        r.duration = np.zeros(0, np.float32)
        r.map_start[:] = -1; r.map_stop[:] = -1
    raw, jobs, dur, b2e = pc.pack(reads)
    got = eng.polya_batch(raw, jobs, dur, b2e)
    for r, g in zip(reads, got):
        failed = (not r.loaded) or r.duration.shape[0] == 0
        assert (int(g["qc"]) == polya.READ_FAILED_LOAD) == failed, r.name


def test_refused_inputs(eng):
    rng = np.random.default_rng(15)
    r = pc.synth_read(rng, "one_sample", 1)
    raw, jobs, dur, b2e = pc.pack([r])
    with pytest.raises(_lib.NphError):
        eng.polya_batch(raw, jobs, dur, b2e)
    r = pc.synth_read(rng, "bad_map", 500)
    r.map_start[3], r.map_stop[3] = 2, 1
    raw, jobs, dur, b2e = pc.pack([r])
    with pytest.raises(_lib.NphError):
        eng.polya_batch(raw, jobs, dur, b2e)
    r = pc.synth_read(rng, "map_past_events", 500)
    r.map_start[3], r.map_stop[3] = 0, r.duration.shape[0]
    raw, jobs, dur, b2e = pc.pack([r])
    with pytest.raises(_lib.NphError):
        eng.polya_batch(raw, jobs, dur, b2e)
    # a read that failed to load is not computed, so it is not checked either
    r = pc.synth_read(rng, "unloaded_one_sample", 1)
    r.loaded = False
    raw, jobs, dur, b2e = pc.pack([r])
    got = eng.polya_batch(raw, jobs, dur, b2e)
    assert int(got[0]["qc"]) == polya.READ_FAILED_LOAD


def test_libm_exact_on_device_every_float():
    """the device build of csrc/libm_exact.cuh equals this machine's host expf / logf on every float of their domains"""
    exe = os.path.join(ROOT, "build", "checks", "check_libm_exact")
    r = subprocess.run([exe, "--device"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "expf: 0 bad, logf: 0 bad" in r.stdout
