"""The CUDA event detector against the port oracle on every edge read of tests/events_cases.py, bit for bit, under every
parameter set and every forced warps-per-read and warm-up, in one mixed-length batch; and the path each read took.
NPH_EVENTS_STATS makes the library report the repair walks, the reads sent to the streaming fallback and how many of those
the fused kernel refused (guard or slice); each must equal what events_cases.predict restates for the batch, so a kernel
that reaches the right events by another path fails too.  Also: the warps-per-read heuristic, capacity at and below the
event count, refused parameters, and ADC-quantised traces up to 2^20 samples on the fast path."""
import re

import numpy as np
import pytest
import torch

from nanopolish_b200 import synth
from tests import events_cases as ec
from tests.test_gpu_events import _same

pytestmark = pytest.mark.gpu
NPH_ERR_UNSUPPORTED = -6


@pytest.fixture(scope="module")
def edges(port_oracle):
    reads = ec.edge_reads()
    _, _, preds = ec.check_edges(port_oracle, reads)
    raw, rr = ec.batch(reads)
    return reads, raw, rr, preds


def _run(engine, capfd, monkeypatch, raw, rr, prm, env):
    for k in ("NPH_EVENTS_WPR", "NPH_EVENTS_WARMUP", "NPH_EVENTS_FORCE_STREAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in {**env, "NPH_EVENTS_STATS": "1"}.items():
        monkeypatch.setenv(k, v)
    capfd.readouterr()
    got = engine.detect_events_batch(raw, rr, prm)
    err = capfd.readouterr().err
    m = re.search(r"repair walks (\d+)\s+streaming fallback (\d+) \(guard/slice (\d+)\)", err)
    assert m, err
    return got, tuple(int(v) for v in m.groups())


@pytest.mark.parametrize("config", ec.CONFIGS, ids=lambda c: f"wpr{c[0]}-warm{c[1]}")
def test_edge_reads_bit_exact_on_the_predicted_path(engine, port_oracle, edges, capfd, monkeypatch, config):
    reads, raw, rr, preds = edges
    wpr, warm = config
    env = {"NPH_EVENTS_WPR": str(wpr)}
    if warm is not None:
        env["NPH_EVENTS_WARMUP"] = warm
    for pname, prm in ec.PARAMS.items():
        got, stats = _run(engine, capfd, monkeypatch, raw, rr, prm, env)
        for r, g in zip(reads, got):
            try:
                _same(g, port_oracle.detect_events(r.x, prm))
            except AssertionError as ex:
                raise AssertionError(f"{r.name} under {pname}: {ex}") from ex
        assert stats == ec.batch_stats(preds, reads, pname, config), f"{pname}: (repair walks, fallback, guard/slice)"


@pytest.mark.parametrize("want", [1, 2, 4])
def test_warps_per_read_heuristic(engine, port_oracle, capfd, monkeypatch, want):
    """without $NPH_EVENTS_WPR the batch size and the longest read choose 1, 2 or 4 warps per read; the repair walks of reads
    with a long plateau depend on the lane count, so the stats show which one ran"""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    longest = {1: 12000, 2: 20000, 4: 40000}[want]
    assert ec.heuristic_wpr(3, longest, sm) == want
    reads = []
    for i, n in enumerate((longest, 9000, 5000)):
        x = ec._steps(n, 70 + i)
        x[n // 8:] = np.float32(91.5)
        reads.append(ec.EdgeRead(f"plateau-{n}", x, frozenset()))
    raw, rr = ec.batch(reads)
    prm = ec.PARAMS["dna"]
    got, stats = _run(engine, capfd, monkeypatch, raw, rr, prm, {})
    want_rep = 0
    for r, g in zip(reads, got):
        _same(g, port_oracle.detect_events(r.x, prm))
        pr = ec.predict(ec.Trace(port_oracle, r.x, prm), 32 * want, ec.FUSED_WARM, ec.room(r.x.shape[0]))
        assert pr.path == "fast"
        want_rep += pr.repairs
    others = [sum(ec.predict(ec.Trace(port_oracle, r.x, prm), 32 * w, ec.FUSED_WARM, ec.room(r.x.shape[0])).repairs for r in reads)
              for w in (1, 2, 4) if w != want]
    assert want_rep not in others
    assert stats == (want_rep, 0, 0)


@pytest.mark.parametrize("wpr", ["1", "2", "4"])
def test_capacity(engine, port_oracle, capfd, monkeypatch, wpr):
    """event_cap equal to the event count succeeds (on the path the restatement predicts: a room that tight crowds some lane's
    slice), one less is refused; a room below one boundary per lane (R = 0) comes back exact through the fallback; a read without
    a boundary fits event_cap = 1 on the fast path"""
    from nanopolish_b200._lib import NphError
    prm = ec.PARAMS["dna"]
    x = ec._steps(6000, 5)
    want = port_oracle.detect_events(x, prm)
    ne = want.shape[0]
    rd = np.zeros(1, synth.RAW_READ_DT)
    rd[0] = (0, 0, 6000, ne)
    got, stats = _run(engine, capfd, monkeypatch, x, rd, prm, {"NPH_EVENTS_WPR": wpr})
    _same(got[0], want)
    pr = ec.predict(ec.Trace(port_oracle, x, prm), 32 * int(wpr), ec.FUSED_WARM, ne)
    assert stats == (pr.repairs, int(pr.path != "fast"), int(pr.path != "fast"))
    rd[0] = (0, 0, 6000, ne - 1)
    with pytest.raises(NphError):
        engine.detect_events_batch(x, rd, prm)
    # R = 0: room for the events, fewer than one boundary per lane
    x = ec._steps(100, 6, dwell=5.0)
    want = port_oracle.detect_events(x, prm)
    ne = want.shape[0]
    assert 1 < ne < 32
    rd[0] = (0, 0, 100, ne)
    got, stats = _run(engine, capfd, monkeypatch, x, rd, prm, {"NPH_EVENTS_WPR": wpr})
    _same(got[0], want)
    assert stats[1:] == (1, 1)
    rd[0] = (0, 0, 100, ne - 1)
    with pytest.raises(NphError):
        engine.detect_events_batch(x, rd, prm)
    # no boundary: one event in a room of one
    flat = np.full(3000, 77.25, np.float32)
    rd[0] = (0, 0, 3000, 1)
    got, stats = _run(engine, capfd, monkeypatch, flat, rd, prm, {"NPH_EVENTS_WPR": wpr})
    _same(got[0], port_oracle.detect_events(flat, prm))
    assert got[0].shape[0] == 1 and stats[1] == 0


@pytest.mark.parametrize("w1,w2", [(0, 6), (0, 0), (7, 6), (15, 14), (3, 17), (17, 17)])
def test_refused_windows(engine, w1, w2):
    from nanopolish_b200._lib import NphError
    x = ec._steps(1000, 1)
    rd = np.zeros(1, synth.RAW_READ_DT)
    rd[0] = (0, 0, 1000, ec.room(1000))
    with pytest.raises(NphError) as ex:
        engine.detect_events_batch(x, rd, ec.params(w1, w2))
    assert ex.value.status == NPH_ERR_UNSUPPORTED


@pytest.mark.parametrize("rna", [False, True])
def test_adc_quantised_traces_take_the_fast_path(engine, port_oracle, capfd, monkeypatch, rna):
    """real raw current, (adc + offset) * range / digitisation at 40-250 pA, passes the guard up to 2^20 samples"""
    reads = [ec.EdgeRead(f"adc-{n}", ec.adc(n, 800 + n, noise=1.5 if n % 2 else 0.0), frozenset())
             for n in (1 << 20, (1 << 20) - 1, 300000, 65536, 4097)]
    raw, rr = ec.batch(reads)
    prm = synth.event_params(rna)
    for r in reads:
        g = ec.guard(r.x)
        assert g.exact and r.x.min() >= 40 and r.x.max() <= 250
    got, stats = _run(engine, capfd, monkeypatch, raw, rr, prm, {})
    for r, g in zip(reads, got):
        _same(g, port_oracle.detect_events(r.x, prm))
    assert stats[1:] == (0, 0)
