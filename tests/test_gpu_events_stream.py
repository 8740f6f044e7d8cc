"""The streaming fallback of the CUDA event detector (detect_events_stream_kernel) at its edges: ragged and degenerate
lengths, DNA and RNA parameters, windows wider than the fused kernel stages, and a signal without any boundary.  Every
read must come back with the oracle's boundaries and bit-identical length / mean / stdv.  NPH_EVENTS_STATS makes the
library report how many reads took the fallback, so each test also checks that the fallback, and not the fast path, ran."""
import re

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests.test_gpu_events import _same

pytestmark = pytest.mark.gpu

LENS = [1, 2, 5, 6, 11, 12, 13, 25, 100, 3333, 20000]


def _ragged(lens, seed):
    rng = np.random.default_rng(seed)
    raws, reads, so, eo = [], np.zeros(len(lens), synth.RAW_READ_DT), 0, 0
    for i, n in enumerate(lens):
        x = (90 + 12 * np.sign(np.sin(np.arange(n) / 7.0)) + rng.standard_normal(n)).astype(np.float32)
        raws.append(x); reads[i] = (so, eo, n, n + 2); so += n; eo += n + 2
    return np.concatenate(raws), reads


def _detect_on_fallback(engine, capfd, raw, reads, prm):
    capfd.readouterr()
    got = engine.detect_events_batch(raw, reads, prm)
    m = re.search(r"streaming fallback (\d+)", capfd.readouterr().err)
    assert m and int(m.group(1)) == reads.shape[0]
    return got


def _check(got, raw, reads, prm, port_oracle):
    for r, g in zip(reads, got):
        x = np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])])
        _same(g, port_oracle.detect_events(x, prm))


def _params(w1, w2, t1, t2, ph):
    p = synth.event_params(False)
    p[0] = (w1, w2, t1, t2, ph, 0)
    return p


@pytest.mark.parametrize("rna", [False, True])
def test_forced_fallback_on_ragged_and_degenerate_lengths(engine, port_oracle, monkeypatch, capfd, rna):
    monkeypatch.setenv("NPH_EVENTS_FORCE_STREAM", "1")
    monkeypatch.setenv("NPH_EVENTS_STATS", "1")
    raw, reads = _ragged(LENS, 9)
    prm = synth.event_params(rna)
    _check(_detect_on_fallback(engine, capfd, raw, reads, prm), raw, reads, prm, port_oracle)


@pytest.mark.parametrize("w1,w2,t1,t2,ph", [(7, 15, 2.5, 9.0, 1.0), (8, 16, 2.5, 9.0, 1.0), (3, 16, 1.4, 9.0, 0.2),
                                             (1, 15, 1.4, 9.0, 0.2), (16, 16, 2.5, 9.0, 1.0)])
def test_windows_wider_than_the_fused_kernel_take_the_fallback(engine, port_oracle, monkeypatch, capfd, w1, w2, t1, t2, ph):
    """w2 > 14 sends every read down the fallback without any knob."""
    monkeypatch.setenv("NPH_EVENTS_STATS", "1")
    nuc = synth.load_model("nucleotide")
    sraw, sreads = synth.gen_raw(4, 9000, nuc, seed=31, mean_dwell=30.0)
    raw, reads = _ragged(LENS, 10)
    reads["sample_off"] += sraw.shape[0]
    reads["event_off"] += int(sreads["event_off"][-1] + sreads["event_cap"][-1])
    raw, reads = np.concatenate([sraw, raw]), np.concatenate([sreads, reads])
    prm = _params(w1, w2, t1, t2, ph)
    got = _detect_on_fallback(engine, capfd, raw, reads, prm)
    _check(got, raw, reads, prm, port_oracle)
    assert all(g.shape[0] > 10 for g in got[:4])                       # the synthetic reads do have boundaries


@pytest.mark.parametrize("env,prm", [({"NPH_EVENTS_FORCE_STREAM": "1"}, synth.event_params(False)),
                                     ({"NPH_EVENTS_FORCE_STREAM": "1"}, synth.event_params(True)),
                                     ({}, _params(8, 16, 2.5, 9.0, 1.0))])
def test_constant_signal_on_the_fallback_is_one_event(engine, port_oracle, monkeypatch, capfd, env, prm):
    for k, v in {**env, "NPH_EVENTS_STATS": "1"}.items():
        monkeypatch.setenv(k, v)
    flat = np.full(500, 80.0, np.float32)
    rd = np.zeros(1, synth.RAW_READ_DT); rd[0] = (0, 0, 500, 16)
    got = _detect_on_fallback(engine, capfd, flat, rd, prm)
    _check(got, flat, rd, prm, port_oracle)
    g = got[0]
    assert g.shape[0] == 1 and g["start"][0] == 0 and g["length"][0] == 500.0 and g["mean"][0] == 80.0 and g["stdv"][0] == 0.0
