"""Parity of the CUDA event detector (scrappie detect_events through the C ABI) with the oracle, which
tests/test_oracle_vs_ref.py pins to scrappie's C source compiled unmodified: identical boundaries, bit-identical
length / mean / stdv."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import events_cases as ec

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rna,n_samples,n_reads", [(False, 36000, 40), (True, 50000, 12), (False, 700, 150)])
def test_events_identical(engine, port_oracle, rna, n_samples, n_reads):
    nuc = synth.load_model("nucleotide")
    raw, reads = synth.gen_raw(n_reads, n_samples, nuc, seed=4000 + n_samples, mean_dwell=30.0 if rna else 9.0)
    prm = synth.event_params(rna)
    got = engine.detect_events_batch(raw, reads, prm)
    for r, g in zip(reads, got):
        x = np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])])
        ec.same(g, port_oracle.detect_events(x, prm))
    assert sum(g.shape[0] for g in got) > n_reads * n_samples / (60 if rna else 25)


def test_ragged_and_degenerate(engine, port_oracle):
    nuc = synth.load_model("nucleotide")
    rng = np.random.default_rng(9)
    lens = [1, 2, 5, 6, 11, 12, 13, 25, 100, 3333, 20000]
    raws, reads, so, eo = [], np.zeros(len(lens), synth.RAW_READ_DT), 0, 0
    for i, n in enumerate(lens):
        x = (90 + 12 * np.sign(np.sin(np.arange(n) / 7.0)) + rng.standard_normal(n)).astype(np.float32)
        raws.append(x); reads[i] = (so, eo, n, n + 2); so += n; eo += n + 2
    raw = np.concatenate(raws)
    prm = synth.event_params(False)
    got = engine.detect_events_batch(raw, reads, prm)
    for r, g in zip(reads, got):
        x = np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])])
        ec.same(g, port_oracle.detect_events(x, prm))
    # constant signal: no peak, one event covering the read
    flat = np.full(500, 80.0, np.float32)
    rd = np.zeros(1, synth.RAW_READ_DT); rd[0] = (0, 0, 500, 16)
    g = engine.detect_events_batch(flat, rd, prm)[0]
    assert g.shape[0] == 1 and g["length"][0] == 500.0 and g["mean"][0] == 80.0 and g["stdv"][0] == 0.0


def test_event_capacity_overflow_is_reported(engine):
    from nanopolish_b200._lib import NphError
    nuc = synth.load_model("nucleotide")
    raw, reads = synth.gen_raw(2, 5000, nuc, seed=1)
    reads = reads.copy(); reads["event_cap"] = 3
    reads["event_off"] = [0, 3]
    with pytest.raises(NphError):
        engine.detect_events_batch(raw, reads, synth.event_params(False))


@pytest.mark.parametrize("env", [{"NPH_EVENTS_WPR": "1"}, {"NPH_EVENTS_WPR": "2"}, {"NPH_EVENTS_WPR": "4"},
                                 {"NPH_EVENTS_WPR": "1", "NPH_EVENTS_WARMUP": "0"}, {"NPH_EVENTS_WPR": "2", "NPH_EVENTS_WARMUP": "0"},
                                 {"NPH_EVENTS_WPR": "4", "NPH_EVENTS_WARMUP": "32"}, {"NPH_EVENTS_FORCE_STREAM": "1"}])
def test_every_walk_of_the_detector_is_exact(engine, port_oracle, monkeypatch, env):
    """The fused kernel's shapes — 1 / 2 / 4 warps per read, no warm-up at all (every segment starts from a wrong state and is re-walked
    from its neighbour's final state until the chain verifies), a short warm-up — and the streaming fallback all return the oracle's events."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    nuc = synth.load_model("nucleotide")
    raw, reads = synth.gen_raw(6, 9000, nuc, seed=77)
    flat = np.full(700, 75.5, np.float32)                                   # no boundary at all: one event
    reads = np.concatenate([reads, np.zeros(1, synth.RAW_READ_DT)])
    reads[-1] = (raw.shape[0], int(reads[-2]["event_off"] + reads[-2]["event_cap"]), 700, 64)
    raw = np.concatenate([raw, flat])
    for rna in (False, True):
        prm = synth.event_params(rna)
        got = engine.detect_events_batch(raw, reads, prm)
        for r, g in zip(reads, got):
            x = np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])])
            ec.same(g, port_oracle.detect_events(x, prm))


def test_samples_the_guard_refuses_take_the_streaming_kernel(engine, port_oracle):
    """Signals whose prefix sums are not provably exact (huge dynamic range, denormals) or outside the range the cached-reciprocal
    divisions are proven for must come back identical too (through detect_events_stream_kernel)."""
    rng = np.random.default_rng(5)
    n = 4000
    base = (90 + 12 * np.sign(np.sin(np.arange(n) / 7.0)) + rng.standard_normal(n)).astype(np.float32)
    wide = base.copy(); wide[::97] *= np.float32(2.0 ** 40)                 # span > 53 bits
    tiny = (base * np.float32(2.0 ** -60)).astype(np.float32)               # squares below 2^-61
    sigs = [wide, tiny, base]
    reads = np.zeros(3, synth.RAW_READ_DT); so = eo = 0
    for i, x in enumerate(sigs):
        reads[i] = (so, eo, n, n + 2); so += n; eo += n + 2
    raw = np.concatenate(sigs)
    prm = synth.event_params(False)
    got = engine.detect_events_batch(raw, reads, prm)
    for r, g in zip(reads, got):
        x = np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])])
        ec.same(g, port_oracle.detect_events(x, prm))
