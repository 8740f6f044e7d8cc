"""eventalign.tsv written on the device (nph_eventalign_tsv, csrc/eventalign_tsv.cu) and EventAligner::run_tsv above it.

The expectation is the one tests/test_eventalign.py holds the host writer to: oracle/eventalign_py.py's restatement of
emit_event_alignment_tsv (pinned to the compiled reference and to tests/golden/eventalign_golden.npz) with the same switches, the
golden TSV itself for the switch-free case, and tsv_batch after run() always.  Then the refusals (each a returned status or a
per-read flag, never a device fault), the call-sequence rules of the resident records, and a batch of a few thousand reads.
"""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from oracle import eventalign_py as EP
from tests import eventalign_cases as EC
from tests.test_host_mirror import HOST_SO, _register, _register_reads

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "eventalign_golden.npz")
NPH_ERR_INVALID, NPH_ERR_STATE = -3, -5
NAMES, SCALE, INDEX, SAMPLES = 1, 2, 4, 8            # the switches of nphh_ea_run_tsv / nphh_ea_tsv_all_opt
RATE = 4000.0


@pytest.fixture(scope="module")
def host():
    lib = C.CDLL(HOST_SO)
    lib.nphh_last_error.restype = C.c_char_p
    for f in ("nphh_ea_run", "nphh_ea_run_tsv", "nphh_ea_tsv_all_opt", "nphh_ea_text", "nphh_ea_num_segments"):
        getattr(lib, f).restype = C.c_longlong
    return lib


@pytest.fixture(scope="module")
def cases():
    return EC.build_cases()


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLD)
    return {k: z[k].tobytes().decode() for k in z.files}


@pytest.fixture(scope="module")
def restated(cases, port_oracle):
    model, rs, cs = cases
    return [EP.align_read_to_ref(c["read"], c["contig_name"], c["fetched"], c["ref_pos"], c["flag"], c["cigar"], c["read_idx"],
                                 EC.port_align_fn(port_oracle, rs, model, EC.read_slot(c, rs.n_reads)), *c["region"]) for c in cs]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _raw_samples(slot):
    """the trimmed raw samples SRF_LOAD_RAW_SAMPLES keeps, as tests/test_eventalign.py stands in for them"""
    return np.random.default_rng(900 + slot).normal(90.0, 12.0, 420_000).astype(np.float32)


def _setup(host, cases, samples_of=_raw_samples):
    model, rs, cs = cases
    host.nphh_clear()
    mh = _register(host, model)
    rh = _register_reads(host, rs, mh)
    host.nphh_ea_begin()
    for c in cs:
        slot, r = EC.read_slot(c, rs.n_reads), c["read"]
        a, b = np.ascontiguousarray(r.b2e_start, np.int32), np.ascontiguousarray(c["b2e_stop"], np.int32)
        assert host.nphh_read_set_eventalign(rh[slot], r.name.encode(), r.read_sequence.encode(), _p(a), _p(b), C.c_size_t(a.shape[0]),
                                             _p(np.ascontiguousarray(r.stdv)), _p(np.ascontiguousarray(r.duration))) == 0
        smp = samples_of(slot)
        if smp is not None:
            assert host.nphh_read_set_samples(rh[slot], _p(smp), C.c_size_t(smp.shape[0]), C.c_double(RATE)) == 0
        idx = host.nphh_ea_add_read(rh[slot], c["contig_name"].encode(), c["ref_pos"], c["flag"], c["mapq"], _p(c["cigar"]),
                                    int(c["cigar"].shape[0]), c["fetched"].encode(), c["read_idx"], c["region"][0], c["region"][1])
        assert idx == c["read_idx"], host.nphh_last_error()


def _run_tsv(host, n_reads, switches, cap=1 << 25):
    buf = np.zeros(cap, np.uint8)
    read_off, on_host, batches = np.zeros(n_reads + 1, np.uint64), np.zeros(n_reads, np.uint8), C.c_longlong(0)
    n = host.nphh_ea_run_tsv(C.c_double(1.0), switches, _p(buf), C.c_size_t(cap), _p(read_off), _p(on_host), C.byref(batches))
    assert n >= 0, host.nphh_last_error()
    return buf[:n].tobytes().decode(), read_off, on_host, batches.value


def _host_rows(host, n_reads, switches, cap=1 << 25):
    """run() + tsv_batch: the host writer's bytes and per-read offsets"""
    assert host.nphh_ea_run(C.c_double(1.0)) >= 0, host.nphh_last_error()
    buf, read_off = np.zeros(cap, np.uint8), np.zeros(n_reads + 1, np.uint64)
    n = host.nphh_ea_tsv_all_opt(switches, _p(buf), C.c_size_t(cap), _p(read_off))
    assert n >= 0, host.nphh_last_error()
    return buf[:n].tobytes().decode(), read_off


def _restated_rows(cases, restated, switches):
    model, rs, cs = cases
    return [EP.tsv(c["read"], al, print_read_names=bool(switches & NAMES), scale_events=bool(switches & SCALE),
                   samples=_raw_samples(EC.read_slot(c, rs.n_reads)) if switches & SAMPLES else None, sample_rate=RATE)
            for c, al in zip(cs, restated)]


@pytest.mark.parametrize("switches", [0, NAMES, SCALE, INDEX, SAMPLES, INDEX | SAMPLES, NAMES | SCALE | INDEX | SAMPLES])
def test_device_rows_are_the_reference_rows(host, cases, restated, golden, switches):
    """Forward, reverse-strand, two-segment, windowed and unmapped records over a soft-masked reference with an ambiguity code:
    the device's bytes are the restated reference's, the golden file's, and tsv_batch's."""
    model, rs, cs = cases
    _setup(host, cases)
    got, read_off, on_host, batches = _run_tsv(host, len(cs), switches)
    assert batches == 1 and not on_host.any()                    # every row came from the device
    if switches & (INDEX | SAMPLES) in (0, INDEX | SAMPLES):     # the restatement writes the two sample columns together
        want = _restated_rows(cases, restated, switches)
        assert got == "".join(want)
        assert [got[int(read_off[i]):int(read_off[i + 1])] for i in range(len(cs))] == want
    if switches == 0:
        assert got == "".join(golden[f"tsv_{c['read_idx']}"] for c in cs)          # the compiled reference's bytes
        assert len(got) > 400_000
    # the records are fetched when something asks for them: the host writer then reproduces the device's bytes
    assert host.nphh_ea_num_segments(0) > 0
    _setup(host, cases)
    rows, host_off = _host_rows(host, len(cs), switches)
    assert got == rows and np.array_equal(read_off, host_off)
    host.nphh_ea_begin()


def test_formatter_checks_on_device():
    """"%g" on a strided sample of its domain and its edges, and the eventalign row, through the device copies of tsv_format.cuh"""
    exe = os.path.join(ROOT, "build", "checks", "check_g_format")
    r = subprocess.run([exe, "--device"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_large_windows_take_the_round_driver(host, cases, golden):
    model, rs, cs = cases
    _setup(host, cases)
    os.environ["NPH_EA_EVENT_CAP"] = "150"                       # most windows span ~170 events
    try:
        got, read_off, on_host, batches = _run_tsv(host, len(cs), 0)
    finally:
        del os.environ["NPH_EA_EVENT_CAP"]
    assert batches > 1 and on_host.any()
    assert got == "".join(golden[f"tsv_{c['read_idx']}"] for c in cs)
    assert int(read_off[-1]) == len(got)
    host.nphh_ea_begin()


def test_a_read_with_a_non_finite_stdv_takes_the_host_writer(host, cases, golden):
    model, rs, cs = cases
    bad = [dict(c) for c in cs]
    stdv = cs[1]["read"].stdv.copy()
    stdv[100::200] = np.inf
    bad[1]["read"] = dataclasses.replace(cs[1]["read"], stdv=stdv)
    bad[5]["read"] = bad[1]["read"]                              # the windowed record is built on the same read
    _setup(host, (model, rs, bad))
    got, read_off, on_host, batches = _run_tsv(host, len(cs), 0)
    assert [int(v) for v in on_host] == [0, 1, 0, 0, 0, 1] and batches == 1
    for i in (0, 2, 3):                                           # the other reads are the device's, unchanged
        assert got[int(read_off[i]):int(read_off[i + 1])] == golden[f"tsv_{i}"]
    assert "\tinf\t" in got[int(read_off[1]):int(read_off[2])]
    _setup(host, (model, rs, bad))
    rows, host_off = _host_rows(host, len(cs), 0)
    assert got == rows and np.array_equal(read_off, host_off)
    host.nphh_ea_begin()


def test_run_tsv_reports_a_read_without_samples(host, cases):
    """what tsv_batch raises for such a batch (test_tsv_batch_reports_a_read_without_samples), before anything is launched"""
    _setup(host, cases, samples_of=lambda slot: None if slot == 2 else _raw_samples(slot))
    buf = np.zeros(1 << 20, np.uint8)
    assert host.nphh_ea_run_tsv(C.c_double(1.0), SAMPLES, _p(buf), C.c_size_t(buf.shape[0]), None, None, None) < 0
    assert "--samples" in host.nphh_last_error().decode()
    host.nphh_ea_begin()


# ---- the C ABI on synthetic reads ------------------------------------------------------------------------------------------
def _synth_batch(n_reads, n_events, seed, with_samples):
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(n_reads, n_events, model, seed=seed, drift=True)
    return model, rs, synth.eventalign_tsv_inputs(rs, seed=seed, with_samples=with_samples)


def _chain_run(eng, model, rs):
    mid = eng.model_upload(model)
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    pairs, maps, rf, rr, chains = synth.eventalign_chains(rs, mid)
    results = eng.eventalign_chain_run(pairs, maps, rf, rr, chains)
    assert (results["status"] == 0).all()
    return chains, results


def test_refusals_are_per_read():
    model, rs, inp = _synth_batch(6, 900, 31, True)
    eng = Engine(0)
    try:
        chains, results = _chain_run(eng, model, rs)
        rows = int(results["n_records"].sum())
        text, read_off, refused, row_off = eng.eventalign_tsv(inp, signal_index=True, samples=True, want_row_off=rows)
        assert not refused.any() and int(read_off[-1]) == len(text) == int(row_off[-1]) and text.count(b"\n") == rows
        assert np.array_equal(read_off[:-1], row_off[np.concatenate([[0], np.cumsum(results["n_records"])[:-1]]).astype(np.int64)])
        per_read = [text[int(read_off[i]):int(read_off[i + 1])] for i in range(6)]
        # the records the rows were written from are still there
        rec = eng.eventalign_records_fetch(int((chains["out_off"] + chains["out_cap"]).max()))
        first = rec[int(chains[2]["out_off"])]
        assert per_read[2].split(b"\t", 2)[1] == str(int(first["ref_position"])).encode()
        # read 1 keeps fewer samples than its last events span; read 4 has an event whose stdv is not finite
        bad = dict(inp)
        bad["reads"] = inp["reads"].copy()
        bad["reads"][1]["n_samples"] = 1000
        bad["ev_stdv"] = inp["ev_stdv"].copy()
        bad["ev_stdv"][int(rs.reads[4]["event_off"]) + 300] = np.nan
        text2, off2, refused2, _ = eng.eventalign_tsv(bad, signal_index=True, samples=True)
        assert [int(v) for v in refused2] == [0, 1, 0, 0, 1, 0]
        got = [text2[int(off2[i]):int(off2[i + 1])] for i in range(6)]
        assert got[1] == got[4] == b"" and [got[i] for i in (0, 2, 3, 5)] == [per_read[i] for i in (0, 2, 3, 5)]
        # room one byte short: the status and the size to come back with
        out = np.zeros(len(text) - 1, np.uint8)
        with pytest.raises(NphError) as e:
            eng.eventalign_tsv(inp, signal_index=True, samples=True, out=out)
        assert e.value.status == NPH_ERR_INVALID and str(len(text)) in str(e.value)
    finally:
        eng.close()


def test_rows_need_the_resident_records():
    model, rs, inp = _synth_batch(3, 600, 32, False)
    eng = Engine(0)
    try:
        eng.model_upload(model)
        eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
        with pytest.raises(NphError) as e:                       # no chain run yet
            eng.eventalign_tsv(inp)
        assert e.value.status == NPH_ERR_STATE
        _chain_run(eng, model, rs)
        assert len(eng.eventalign_tsv(inp)[0]) > 0
        jobs = synth.scorereads_jobs(rs, 250)
        eng.hmm_align(jobs.kmer_ranks, jobs.jobs)                # another alignment takes the scratch the records were in
        with pytest.raises(NphError) as e:
            eng.eventalign_tsv(inp)
        assert e.value.status == NPH_ERR_STATE
        with pytest.raises(NphError) as e:
            eng.eventalign_records_fetch(1)
        assert e.value.status == NPH_ERR_STATE
    finally:
        eng.close()


def test_a_batch_of_a_few_thousand_reads(host):
    """3 000 reads of 400 events (about 1.2 million rows): run_tsv's bytes are run() + tsv_batch's, with and without switches"""
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(3000, 400, model, seed=33, drift=True)
    rng = np.random.default_rng(34)
    host.nphh_clear()
    rh = _register_reads(host, rs, _register(host, model))
    one_sample = np.zeros(1, np.float32)

    def queue():
        host.nphh_ea_begin()
        for i in range(rs.n_reads):
            seq = synth._CODE2DNA[rs.seq_codes[i]].tobytes()
            nk = len(seq) - model.k + 1
            cigar = EP.pack_cigar([(len(seq), "M")])
            assert host.nphh_ea_add_read(rh[i], b"chr_synth", 1000 + i, 0, 60, _p(cigar), 1, seq, i, -1, -1) == i, host.nphh_last_error()

    for i in range(rs.n_reads):
        seq = synth._CODE2DNA[rs.seq_codes[i]].tobytes()
        nk = len(seq) - model.k + 1
        start, stop, _ = synth.closest_event_map(rs.ev_kmer[i], nk)
        E = int(rs.reads[i]["n_events"])
        stdv, dur = rng.uniform(0.5, 3.0, E).astype(np.float32), np.full(E, 0.002, np.float32)
        a, b = np.ascontiguousarray(start, np.int32), np.ascontiguousarray(stop, np.int32)
        assert host.nphh_read_set_eventalign(rh[i], f"read_{i}".encode(), seq, _p(a), _p(b), C.c_size_t(nk), _p(stdv), _p(dur)) == 0
        assert host.nphh_read_set_samples(rh[i], _p(one_sample), C.c_size_t(1), C.c_double(RATE)) == 0     # --signal-index reads no sample
    for switches in (0, NAMES | SCALE | INDEX):
        queue()
        got, read_off, on_host, batches = _run_tsv(host, rs.n_reads, switches, cap=1 << 28)
        assert batches == 1 and not on_host.any() and got.count("\n") > 1_000_000
        queue()
        rows, host_off = _host_rows(host, rs.n_reads, switches, cap=1 << 28)
        assert got == rows and np.array_equal(read_off, host_off)
    host.nphh_ea_begin()
