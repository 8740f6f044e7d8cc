"""The device's trim, calibration and one-call load_from_raw against the port oracle at the edges of tests/prep_cases.py, bit for
bit: every trimmed range, every nph_calibration field, the whole base_to_event_out (ranks no job covers included), the event
arrays and nph_last_trim_ranges; and the device's answers against the compiled reference's recorded hashes
(tests/golden/ref_prep_edges.pkl.xz).  Batch sizes are taken from the device's SM count: blocks that loop over reads, warps that
loop over jobs, and a convert grid that loops over live reads."""
import numpy as np
import pytest
import torch

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from oracle.prep_chain import oracle_chain, squiggle_events
from tests import prep_cases as pc
from tests import ref_calls

pytestmark = pytest.mark.gpu

NPH_ERR_INVALID = -3
NPH_ERR_UNSUPPORTED = -6


@pytest.fixture(scope="module")
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pack(signals):
    reads = np.zeros(len(signals), synth.RAW_READ_DT)
    off = 0
    for i, x in enumerate(signals):
        reads[i] = (off, 0, x.shape[0], 0)
        off += x.shape[0]
    flat = np.concatenate([np.asarray(x, np.float32) for x in signals]) if off else np.zeros(1, np.float32)
    return flat, reads


def _status(fn, *a, **k):
    try:
        fn(*a, **k)
    except NphError as ex:
        return ex.status
    return 0


# ---- trim --------------------------------------------------------------------------------------------------------------
def test_trim_edges_identical(engine, port_oracle):
    cases = pc.trim_cases()
    rec = ref_calls.case_answers("ref_prep_edges.pkl.xz", "trim")
    groups = {}
    for i, c in enumerate(cases):
        groups.setdefault(c.params, []).append(i)
    n_ref = 0
    for prm, idx in groups.items():
        flat, reads = _pack([cases[i].x for i in idx])
        got = engine.trim_raw_batch(flat, reads, *prm)
        for r, i in enumerate(idx):
            c = cases[i]
            t = pc.TrimTrace(port_oracle, c)
            g = (int(got[r]["start"]), int(got[r]["end"]))
            assert g == (t.start, t.end), f"{c.name}: device {g}, port {(t.start, t.end)}"
            fp = pc.fingerprint(c.x, *c.params)
            assert fp in rec, f"{c.name}: inputs differ from the recorded ones"
            want = rec[fp][0]
            if want is not None:
                assert pc.range_hash(g[1] > g[0], *g) == want, f"{c.name}: device range differs from the reference's"
                n_ref += 1
    assert n_ref > 150


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_trim_blocks_loop_over_reads(engine, port_oracle, sm_count, delta):
    """sm_count * 8 - 1, sm_count * 8 and sm_count * 8 + 1 reads: the last block takes a second read and reuses its shared
    s_first, s_last and s_stat; empty reads, reads shorter than a chunk and tie cases are mixed in"""
    n = sm_count * pc.BLOCKS_PER_SM + delta
    rng = np.random.default_rng(70 + delta)
    pool = [c for c in pc.trim_cases() if c.chunk == 101 and c.params[:2] in ((5, 5), (2, 2), (3, 2))]
    signals = []
    for i in range(n):
        k = i % 7
        if k == 0:
            signals.append(np.zeros(0, np.float32))
        elif k == 1:
            signals.append(rng.normal(100, 5, 57).astype(np.float32))
        else:
            signals.append(pool[(i * 5) % len(pool)].x)
    signals[-1] = pool[0].x                         # the read a block takes second is a full one
    flat, reads = _pack(signals)
    got = engine.trim_raw_batch(flat, reads, 3, 2, 101, 0.0)
    for i, x in enumerate(signals):
        ok, s, e = port_oracle.trim_raw(x, 3, 2, 101, 0.0)
        assert (int(got[i]["start"]), int(got[i]["end"])) == (s, e), f"read {i} of {n}"
    assert pc.trim_grid(n, sm_count) == min(n, sm_count * 8)


def test_trim_refusals(engine):
    rng = np.random.default_rng(3)
    x = rng.normal(100, 5, 3000).astype(np.float32)
    flat, reads = _pack([x])
    assert _status(engine.trim_raw_batch, flat, reads, 200, 10, 1, 0.0) == NPH_ERR_INVALID
    assert _status(engine.trim_raw_batch, flat, reads, 200, 10, 129, 0.0) == NPH_ERR_UNSUPPORTED
    assert _status(engine.trim_raw_batch, flat, reads, 200, 10, 128, 0.0) == 0
    for v in (np.nan, np.inf, -np.inf):
        for where in (17, 2999):
            y = flat.copy()
            y[where] = v
            assert _status(engine.trim_raw_batch, y, reads, 200, 10, 100, 0.0) == NPH_ERR_INVALID, (v, where)
    # a non-finite sample outside every read is refused too (the whole buffer is checked)
    y = np.concatenate([flat, np.float32([np.nan])])
    assert _status(engine.trim_raw_batch, y, reads, 200, 10, 100, 0.0) == NPH_ERR_INVALID
    big = np.float32([3.0e38, -3.0e38] * 200)
    assert _status(engine.trim_raw_batch, big, _pack([big])[1], 0, 0, 100, 0.0) == 0


# ---- calibration -------------------------------------------------------------------------------------------------------
def _cal_batch(cases, gap=5):
    """one batch of calibration jobs sharing a model: `gap` ranks no job covers before each job's ranks"""
    reads = np.zeros(len(cases), synth.READ_DT)
    jobs = np.zeros(len(cases), synth.ABEA_JOB_DT)
    res = np.zeros(len(cases), synth.ABEA_RES_DT)
    ev, ranks, pairs = [], [], []
    eo = ro = po = 0
    for j, c in enumerate(cases):
        r = c.read()[0]
        r["event_off"] = eo
        reads[j] = r
        ranks.append(np.zeros(gap, np.uint32))
        ro += gap
        rk = c.ranks
        jobs[j] = (ro, po, j, rk.shape[0], max(c.pairs.shape[0], 1), 0)
        res[j]["n_pairs"] = c.pairs.shape[0]
        ev.append(c.ev_mean)
        ranks.append(rk)
        pairs.append(c.pairs)
        pairs.append(np.zeros(max(c.pairs.shape[0], 1) - c.pairs.shape[0], synth.PAIR_DT))
        eo += c.ev_mean.shape[0]
        ro += rk.shape[0]
        po += max(c.pairs.shape[0], 1)
    ranks.append(np.zeros(gap, np.uint32))
    return (reads, np.concatenate(ev).astype(np.float32), np.concatenate(ranks).astype(np.uint32), jobs,
            np.concatenate(pairs), res)


def _by_model(cases):
    groups = {}
    for i, c in enumerate(cases):
        groups.setdefault(id(c.model), []).append(i)
    return groups.values()


def _check_cal_job(c, t, b2e_dev, cal_dev, ref_hash):
    n = c.n_kmers
    assert b2e_dev.tobytes() == t.b2e.tobytes(), f"{c.name}: base_to_event_map differs"
    for f in ("shift", "scale", "drift", "var", "events_per_base"):
        assert np.float64(cal_dev[f]).view(np.uint64) == np.float64(t.cal[f]).view(np.uint64), f"{c.name}: {f} {cal_dev[f]!r} != {t.cal[f]!r}"
    assert (int(cal_dev["n_used"]), int(cal_dev["status"])) == (int(t.cal["n_used"]), int(t.cal["status"])), \
        f"{c.name}: n_used/status {(int(cal_dev['n_used']), int(cal_dev['status']))} != {(int(t.cal['n_used']), int(t.cal['status']))}"
    assert pc.port_cal_hash(cal_dev, c.pairs.shape[0]) == ref_hash, f"{c.name}: device calibration differs from the reference's"
    assert b2e_dev.shape[0] == n


def test_calibration_edges_identical(engine, port_oracle):
    cases = pc.cal_cases()
    rec = ref_calls.case_answers("ref_prep_edges.pkl.xz", "cal")
    for idx in _by_model(cases):
        group = [cases[i] for i in idx]
        mid = engine.model_upload(group[0].model)
        reads, ev, ranks, jobs, pairs, res = _cal_batch(group)
        b2e, cal = engine.recalibrate_batch(reads, ev, ranks, jobs, mid, pairs, res)
        covered = np.zeros(ranks.shape[0], bool)
        for j, i in enumerate(idx):
            c = cases[i]
            fp = pc.cal_fingerprint(c)
            assert fp in rec, f"{c.name}: inputs differ from the recorded ones"
            o, n = int(jobs[j]["rank_off"]), int(jobs[j]["n_kmers"])
            covered[o:o + n] = True
            _check_cal_job(c, pc.CalTrace(port_oracle, c), b2e[o:o + n], cal[j], rec[fp])
        assert (b2e["start"][~covered] == -1).all() and (b2e["stop"][~covered] == -1).all(), "ranks no job covers must be {-1,-1}"


def test_calibration_uncovered_ranks_after_other_work(engine, port_oracle):
    """the align scratch the map is built in holds another call's data first; ranks no job covers still come back {-1,-1}"""
    model = synth.load_model("nucleotide")
    mid = engine.model_upload(model)
    rs = synth.gen_reads(3, 900, model, seed=8)
    jobs, ranks, total = synth.abea_jobs(rs)
    engine.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs, mid, total)
    c = next(c for c in pc.cal_cases() if c.name == "n-used-201")
    reads, ev, rk, jb, pairs, res = _cal_batch([c], gap=4000)
    b2e, cal = engine.recalibrate_batch(reads, ev, rk, jb, engine.model_upload(c.model), pairs, res)
    o, n = int(jb[0]["rank_off"]), int(jb[0]["n_kmers"])
    out = np.ones(rk.shape[0], bool)
    out[o:o + n] = False
    assert (b2e["start"][out] == -1).all() and (b2e["stop"][out] == -1).all()
    _, wc = port_oracle.recalibrate(reads, ev, c.model, rk, jb[0], pairs, c.pairs.shape[0])
    assert cal[0].tobytes() == wc.tobytes()


def test_calibration_warps_loop_over_jobs(engine, port_oracle, sm_count):
    """8 * sm_count * 8 + 1 jobs: a warp takes a second job (and builds its map where another warp's job left its scratch)"""
    base = [c for c in pc.cal_cases() if c.name in ("n-used-200", "n-used-199", "carry-gap", "odd-pairs")]
    base = [c for c in base if c.model is base[0].model]
    n = pc.warp_jobs_loop(sm_count)
    group = [base[i % len(base)] for i in range(n)]
    reads, ev, ranks, jobs, pairs, res = _cal_batch(group, gap=1)
    mid = engine.model_upload(base[0].model)
    b2e, cal = engine.recalibrate_batch(reads, ev, ranks, jobs, mid, pairs, res)
    traces = [pc.CalTrace(port_oracle, c) for c in base]
    assert pc.warp_grid(n, sm_count) == sm_count * 8
    for j in range(n):
        t = traces[j % len(base)]
        o, k = int(jobs[j]["rank_off"]), int(jobs[j]["n_kmers"])
        assert b2e[o:o + k].tobytes() == t.b2e.tobytes(), f"job {j}"
        assert cal[j].tobytes() == t.cal.tobytes(), f"job {j}"


def test_calibration_refusals(engine):
    c = next(c for c in pc.cal_cases() if c.name == "n-used-201")
    mid = engine.model_upload(c.model)
    reads, ev, ranks, jobs, pairs, res = _cal_batch([c, c], gap=0)
    assert _status(engine.recalibrate_batch, reads, ev, ranks, jobs, mid, pairs, res) == 0       # adjacent ranges are fine
    b2e_r, cal_r = engine.recalibrate_batch(reads, ev, ranks, jobs[::-1].copy(), mid, pairs, res[::-1].copy())   # in any order
    assert cal_r[0].tobytes() == cal_r[1].tobytes() and int(cal_r[0]["status"]) == 0
    for shift in (0, 1, int(jobs[1]["rank_off"]) - 1):                                             # any shared rank is refused
        bad = jobs.copy()
        bad[1]["rank_off"] = int(jobs[0]["rank_off"]) + shift
        assert _status(engine.recalibrate_batch, reads, ev, ranks, bad, mid, pairs, res) == NPH_ERR_INVALID, shift
    bad = pairs.copy()
    bad[3]["read_pos"] = int(reads[0]["n_events"])                                                 # a pair outside its read
    assert _status(engine.recalibrate_batch, reads, ev, ranks, jobs, mid, bad, res) == NPH_ERR_INVALID
    b2e, cal = engine.recalibrate_batch(reads, ev, ranks, jobs, mid, pairs, res)                   # the context still works
    assert cal[0].tobytes() == cal[1].tobytes() and int(cal[0]["status"]) == 0


# ---- load_from_raw -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


def _raw_jobs(signals, seqs, k, rates):
    jobs = np.zeros(len(signals), synth.RAW_JOB_DT)
    ranks = []
    soff = roff = 0
    for i, (x, c) in enumerate(zip(signals, seqs)):
        rk = synth.kmer_ranks_from_codes(c, k, 4)
        jobs[i] = (soff, roff, x.shape[0], rk.shape[0], rates[i])
        ranks.append(rk)
        soff += x.shape[0]
        roff += rk.shape[0]
    return np.concatenate(signals).astype(np.float32), np.concatenate(ranks).astype(np.uint32), jobs


def _check_lfr(model, port, signals, seqs, rates, jobs, out, prm):
    off, mean, stdv, start, dur, b2e, cal = out
    covered = np.zeros(b2e.shape[0], bool)
    for i, x in enumerate(signals):
        w = oracle_chain(port, model, [x], [seqs[i]], sample_rate=rates[i], params=prm)[0]
        o, n = int(off[i]), int(off[i + 1] - off[i])
        ro, nk = int(jobs[i]["rank_off"]), int(jobs[i]["n_kmers"])
        if w["events"] is None:
            assert n == 0 and int(cal[i]["status"]) == 17, f"read {i}"
            continue
        ev = w["events"]
        assert n == ev.shape[0], f"read {i}: {n} events, port {ev.shape[0]}"
        assert np.array_equal(mean[o:o + n], ev["mean"]) and np.array_equal(stdv[o:o + n], ev["stdv"]), f"read {i}"
        assert np.array_equal(dur[o:o + n].view(np.uint32), w["duration"].view(np.uint32)), f"read {i}: durations"
        assert np.array_equal(start[o:o + n].view(np.uint64), np.asarray(w["start_time"], np.float64).view(np.uint64)), f"read {i}: start times"
        if "cal" in w:
            assert cal[i].tobytes() == w["cal"].tobytes(), f"read {i}: {cal[i]} != {w['cal']}"
            assert b2e[ro:ro + nk].tobytes() == w["b2e"].tobytes(), f"read {i}: base_to_event_map"
            covered[ro:ro + nk] = True
    assert (b2e["start"][~covered] == -1).all() and (b2e["stop"][~covered] == -1).all()


def _dead(rng, kind):
    return np.full(3000, 77.0, np.float32) if kind == 0 else rng.normal(100, 5, 80).astype(np.float32)


def test_load_from_raw_rates_and_dead_reads(engine, nuc, port_oracle):
    """a different sample rate in every read, reads dead after the trim first, last and at consecutive positions: each live
    read's durations and start times use its own rate"""
    model, mid = nuc
    raw, rr, seqs = synth.gen_raw(6, 5000, model, seed=4100, return_seqs=True)
    live = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])] for r in rr]
    rng = np.random.default_rng(41)
    signals, sq = [], []
    layout = ["d", "l", "l", "d", "d", "l", "l", "d", "l", "l", "d"]
    li = 0
    for k, kind in enumerate(layout):
        if kind == "d":
            signals.append(_dead(rng, k % 2)); sq.append(seqs[0][:40])
        else:
            signals.append(live[li]); sq.append(seqs[li]); li += 1
    rates = [3012.0 + 977.25 * i for i in range(len(signals))]
    flat, ranks, jobs = _raw_jobs(signals, sq, model.k, rates)
    prm = synth.event_params(False)
    out = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm)
    _check_lfr(model, port_oracle, signals, sq, rates, jobs, out, prm)
    kept = engine.last_trim_ranges(len(signals))
    for i, x in enumerate(signals):
        ok, s, e = port_oracle.trim_raw(x)
        assert (int(kept[i]["start"]), int(kept[i]["end"])) == ((s, e) if ok else (0, 0))
    assert (out[6]["status"][[0, 3, 4, 7, 10]] == 17).all() and (out[6]["status"][[1, 2, 5, 6, 8, 9]] != 17).all()


def test_load_from_raw_all_reads_dead(engine, nuc):
    model, mid = nuc
    rng = np.random.default_rng(5)
    signals = [_dead(rng, i % 2) for i in range(5)]
    seqs = [rng.integers(0, 4, 30).astype(np.uint8) for _ in signals]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k, [4000.0] * 5)
    off, mean, stdv, start, dur, b2e, cal = engine.load_from_raw_batch(flat, ranks, jobs, mid, synth.event_params(False))
    assert (off == 0).all() and mean.shape[0] == 0
    assert (cal["status"] == 17).all() and (b2e["start"] == -1).all() and (b2e["stop"] == -1).all()
    assert (engine.last_trim_ranges(5)["end"] == 0).all()


def test_load_from_raw_events_cap(engine, nuc, port_oracle):
    """events_cap equal to the event total works; one below is NPH_ERR_UNSUPPORTED and leaves a working context"""
    model, mid = nuc
    raw, rr, seqs = synth.gen_raw(4, 6000, model, seed=77, return_seqs=True)
    signals = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])] for r in rr]
    rates = [4000.0, 4100.0, 3900.0, 5000.0]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k, rates)
    prm = synth.event_params(False)
    first = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm)
    total = int(first[0][-1])
    at = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm, events_cap=total)
    for a, b in zip(first, at):
        assert a.tobytes() == b.tobytes()
    assert _status(engine.load_from_raw_batch, flat, ranks, jobs, mid, prm, events_cap=total - 1) == NPH_ERR_UNSUPPORTED
    again = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm)
    for a, b in zip(first, again):
        assert a.tobytes() == b.tobytes()
    _check_lfr(model, port_oracle, signals, seqs, rates, jobs, again, prm)


@pytest.mark.parametrize("reverse", [0, 1])
def test_load_from_raw_event_counts_around_the_fold(engine, nuc, port_oracle, reverse):
    """live reads of 1, 2, 3, 31, 32, 33 and 65 events around convert_kernel's 32-event start-time fold, in acquisition order and
    turned around (reverse_events), odd counts included"""
    model, mid = nuc
    prm = synth.event_params(False)
    prm[0]["reverse_events"] = reverse
    rng = np.random.default_rng(9 + reverse)
    signals = [pc.read_with_events(port_oracle, t, prm, t) for t in (2, 3, 31, 32, 33, 65)]
    seqs = [rng.integers(0, 4, max(t, 12) + model.k - 1).astype(np.uint8) for t in (2, 3, 31, 32, 33, 65)]
    rates = [4000.0 + 111.0 * i for i in range(len(signals))]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k, rates)
    out = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm)
    assert [int(v) for v in np.diff(out[0])] == [2, 3, 31, 32, 33, 65]
    _check_lfr(model, port_oracle, signals, seqs, rates, jobs, out, prm)
    # one event per read: thresholds no t-statistic reaches
    quiet = prm.copy()
    quiet[0]["threshold1"] = quiet[0]["threshold2"] = 1e30
    out = engine.load_from_raw_batch(flat, ranks, jobs, mid, quiet)
    assert (np.diff(out[0]) == 1).all()
    _check_lfr(model, port_oracle, signals, seqs, rates, jobs, out, quiet)


def test_load_from_raw_convert_grid_loops(engine, nuc, port_oracle, sm_count):
    """more live reads than convert_kernel's grid has warps (8 * sm_count * 8): warps take a second read"""
    model, mid = nuc
    n = pc.warp_jobs_loop(sm_count) + 3
    prm = synth.event_params(False)
    rng = np.random.default_rng(12)
    protos = [pc.step_read(np.random.default_rng(s), 20 + s) for s in range(5)]
    seqs5 = [rng.integers(0, 4, 30 + model.k - 1).astype(np.uint8) for _ in protos]
    rates5 = [4000.0, 3012.0, 4321.5, 5000.0, 2999.0]
    signals = [protos[i % 5] for i in range(n)]
    seqs = [seqs5[i % 5] for i in range(n)]
    rates = [rates5[(i // 5) % 5] for i in range(n)]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k, rates)
    off, mean, stdv, start, dur, b2e, cal = engine.load_from_raw_batch(flat, ranks, jobs, mid, prm)
    assert pc.warp_grid(n, sm_count, pc.CONV_WARPS) == sm_count * 8
    want = {}
    for i in range(n):
        key = (i % 5, rates[i])
        if key not in want:
            want[key] = oracle_chain(port_oracle, model, [signals[i]], [seqs[i]], sample_rate=rates[i], params=prm)[0]
        w = want[key]
        o, k = int(off[i]), int(off[i + 1] - off[i])
        assert k == w["events"].shape[0] > 0, f"read {i}"
        assert np.array_equal(mean[o:o + k], w["events"]["mean"]), f"read {i}"
        assert np.array_equal(dur[o:o + k], w["duration"]) and np.array_equal(start[o:o + k], w["start_time"]), f"read {i}"
        assert cal[i].tobytes() == w["cal"].tobytes(), f"read {i}"
    d, t = squiggle_events(want[(0, 4000.0)]["events"], 4000.0)
    assert np.array_equal(dur[:int(off[1])], d)


def test_load_from_raw_shared_ranks_refused(engine, nuc):
    model, mid = nuc
    raw, rr, seqs = synth.gen_raw(2, 4000, model, seed=3, return_seqs=True)
    signals = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])] for r in rr]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k, [4000.0, 4000.0])
    prm = synth.event_params(False)
    for ro in (0, 1, int(jobs[1]["rank_off"]) - 1):
        bad = jobs.copy()
        bad[1]["rank_off"] = ro
        bad[1]["n_kmers"] = min(int(jobs[1]["n_kmers"]), ranks.shape[0] - ro)
        assert _status(engine.load_from_raw_batch, flat, ranks, bad, mid, prm) == NPH_ERR_INVALID, ro
    assert _status(engine.load_from_raw_batch, flat, ranks, jobs, mid, prm) == 0
