"""Pin the port oracle's trim and calibration (npo_trim_raw, npo_recalibrate in oracle/np_oracle.c) to the compiled reference on
every edge case of tests/prep_cases.py: the trimmed range and every chunk's MAD with the threshold (scrappie's own madf and
quantilef through npref_trim_mads), and shift, scale, drift, var and events_per_base bit for bit with the 'M'-event count and
the calibrated flag (get_eventalignment_for_1d_basecalls + recalibrate_model through npref_calibrate, custom models).  The
builders' edge claims are checked on the oracle's traces here too, and the coverage tables go to the test log.

The reference's answers live in tests/golden/ref_prep_edges.pkl.xz: per case a fingerprint of the inputs and hashes of the
answers.  Where oracle/_ref/libnpref.so exists and exports npref_trim_mads the reference is called live; elsewhere the record
is replayed.  Trim cases the reference asserts or wraps on (see prep_cases.trim_deviations) are never sent to it.
NPH_REF_PREP_RECORD=<path> pytest tests/test_prep_edges_oracle.py writes a new record."""
import os
import re

import numpy as np
import pytest

from oracle.oracle_py import RefOracle
from tests import prep_cases as pc
from tests import ref_calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_prep_edges.pkl.xz")
PREP = os.path.join(ROOT, "nanopolish_b200", "csrc", "squiggle_prep.cu")
LFR = os.path.join(ROOT, "nanopolish_b200", "csrc", "load_from_raw.cu")


@pytest.fixture(scope="module")
def reference():
    """(live RefOracle or None, recorded answers, record path or None)"""
    path = os.environ.get("NPH_REF_PREP_RECORD")
    live = RefOracle() if RefOracle.available() else None
    if live is not None and not live.has("npref_trim_mads"):
        live = None                 # a library built from an older harness, without the entry point: replay the record
    if path and live is None:
        pytest.fail("NPH_REF_PREP_RECORD needs the compiled reference with npref_trim_mads (oracle/_ref/libnpref.so)")
    rec = {} if path else ref_calls.load(GOLDEN)
    yield live, rec, path
    if path:
        ref_calls.save(rec, path)


def test_kernel_constants():
    """the constants, grids, QC thresholds, event room and hard-coded trim prep_cases.py restates are the sources'"""
    src, lfr = open(PREP).read(), open(LFR).read()
    assert re.search(r"constexpr int kTrimThreads = (\d+);", src).group(1) == str(pc.TRIM_THREADS)
    assert re.search(r"constexpr int kMaxChunk = (\d+);", src).group(1) == str(pc.MAX_CHUNK)
    assert re.search(r"constexpr int kCalWarps = (\d+);", src).group(1) == str(pc.CAL_WARPS)
    assert re.search(r"constexpr int kConvWarps = (\d+);", lfr).group(1) == str(pc.CONV_WARPS)
    assert "trim_kernel<<<(unsigned)std::min<size_t>(n_reads, (size_t)ctx->sm_count * 8), kTrimThreads" in src
    assert "std::min<size_t>((args.n_jobs + kCalWarps - 1) / kCalWarps, (size_t)ctx->sm_count * 8)" in src
    assert "std::min<size_t>((nl + kConvWarps - 1) / kConvWarps, (size_t)ctx->sm_count * 8), kConvWarps * 32" in lfr
    assert "for (int k0 = 0; k0 < nk; k0 += 32)" in src                                  # the 32-k-mer tile
    assert f"if (n_used < {pc.MIN_M})" in src
    assert f"if (var > {pc.MAX_VAR})" in src and f"else if (cal.events_per_base > {pc.MAX_EPB})" in src
    assert "if (mad[i] > thresh)" in src
    assert "rank += (o < me || (o == me && j < i)) ? 1u : 0u;" in src
    assert "x4[s] = (lane + 32 * s < p.chunk) ? xc[lane + 32 * s] : inf;" in src
    assert "ns / 2 + 8" in lfr and "n_samples / 2 + 8" in lfr
    ts, te, ch, perc = pc.LFR_TRIM
    assert f"nph_trim_device(ctx, d_raw, n_samples_total, rr.data(), n_jobs, {ts}, {te}, {ch}, {perc}f, arena, range.data())" in lfr
    assert f"nph_trim_scratch_bytes(rr.data(), n_jobs, {ch})" in lfr
    for n, sm in ((1, 132), (1056, 132), (1057, 132)):
        assert pc.trim_grid(n, sm) == min(n, 1056)


def test_trim_edges_match_reference(reference, port_oracle):
    live, record, path = reference
    want_rows = None if path else record.get("trim")
    assert path or want_rows is not None, f"no recorded reference answers ({GOLDEN}); re-record"
    cases = pc.trim_cases()
    rows, n_ref = [], 0
    for i, c in enumerate(cases):
        t = pc.TrimTrace(port_oracle, c)
        fp = pc.fingerprint(c.x, *c.params)
        if not t.ref_ok(c):
            rows.append((fp, None, None))
            continue
        mine = (pc.range_hash(t.ok, t.start, t.end), pc.mads_hash(t.mads, t.thresh))
        if live is not None:
            ok, s, e = live.trim_raw(c.x, *c.params)
            mads, thr = live.trim_mads(c.x, c.chunk, c.perc)
            got = (pc.range_hash(ok, s, e), pc.mads_hash(mads, thr))
            assert np.array_equal(mads.view(np.uint32), t.mads.view(np.uint32)), f"{c.name}: MADs differ from scrappie's"
        else:
            fp_w, *got = want_rows[i]
            assert fp_w == fp, f"{c.name}: inputs differ from the recorded ones; re-record"
            got = tuple(got)
        rows.append((fp, *got))
        assert mine == got, f"{c.name}: the port's trim differs from scrappie's"
        n_ref += 1
    if path:
        record["trim"] = rows
    elif live is not None and want_rows is not None:
        assert want_rows == rows, "the compiled reference's answers differ from the record"
    assert n_ref >= len(cases) - len(pc.trim_deviations(cases, {c.name: pc.TrimTrace(port_oracle, c) for c in cases}))
    assert n_ref > 150


def _ref_cal(live, c, handles):
    key = id(c.model)
    if key not in handles:
        handles[key] = live.custom_model(c.model)
    mh = handles[key]
    live.clear_reads()
    rh = live.register_reads(c.read(), c.ev_mean, np.arange(c.ev_mean.shape[0], dtype=np.float64), mh)
    w = live.calibrate(rh[0], mh, c.seq(), np.stack([c.pairs["ref_pos"], c.pairs["read_pos"]], 1))
    return "no-alignment" if w is None else pc.cal_hash(w["shift"], w["scale"], w["drift"], w["var"], w["events_per_base"],
                                                         w["n_used"], w["calibrated"])


def port_cal_hash(cal, n_pairs):
    if n_pairs == 0:
        return "no-alignment"
    return pc.cal_hash(cal["shift"], cal["scale"], cal["drift"], cal["var"], cal["events_per_base"], cal["n_used"],
                       int(cal["n_used"]) >= pc.MIN_M)


def test_calibration_edges_match_reference(reference, port_oracle):
    live, record, path = reference
    want_rows = None if path else record.get("cal")
    assert path or want_rows is not None, f"no recorded reference answers ({GOLDEN}); re-record"
    rows, handles = [], {}
    for i, c in enumerate(pc.cal_cases()):
        t = pc.CalTrace(port_oracle, c)
        fp = pc.cal_fingerprint(c)
        mine = port_cal_hash(t.cal, c.pairs.shape[0])
        if live is not None:
            got = _ref_cal(live, c, handles)
        else:
            fp_w, got = want_rows[i]
            assert fp_w == fp, f"{c.name}: inputs differ from the recorded ones; re-record"
        rows.append((fp, got))
        assert mine == got, f"{c.name}: the port's calibration differs from the reference's ({t.cal})"
    if path:
        record["cal"] = rows
    elif live is not None and want_rows is not None:
        assert want_rows == rows, "the compiled reference's answers differ from the record"


def test_builders_reach_every_edge(port_oracle):
    cover, traces = pc.check_trim_edges(port_oracle)
    print("\n" + pc.coverage_table(cover, "trim"))
    cases = pc.trim_cases()
    print("trim cases compared device against port only:", ", ".join(pc.trim_deviations(cases, traces)))
    assert not [k for k, v in cover.items() if not v]
    cover, _ = pc.check_cal_edges(port_oracle)
    print(pc.coverage_table(cover, "calibration"))
    assert not [k for k, v in cover.items() if not v]


def test_the_tie_matters_and_the_unreachable_branch():
    """the pivot-tie case decides on the first-wins rule (restated solve, either pivot); and no chunk count makes
    nextafterf(1, 0) * (n - 1) round up to n - 1 in float, so quantilef's p == 1 branch needs p == 1"""
    c = next(c for c in pc.cal_cases() if c.name == "pivot-tie")
    s = pc.sums_of(c.model.level_mean[c.ranks], c.ev_mean.astype(np.float64))
    assert s[0] == s[2] and pc.lu_solve(*s)[:2] != pc.lu_solve(*s, force=(1, 1))[:2]
    p = np.nextafter(np.float32(1), np.float32(0))
    n = np.arange(2, 1 << 22, dtype=np.int64)
    assert not ((p * (n - 1).astype(np.float32)).astype(np.int64) == n - 1).any()
