"""Pin the port oracle's trim and calibration (npo_trim_raw, npo_recalibrate in oracle/np_oracle.c) to the compiled reference on
every edge case of tests/prep_cases.py: the trimmed range and every chunk's MAD with the threshold (scrappie's own madf and
quantilef through npref_trim_mads), and shift, scale, drift, var and events_per_base bit for bit with the 'M'-event count and
the calibrated flag (get_eventalignment_for_1d_basecalls + recalibrate_model through npref_calibrate, custom models).  The
builders' edge claims are checked on the oracle's traces here too, and the coverage tables go to the test log.

The reference's answers live in tests/golden/ref_prep_edges.pkl.xz: per case a fingerprint of the inputs and hashes of the
answers (a ref_calls.CaseRecord: asked live where oracle/_ref/libnpref.so exists and exports npref_trim_mads and
npref_calibrate and compared with the record, replayed elsewhere).  Trim cases the reference asserts or wraps on (see
prep_cases.trim_deviations) are never sent to it.
NPH_REF_CASES_RECORD=<dir> pytest tests/test_prep_edges_oracle.py writes a new record to <dir>."""
import os
import re

import numpy as np

from tests import prep_cases as pc
from tests import ref_calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PREP = os.path.join(ROOT, "nanopolish_b200", "csrc", "squiggle_prep.cu")
LFR = os.path.join(ROOT, "nanopolish_b200", "csrc", "load_from_raw.cu")

reference = ref_calls.case_fixture("ref_prep_edges.pkl.xz", needs=("npref_trim_mads", "npref_calibrate"))


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


def _ref_trim(live, c):
    ok, s, e = live.trim_raw(c.x, *c.params)
    mads, thr = live.trim_mads(c.x, c.chunk, c.perc)
    return pc.range_hash(ok, s, e), pc.mads_hash(mads, thr)


def test_trim_edges_match_reference(reference, port_oracle):
    cases = pc.trim_cases()
    traces = [pc.TrimTrace(port_oracle, c) for c in cases]
    got = reference.answers("trim", [pc.fingerprint(c.x, *c.params) for c in cases], lambda i: _ref_trim(reference.live, cases[i]),
                            skip={i: (None, None) for i, (c, t) in enumerate(zip(cases, traces)) if not t.ref_ok(c)}, flat=True)
    n_ref = 0
    for c, t, g in zip(cases, traces, got):
        if t.ref_ok(c):
            mine = (pc.range_hash(t.ok, t.start, t.end), pc.mads_hash(t.mads, t.thresh))
            assert mine == g, f"{c.name}: the port's trim differs from scrappie's"
            n_ref += 1
    assert n_ref >= len(cases) - len(pc.trim_deviations(cases, {c.name: t for c, t in zip(cases, traces)}))
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


def test_calibration_edges_match_reference(reference, port_oracle):
    cases, handles = pc.cal_cases(), {}
    got = reference.answers("cal", [pc.cal_fingerprint(c) for c in cases], lambda i: _ref_cal(reference.live, cases[i], handles))
    for c, g in zip(cases, got):
        t = pc.CalTrace(port_oracle, c)
        assert pc.port_cal_hash(t.cal, c.pairs.shape[0]) == g, f"{c.name}: the port's calibration differs from the reference's ({t.cal})"


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
