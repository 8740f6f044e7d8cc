"""Pin the port oracle's event detector (npo_detect_events, oracle/np_oracle.c) to the compiled scrappie on every edge read of
tests/events_cases.py under every parameter set: identical starts, bit-identical length, mean and stdv.  The builders' edge
claims are checked on the oracle's run here too, and the coverage table goes to the test log.

The reference's answers live in tests/golden/ref_events_edges.pkl.xz, one row per (read, parameter set): a fingerprint of
the samples and parameters, and a hash of the events (a ref_calls.CaseRecord: asked live where oracle/_ref/libnpref.so exists
and exports npref_detect_events_params and compared with the record, replayed elsewhere).  A read without any boundary never
goes to the reference (create_events reads peaks[-1] there); the port's one-event answer for it is compared with the device
only.  NPH_REF_CASES_RECORD=<dir> pytest tests/test_events_edges_oracle.py writes a new record to <dir>."""
import os
import re

import pytest

from tests import events_cases as ec
from tests import ref_calls

KERNEL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nanopolish_b200", "csrc", "event_detect.cu")

reference = ref_calls.case_fixture("ref_events_edges.pkl.xz", needs=("npref_detect_events_params",))


@pytest.fixture(scope="module")
def reads():
    return ec.edge_reads()


def test_kernel_constants():
    """the constants, templated window pairs, lane geometry, slice size, warps-per-read rule and guard events_cases.py restates
    are event_detect.cu's"""
    src = open(KERNEL).read()
    assert re.search(r"constexpr int kFusedMaxW2 = (\d+);", src).group(1) == str(ec.FUSED_MAX_W2)
    assert re.search(r"constexpr int kMaxW2 = (\d+);", src).group(1) == str(ec.MAX_W2)
    assert re.search(r"constexpr int kPeakWarps = (\d+);", src).group(1) == str(ec.PEAK_WARPS)
    assert re.search(r"constexpr uint32_t kFusedWarm = (\d+);", src).group(1) == str(ec.FUSED_WARM)
    pairs = tuple((int(a), int(b)) for a, b in re.findall(r"f\.w1 == (\d+) && f\.w2 == (\d+)\) kern = ed_fused_kernel<\1, \2, WPR>", src))
    assert pairs == ec.TEMPLATED
    assert "const uint32_t seg = ((n + LANES - 1) / LANES + 31) / 32 * 32;" in src
    assert "const uint32_t b0 = (unsigned long long)gl * seg < n ? gl * seg : n, b1 = min(n, b0 + seg);" in src
    assert "const uint32_t a0 = b0 > p.warm ? b0 - p.warm : 0;" in src
    assert "const uint32_t cap_peaks = rd.event_cap ? rd.event_cap - 1 : 0;" in src and "const uint32_t R = cap_peaks / LANES;" in src
    assert "const size_t want = (size_t)ctx->sm_count * 20;" in src
    assert "while (wpr < 4 && n_reads * wpr < want && n_samples[order[0]] / (64u * wpr) >= 2 * p.warm) wpr *= 2;" in src
    assert "((uint32_t)atoi(getenv(\"NPH_EVENTS_WARMUP\")) + 31u) / 32u * 32u : kFusedWarm" in src
    assert "while ((1ull << lg) < (unsigned long long)n + 1) ++lg;" in src
    assert "evn >= 97 && evx <= 157 && lg + evx + 24 - evn <= 53" in src
    assert "eqn >= 66 && eqx <= 188 && lg + eqx + 24 - eqn <= 53" in src
    assert "if (params->window_length2 > kMaxW2 || params->window_length1 > params->window_length2 || params->window_length1 == 0)" in src


def test_lane_geometry():
    """every lane's owned range tiles [0, n) in segments that are multiples of 32, and lanes past the end own nothing"""
    for lanes in (32, 64, 128):
        for n in list(range(1, 300)) + [32 * lanes * k + d for k in (1, 2, 3) for d in (-1, 0, 1)]:
            r = ec.lane_ranges(n, lanes, ec.FUSED_WARM)
            seg = ec.seg_len(n, lanes)
            assert seg % 32 == 0 and seg * lanes >= n and len(r) <= lanes
            assert r[0][1] == 0 and r[-1][2] == n and all(r[i][2] == r[i + 1][1] for i in range(len(r) - 1))
            assert all(b0 % 32 == 0 and (b0 - a0) % 32 == 0 and b0 - a0 <= ec.FUSED_WARM for a0, b0, _ in r)


def test_sample_span_binds_only_past_2_27_samples():
    """the guard's sample span can be 53 with the square span passing only at ceil(log2(n + 1)) = 28 or 29 (reads of 2^27 samples
    or more): below that the square span binds first, so the span-53 and span-54 reads are built on the squares"""
    for lg in range(1, 33):
        ok = False
        for d in range(0, 40):                      # biased-exponent range of |x|: the squares' range is then 2d - 1 or more
            if lg + d + 24 == 53 and lg + max(2 * d - 1, 0) + 24 <= 53:
                ok = True
        assert ok == (28 <= lg <= 29), lg


def test_events_edges_match_reference(reads, reference, port_oracle):
    cases = [(pname, prm, r) for pname, prm in ec.PARAMS.items() for r in reads]
    mine = []
    for pname, prm, r in cases:
        ev = port_oracle.detect_events(r.x, prm)
        mine.append(None if ev.shape[0] == 1 else ec.events_hash(ev["start"], ev["length"], ev["mean"], ev["stdv"]))
    got = reference.answers("events_edges", [ec.fingerprint(r.x, prm) for _, prm, r in cases],
                            lambda i: ec.events_hash(*reference.live.detect_events_params(cases[i][2].x, cases[i][1])),
                            skip={i: None for i, m in enumerate(mine) if m is None})
    for (pname, prm, r), m, g in zip(cases, mine, got):
        assert m == g, f"{r.name} under {pname}: the port's events differ from scrappie's"
    assert sum(m is not None for m in mine) > 1000


def test_builders_reach_every_edge(port_oracle):
    cover, claimed, preds = ec.check_edges(port_oracle)
    print("\n" + ec.coverage_table(cover, claimed))
    missing = sorted((w, c, k) for w, c, k in claimed if k not in cover[(w, c)])
    assert not missing, f"claimed cells without a read: {missing}"
    paths = {p.path for p in preds.values()}
    assert paths == {"fast", "guard", "slice", "wide"}
