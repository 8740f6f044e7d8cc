"""Pin the port oracle's event detector (npo_detect_events, oracle/np_oracle.c) to the compiled scrappie on every edge read of
tests/events_cases.py under every parameter set: identical starts, bit-identical length, mean and stdv.  The builders' edge
claims are checked on the oracle's run here too, and the coverage table goes to the test log.

The reference's answers live in tests/golden/ref_events_edges.pkl.xz, one entry per (read, parameter set): a fingerprint of
the samples and parameters, and a hash of the events.  Where oracle/_ref/libnpref.so exists and exports
npref_detect_events_params the reference is called live; elsewhere (no library, or one built from an older harness) the
record is replayed.  A read without any boundary never goes to the reference (create_events reads peaks[-1]
there); the port's one-event answer for it is compared with the device only.
NPH_REF_EVENTS_RECORD=<path> pytest tests/test_events_edges_oracle.py writes a new record."""
import hashlib
import os
import re

import numpy as np
import pytest

from oracle.oracle_py import RefOracle
from tests import events_cases as ec
from tests import ref_calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_events_edges.pkl.xz")
KERNEL = os.path.join(ROOT, "nanopolish_b200", "csrc", "event_detect.cu")


def events_hash(start, length, mean, stdv) -> str:
    h = hashlib.sha1()
    for a, dt in ((start, np.uint64), (length, np.float32), (mean, np.float32), (stdv, np.float32)):
        h.update(np.ascontiguousarray(a, dt).tobytes())
    return h.hexdigest()


@pytest.fixture(scope="module")
def reference():
    """(live RefOracle or None, recorded answers, record path or None)"""
    path = os.environ.get("NPH_REF_EVENTS_RECORD")
    live = RefOracle() if RefOracle.available() else None
    if live is not None and not live.has("npref_detect_events_params"):
        live = None                 # a library built from an older harness, without the entry point: replay the record
    if path and live is None:
        pytest.fail("NPH_REF_EVENTS_RECORD needs the compiled reference with npref_detect_events_params (oracle/_ref/libnpref.so)")
    rec = {} if path else ref_calls.load(GOLDEN)
    yield live, rec, path
    if path:
        ref_calls.save(rec, path)


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
    live, record, path = reference
    rows, want_rows = [], None if path else record.get("events_edges")
    assert path or (want_rows is not None), f"no recorded reference answers ({GOLDEN}); re-record"
    n_ref = 0
    for pname, prm in ec.PARAMS.items():
        for r in reads:
            ev = port_oracle.detect_events(r.x, prm)
            fp = ec.fingerprint(r.x, prm)
            mine = events_hash(ev["start"], ev["length"], ev["mean"], ev["stdv"])
            if ev.shape[0] == 1:
                rows.append((fp, None))
                continue
            if live is not None:
                got = events_hash(*live.detect_events_params(r.x, prm))
            else:
                fp_w, got = want_rows[len(rows)]
                assert fp_w == fp, f"{r.name} under {pname}: inputs differ from the recorded ones; re-record"
            rows.append((fp, got))
            assert mine == got, f"{r.name} under {pname}: the port's events differ from scrappie's"
            n_ref += 1
    if path:
        record["events_edges"] = rows
    elif live is not None and want_rows is not None:
        assert [fp for fp, _ in want_rows] == [fp for fp, _ in rows], "edge reads differ from the recorded ones; re-record"
        assert want_rows == rows, "the compiled reference's answers differ from the record"
    assert n_ref > 1000


def test_builders_reach_every_edge(port_oracle):
    cover, claimed, preds = ec.check_edges(port_oracle)
    print("\n" + ec.coverage_table(cover, claimed))
    missing = sorted((w, c, k) for w, c, k in claimed if k not in cover[(w, c)])
    assert not missing, f"claimed cells without a read: {missing}"
    paths = {p.path for p in preds.values()}
    assert paths == {"fast", "guard", "slice", "wide"}
