"""The detect-polyi checkers themselves, without a GPU: the compiled reference's detect-polyi pieces against a plain Python
restatement of its segmentation HMM and Bernoulli stage on crafted and synthetic reads, and the harness's rows against the
row writer the device results go through."""
import os

import numpy as np
import pytest

from tests import polya_cases as pc
from tests import polyi_cases as qc


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(qc.REF_POLYI):
        pytest.skip("oracle/_ref/libnpref_polyi.so not built (it needs the reference sources)")
    return qc.RefPolyi()


@pytest.fixture(scope="module")
def reads(ref):
    rng = np.random.default_rng(7)
    return qc.edge_reads(rng, ref) + [qc.synth_polyi_read(rng, f"synthetic_{i}", int(rng.integers(300, 4000))) for i in range(12)]


def _tail(seg):
    """BernoulliHMM::segmentation's int start / stop: adapter + 1 and polya"""
    return int(seg[2]) + 1, int(seg[3])


def test_reference_pieces_match_restatement(ref, reads):
    for r in reads:
        seg, rl, q, bern, det, row = ref.read(r)
        if not r.loaded:
            assert row == f"{r.name}\t{r.contig}\t{r.pos}\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n"
            continue
        want = qc.restate_segment(r.samples, r.scale, r.shift, r.var)
        assert tuple(int(v) for v in seg) == tuple(int(v) for v in want), r.name
        assert rl[0] == pc.restate_rate(r), r.name
        start, stop = _tail(seg)
        assert bern == qc.restate_bernoulli(r, start, stop), r.name
        assert det == qc.restate_detected(bern[0], bern[1], stop - start), r.name


def test_reference_rows_use_the_tsv_format(ref, reads):
    """the harness's rows against nanopolish_b200.detect_polyi.row over the same numbers"""
    from nanopolish_b200 import detect_polyi
    from nanopolish_b200.synth import POLYI_RES_DT
    for r in reads:
        seg, rl, q, bern, det, row = ref.read(r)
        res = np.zeros(1, POLYI_RES_DT)[0]
        if seg is None:
            res["seg"]["qc"] = detect_polyi.READ_FAILED_LOAD
            res["polyi_last"] = res["polya_first"] = res["detected"] = -1
        else:
            for k, v in zip(("start", "leader", "adapter", "polya", "cliffs"), seg):
                res["seg"][k] = v
            res["seg"]["read_rate"], res["seg"]["polya_length"], res["seg"]["qc"] = rl[0], rl[1], q
            res["polyi_last"], res["polya_first"], res["detected"] = bern[0], bern[1], det
        assert detect_polyi.row(r.name, r.contig, r.pos, res) == row, r.name


def test_edge_reads_reach_their_conditions(ref, reads):
    """Every corner the edge reads are built for is reached: the four tags; tails of 99, 100 and 101 samples; polyi at 200 and
    201; region_length - polya at 200 and 201; centred samples exactly at the clamp bounds 40 and 200 and just beyond them, with
    lI / lA = -inf / -inf = NaN at 200; the sentinel fallback (a real poly(A) end at the sentinel index 3
    moves the tail to [n-1, n-1): 0 samples, NONE); reads of 2 to 5 samples; a zero
    median (infinite read rate) on a read whose tail is detected."""
    out = {r.name: (r, ref.read(r)) for r in reads}
    got = [(r, v) for r, v in out.values() if r.loaded]
    assert {v[4] for _, v in got} == {0, 1, 2, 3}
    tails = {_tail(v[0])[1] - _tail(v[0])[0] for _, v in got}
    assert {99, 100, 101} <= tails
    assert {200, 201} <= {v[3][0] for _, v in got}
    assert {200, 201} <= {(_tail(v[0])[1] - _tail(v[0])[0]) - v[3][1] for _, v in got if v[3][1] > 0}
    assert out["tail_99"][1][3] == (-1, -1) and out["tail_100"][1][3] != (-1, -1)
    # clamp bounds: the placed centred values, the bits they give and the NaN
    for name, ss in (("clamp_high", (200.0, 200.00002, 199.99998)), ("clamp_low", (40.0, 39.999992, 40.000008))):
        r, v = out[name]
        start, stop = _tail(v[0])
        assert stop - start == 1200
        assert [qc.centred(r, start, stop, start + 300 + 40 * i) for i in range(3)] == [np.float32(s) for s in ss]
    with np.errstate(all="ignore"):
        lI = qc._logf(qc._pdf(np.float32(200.0), np.float32(108.498), np.float32(5.257)))
        lA = qc._logf(qc._pdf(np.float32(200.0), np.float32(108.883), np.float32(3.257)))
        assert lI == -np.inf and lA == -np.inf and np.isnan(lI / lA)
    r, v = out["clamp_high"]
    start, stop = _tail(v[0])
    assert qc.restate_bits(r, start, stop)[300] == 0
    # the sentinel fallback
    r, v = out["short_5"]
    assert qc.restate_segment(r.samples, r.scale, r.shift, r.var, sentinel_rule=False)[3] == 3
    assert (int(v[0][2]), int(v[0][3])) == (3, 4) and v[3] == (-1, -1) and v[4] == 0
    for k in (2, 3, 4, 5):
        assert out[f"short_{k}"][0].samples.shape[0] == k and out[f"short_{k}"][1][4] == 0
    r, v = out["zero_median"]
    assert v[1][0] == float("inf") and v[4] != 0
