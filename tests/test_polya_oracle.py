"""The poly(A) checkers themselves, without a GPU: the compiled reference's poly(A) pieces against a plain Python restatement
of segment_squiggle and the read rate on crafted reads, and the exhaustive expf / logf equality behind the device kernel."""
import os
import subprocess

import numpy as np
import pytest

from tests import polya_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(pc.REF_POLYA):
        pytest.skip("oracle/_ref/libnpref_polya.so not built (it needs the reference sources)")
    return pc.RefPolya()


def _reads():
    rng = np.random.default_rng(7)
    return pc.edge_reads(rng) + [pc.synth_read(rng, f"synthetic_{i}", int(rng.integers(300, 4000))) for i in range(12)]


def test_reference_pieces_match_restatement(ref):
    for r in _reads():
        seg, rl, qc, row = ref.read(r)
        if not r.loaded:
            assert row == f"{r.name}\t{r.contig}\t{r.pos}\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n"
            continue
        want = pc.restate_segment(r.samples, r.scale, r.shift, r.var)
        assert tuple(int(v) for v in seg) == tuple(int(v) for v in want), r.name
        assert rl[0] == pc.restate_rate(r), r.name


def test_reference_rows_use_the_tsv_format(ref):
    """the harness's rows against nanopolish_b200.polya.row over the same numbers (the formatting the device results go through)"""
    from nanopolish_b200 import polya
    from nanopolish_b200.synth import POLYA_RES_DT
    for r in _reads():
        seg, rl, qc, row = ref.read(r)
        res = np.zeros(1, POLYA_RES_DT)[0]
        if seg is None:
            res["qc"] = polya.READ_FAILED_LOAD
        else:
            res["start"], res["leader"], res["adapter"], res["polya"], res["cliffs"] = seg
            res["read_rate"], res["polya_length"], res["qc"] = rl[0], rl[1], qc
        assert polya.row(r.name, r.contig, r.pos, res) == row, r.name


def test_libm_exact_on_host_every_float():
    """csrc/libm_exact.cuh's host build equals this machine's expf on every float <= 0 and logf on every float >= 0"""
    exe = os.path.join(ROOT, "build", "checks", "check_libm_exact")
    r = subprocess.run([exe, "--host"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "expf: 0 bad, logf: 0 bad" in r.stdout


def test_edge_reads_reach_their_conditions(ref):
    """The sentinel rule fires on a real boundary at a sentinel index, and an infinite read rate meets a 0-sample tail (NaN
    length, printed as 0).  A real leader end at 1 or adapter end at 2 cannot occur: both need label A at index 2, and the
    backpointer of step 2 cannot point to A (the ADAPTER score of row 1 is -inf and every rule into A is a strict <)."""
    reads = {r.name: r for r in pc.edge_reads(np.random.default_rng(7))}
    raw = pc.restate_segment(reads["short_5"].samples, reads["short_5"].scale, reads["short_5"].shift, reads["short_5"].var, sentinel_rule=False)
    assert raw[3] == 3
    seg, rl, qc, row = ref.read(reads["short_5"])
    assert (int(seg[1]), int(seg[2]), int(seg[3])) == (2, 3, 4)
    seg, rl, qc, row = ref.read(reads["zero_median_no_tail"])
    assert int(seg[3]) == int(seg[2]) + 1 and rl[0] == float("inf") and rl[1] == 0.0
    seg, rl, qc, row = ref.read(reads["zero_median"])
    assert rl[0] == float("inf")
