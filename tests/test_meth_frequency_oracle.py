"""tests/meth_frequency.py (the checker of the device frequency table) against the reference's own
scripts/calculate_methylation_frequency.py, byte for byte, on seeded and crafted methylation_calls.tsv inputs.

Where the reference tree exists ($REF, default /root/reference, as oracle/Makefile finds it) the script runs as a subprocess;
elsewhere its stdout recorded there (tests/golden/meth_frequency_ref.pkl.xz) is replayed.  Recording: run this file with
NPH_FREQ_RECORD=<path> where the script exists; the answers of every case are written to <path>.
"""
from __future__ import annotations

import lzma
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from tests import meth_frequency as mf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "meth_frequency_ref.pkl.xz")
SCRIPT = os.path.join(os.environ.get("REF", "/root/reference"), "scripts", "calculate_methylation_frequency.py")
CONTIGS = ["chr1", "chr10", "chr2", "chrX", "1", "GL000220.1"]
THRESHOLDS = [0.0, 1.0, 2.0, 2.5]


def _row(c, s, e, llr, n, seq, name="read"):
    return "%s\t+\t%d\t%d\t%s\t%.2f\t%.2f\t%.2f\t1\t%d\t%s\n" % (c, s, e, name, llr, llr - 50.0, -50.0, n, seq)


def _random_seq(rng, n_cg, length):
    b = np.array(list("ACGT"))[rng.integers(0, 4, length)]
    for p in rng.choice(length - 1, n_cg, replace=False):
        b[p], b[p + 1] = "C", "G"
    return "".join(b)


def crafted_files(seed: int = 5):
    """two methylation_calls.tsv texts with every rule of the script on show"""
    rng = np.random.default_rng(seed)
    a, b = [], []
    # frequencies 1/80, 1/16, 3/8, 0 and 1 at single-site keys (|llr| = 5 passes every threshold here)
    for start, (meth, total) in zip((100, 200, 300, 400, 500), ((1, 80), (1, 16), (3, 8), (0, 5), (7, 7))):
        for i in range(total):
            (a if i % 2 else b).append(_row("chr2", start, start, 5.0 if i < meth else -5.0, 1, "AACGTT"))
    # llr exactly at +-threshold * n, and both zeros
    for t in THRESHOLDS:
        for n in (1, 2, 3):
            s = 1000 + int(100 * t) + 10 * n
            seq = "GG" + "CGA" * n + "TT"
            a.append(_row("chr1", s, s + 3 * (n - 1), t * n, n, seq))
            a.append(_row("chr1", s, s + 3 * (n - 1), -t * n, n, seq))
            a.append(_row("chr1", s + 5, s + 5 + 3 * (n - 1), t * n - 0.01, n, seq))
    a.append("chr10\t+\t77\t77\tz\t-0.00\t-3.00\t-3.00\t1\t1\tACGTA\n")
    a.append("chr10\t+\t78\t78\tz\t0.00\t-3.00\t-3.00\t1\t1\tACGTA\n")
    # the same key with different sequences (the first one stays), across the two files
    a.append(_row("chrX", 50, 50, 9.0, 1, "TTCGAA"))
    b.append(_row("chrX", 50, 50, 9.0, 1, "TTCGA"))
    # CGCG: two overlapping matches; a multi-site group without CG; a split key on a single-site key
    a.append(_row("GL000220.1", 10, 12, 12.0, 2, "AACGCGTT"))
    a.append(_row("GL000220.1", 30, 36, 12.0, 2, "GATCAAGATC"))
    b.append(_row("GL000220.1", 12, 12, -9.0, 1, "CGCGTT"))
    b.append(_row("GL000220.1", 10, 10, -9.0, 1, "CGTTT"))
    # seeded bulk over every contig, keys that repeat (clear of the keys above)
    for f in (a, b):
        for _ in range(400):
            c = CONTIGS[int(rng.integers(0, len(CONTIGS)))]
            n = int(rng.integers(1, 4))
            s = 2000 + int(rng.integers(0, 40)) * 7
            e = s + (0 if n == 1 else int(rng.integers(2, 30)))
            llr = float(np.round(rng.normal(0.0, 6.0), 2))
            f.append(_row(c, s, e, llr, n, _random_seq(rng, n, 11 + e - s)))
    return [mf.CALLS_HEADER + "".join(a), mf.CALLS_HEADER + "".join(b)]


CASES = [(t, s) for t in THRESHOLDS for s in (False, True)]


def _case_id(t, split):
    return f"c{t}{'-s' if split else ''}"


_recorded: dict = {}


def _script_stdout(tmp_path, files, t, split):
    key = _case_id(t, split)
    if os.path.exists(SCRIPT):
        paths = []
        for i, text in enumerate(files):
            p = tmp_path / f"calls{i}.tsv"
            p.write_text(text)
            paths.append(str(p))
        cmd = [sys.executable, SCRIPT, "-c", repr(t)] + (["-s"] if split else []) + paths
        out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
        if os.environ.get("NPH_FREQ_RECORD"):
            _recorded[key] = out
            with lzma.open(os.environ["NPH_FREQ_RECORD"], "wb", preset=9) as f:
                pickle.dump(_recorded, f, protocol=4)
        return out
    with lzma.open(GOLDEN, "rb") as f:
        return pickle.load(f)[key]


@pytest.mark.parametrize("t,split", CASES, ids=[_case_id(*c) for c in CASES])
def test_restatement_equals_the_script(tmp_path, t, split):
    files = crafted_files()
    want = _script_stdout(tmp_path, files, t, split)
    assert mf.frequency_table(files, t, split) == want
    assert want.count("\n") > 100


def test_crafted_inputs_cover_the_rules():
    """the cases above are not vacuous: the frequencies, the boundary rows and the collisions are in the output"""
    files = crafted_files()
    plain = mf.frequency_table(files, 2.0, False)
    for row in ("chr2\t100\t100\t1\t80\t1\t0.013\t", "chr2\t200\t200\t1\t16\t1\t0.062\t", "chr2\t300\t300\t1\t8\t3\t0.375\t",
                "chr2\t400\t400\t1\t5\t0\t0.000\t", "chr2\t500\t500\t1\t7\t7\t1.000\t", "chrX\t50\t50\t1\t2\t2\t1.000\tTTCGAA\n"):
        assert row in plain
    keys = [tuple(line.split("\t")[:3]) for line in plain.split("\n")[1:] if line]
    names = [k[0] for k in keys]
    assert names == sorted(names) and names.index("chr10") < names.index("chr2") and names[0] == "1"
    # at threshold 0 both zeros count, unmethylated; at 2.0 the rows at exactly 2.0 * n count, the ones 0.01 below do not
    zero = mf.frequency_table(files, 0.0, False)
    assert "chr10\t77\t77\t1\t1\t0\t0.000\tACGTA\n" in zero and "chr10\t78\t78\t1\t1\t0\t0.000\tACGTA\n" in zero
    assert "chr1\t1210\t1210\t1\t2\t1\t0.500\t" in plain
    assert "chr1\t1215\t1215\t" not in plain
    split = mf.frequency_table(files, 2.0, True)
    # CGCG at 10..12 splits into 10 and 12, each meeting a single-site key whose sequence it keeps (the split row came first)
    assert "GL000220.1\t10\t10\t1\t2\t1\t0.500\tsplit-group\n" in split and "GL000220.1\t12\t12\t1\t2\t1\t0.500\tsplit-group\n" in split
    assert "GL000220.1\t30\t" not in split


def test_frequency_number_formatting_on_host():
    """the host copy of tsv_format.cuh's fixed_of<3> against snprintf("%.3f") of every m / n, n <= 5000, and fixed_of<2> unchanged
    on the same values (the device copy runs in the gpu tests)"""
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_tsv_format")
    r = subprocess.run([exe, "--host-only"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ", 0 bad" in r.stdout
