"""phase-reads' call and quality step (nph_phase_quality, csrc/exact_math.cuh) against the restatement of
src/nanopolish_phase_reads.cpp:293-317 in tests/phase_restatement.py: ties, +-inf, NaN, score differences across the log-sum
table and on its 15.7 cut-off, and q at and beside every integer and 30.  The checker (tests/cuda/check_phase_quality.cu) runs the
host form here and compares host with device in the gpu test."""
import os
import struct
import subprocess

import numpy as np
import pytest

from tests import phase_restatement as pr

EXE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_phase_quality")


def _f(h):
    return np.float32(struct.unpack("<f", struct.pack("<I", int(h, 16)))[0])


def _lines(mode):
    out = subprocess.run([EXE, mode], check=(mode == "--host"), capture_output=True, text=True)
    return out


def test_host_quality_equals_restatement():
    lines = _lines("--host").stdout.splitlines()
    assert len(lines) > 160_000
    seen = set()
    for ln in lines:
        r, a, call, q = ln.split()
        want_call, want_q = pr.quality(_f(r), _f(a), b"C", b"T")
        assert (call.encode(), int(q)) == (want_call, want_q), ln
        seen.add(int(q))
    assert set(range(36, 64)) <= seen                       # every quality character from Q3 to Q30


@pytest.mark.gpu
def test_device_quality_equals_host():
    out = _lines("--device")
    assert out.returncode == 0 and out.stdout.splitlines()[-1] == "mismatches 0", out.stdout[-200:] + out.stderr
