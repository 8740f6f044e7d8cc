"""The forward kernel's emission tail, cc + (-0.5*a)*a in one FMUL + one FFMA (exact_math.cuh: add_neg_half_square),
against the reference's literal three-rounding form on the device, bit for bit."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_emission_fold_on_device():
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_emission_fold")
    r = subprocess.run([exe, "500"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches" in r.stdout
