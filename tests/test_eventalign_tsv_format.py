"""The eventalign.tsv row rule of csrc/tsv_format.cuh on the CPU: put_g6 against snprintf("%g") on every float of its domain
(both signs, about 9.4e8 values, plus the refusal of every float outside it) and ea_row_numbers / put_ea_row / ea_scaled_sample
against snprintf with the reference's format strings on seeded random rows, 'B' states included (tests/cuda/check_g_format.cu,
host build; the device build runs in tests/test_gpu_eventalign_tsv.py)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_g_format_and_eventalign_rows_match_the_c_library():
    exe = os.path.join(ROOT, "build", "checks", "check_g_format")
    r = subprocess.run([exe, "--host"], capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
    assert "0 bad" in r.stdout
