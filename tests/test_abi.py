"""The C-ABI library builds, loads and exports every symbol include/nph.h declares; without a GPU
nph_create fails loudly with NPH_ERR_NO_DEVICE (there is no CPU path)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from nanopolish_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "nph.h")).read()
    declared = set(re.findall(r"\b(nph_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.nph_version() == 1


def test_pod_layouts_match_header():
    assert synth.READ_DT.itemsize == 64
    assert synth.HMM_JOB_DT.itemsize == 32
    assert synth.ABEA_JOB_DT.itemsize == 32
    assert synth.PAIR_DT.itemsize == 8
    assert synth.ABEA_RES_DT.itemsize == 24
    assert synth.HMM_JOB_DT.fields["stride"][1] == 28 and synth.HMM_JOB_DT.fields["flags"][1] == 30


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu tests")
    lib = _lib.load()
    ctx = C.c_void_p()
    rc = lib.nph_create(C.byref(ctx), 0)
    assert rc == _lib.NPH_ERR_NO_DEVICE
    assert b"no CPU path" in lib.nph_strerror(rc)
    from nanopolish_b200.engine import Engine
    with pytest.raises(_lib.NphError):
        Engine(0)


def test_score_set_combine_is_host_arithmetic(port_oracle):
    lib = _lib.load()
    rng = np.random.default_rng(3)
    s = rng.uniform(-200, -100, 30).astype(np.float32)
    out = np.zeros(10, np.float32)
    assert lib.nph_score_set_combine(s.ctypes.data_as(C.c_void_p), 10, 3, out.ctypes.data_as(C.c_void_p)) == 0
    for g in range(10):
        want = port_oracle.score_set_combine(s[3 * g:3 * g + 3])
        assert np.float32(want).view(np.uint32) == out[g].view(np.uint32)


def test_dist_library_exports():
    """libnph_dist.so (include/nph_dist.h): the NCCL exchange behind a C signature; libnph.so itself must stay free of NCCL."""
    import subprocess
    hdr = open(os.path.join(ROOT, "include", "nph_dist.h")).read()
    declared = set(re.findall(r"\b(nph_dist_[a-z0-9_]+)\s*\(", hdr))
    assert declared == {"nph_dist_gather_records", "nph_dist_gather_methylation_sites", "nph_dist_reduce_sum_f64"}
    so = os.path.join(ROOT, "nanopolish_b200", "libnph_dist.so")
    syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    for name in declared:
        assert f" T {name}" in syms, name
    needed = subprocess.run(["readelf", "-d", os.path.join(ROOT, "nanopolish_b200", "libnph.so")], capture_output=True, text=True).stdout
    assert "nccl" not in needed


@pytest.mark.gpu
def test_dist_gather_on_visible_gpus():
    """dist_gather_check (tests/cuda/dist_gather_check.cu, built into build/checks/): one host thread per visible GPU, variable-length gather to rank 0, the too-small-root case
    (every rank fails alike, nobody hangs) and the f64 reduce — a C++ caller sharding without Python."""
    import subprocess
    exe = os.path.join(ROOT, "build", "checks", "dist_gather_check")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok" in r.stdout


def test_tsv_number_formatting_on_host():
    """the host copy of csrc/tsv_format.cuh against snprintf (the device copy runs in the gpu tests)"""
    import subprocess
    exe = os.path.join(ROOT, "build", "checks", "check_tsv_format")
    r = subprocess.run([exe, "--host-only"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ", 0 bad" in r.stdout
