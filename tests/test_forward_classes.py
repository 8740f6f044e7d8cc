"""Pin the restatement of csrc/hmm_classes.h in tests/forward_cases.py to the header itself, compiled on the host: the class and
step count of every job with K <= 1000 and E <= 130, of a sparse sample of larger jobs and of every edge job; the strip geometry;
the schedule key; and the 34 classes that jobs with K < 2000 reach.  The edge tests choose their jobs through the restatement, so
a change to the class model shows up here before it silently moves their jobs to other classes."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import forward_cases as fc

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nanopolish_b200", "csrc")

DRIVER = r"""
#include "hmm_classes.h"
extern "C" {
void drv_choose(int n, const uint32_t* K, const uint32_t* E, int32_t* cls, uint32_t* steps)
{
    for (int i = 0; i < n; ++i) cls[i] = nph_choose_class(K[i], E[i], &steps[i]);
}
void drv_geometry(int K, int E, int C, int W, int may_chain, int32_t* out)
{
    const nph_wave_geom g = nph_wave_geometry(K, E, C, W, may_chain != 0);
    const int32_t v[] = {g.strip, g.n_strips, g.kpad, g.P, g.end_lane(), g.end_slot(), g.total_steps()};
    for (int i = 0; i < 7; ++i) out[i] = v[i];
}
uint32_t drv_key_bucket(uint32_t steps, uint32_t chunk) { return nph_key_bucket(steps, chunk); }
}
"""


@pytest.fixture(scope="module")
def header(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a host C++ compiler is needed to compile hmm_classes.h"
    d = tmp_path_factory.mktemp("hmm_classes")
    src, so = d / "driver.cpp", d / "libdriver.so"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-I" + CSRC, "-o", str(so), str(src)], check=True)
    lib = C.CDLL(str(so))
    lib.drv_key_bucket.restype = C.c_uint32
    return lib


def _choose(lib, K, E):
    K = np.ascontiguousarray(K, np.uint32)
    E = np.ascontiguousarray(E, np.uint32)
    cls = np.zeros(K.shape, np.int32)
    steps = np.zeros(K.shape, np.uint32)
    lib.drv_choose(C.c_int(K.shape[0]), K.ctypes.data_as(C.c_void_p), E.ctypes.data_as(C.c_void_p), cls.ctypes.data_as(C.c_void_p),
                   steps.ctypes.data_as(C.c_void_p))
    return cls.astype(np.int64), steps.astype(np.int64)


def _compare(lib, K, E):
    want_c, want_s = _choose(lib, K, E)
    got_c, got_s = fc.choose_class_np(K, E)
    bad = np.flatnonzero((want_c != got_c) | (want_s != got_s))
    assert bad.size == 0, (f"{bad.size} jobs differ, first (K, E) = {list(zip(K[bad[:5]], E[bad[:5]]))}: header "
                           f"{[fc.class_of(int(c)) for c in want_c[bad[:5]]]} steps {want_s[bad[:5]]}, restatement "
                           f"{[fc.class_of(int(c)) for c in got_c[bad[:5]]]} steps {got_s[bad[:5]]}")


def test_class_and_steps_dense(header):
    K, E = np.meshgrid(np.arange(1, 1001), np.arange(1, 131), indexing="ij")
    _compare(header, K.ravel(), E.ravel())


def test_class_and_steps_sparse(header):
    rng = np.random.default_rng(5)
    K = np.concatenate([rng.integers(1, 20000, 40000), rng.integers(1000, 4000, 20000), np.arange(1, 3001)])
    E = np.concatenate([rng.integers(1, 20000, 40000), rng.integers(1, 200, 20000), rng.integers(100, 5000, 3000)])
    _compare(header, K, E)


def test_class_and_steps_of_edge_jobs(header):
    js = fc.all_jobs()
    _compare(header, np.array([j.K for j in js]), np.array([j.E for j in js]))


def test_geometry_and_key(header):
    rng = np.random.default_rng(9)
    out = (C.c_int32 * 7)()
    for _ in range(4000):
        K, E, Cc = int(rng.integers(1, 3000)), int(rng.integers(1, 300)), int(rng.integers(1, 11))
        W = int(rng.choice([4, 8, 16, 32]))
        chain = bool(rng.integers(0, 2)) or K > W * Cc
        header.drv_geometry(K, E, Cc, W, int(chain), out)
        g = fc.wave_geometry(K, E, Cc, W, chain)
        assert list(out) == [g.strip, g.n_strips, g.kpad, g.P, g.end_lane, g.end_slot, g.total_steps], (K, E, Cc, W, chain)
    for steps in list(range(0, 1000)) + [32 * 1000 + 7, 10 ** 6, 2 ** 31]:
        for chunk in (0, 3, 7, 8, 100):
            assert header.drv_key_bucket(steps, chunk) == fc.key_bucket(steps, chunk), (steps, chunk)


def test_reachable_classes(header):
    """K < 2000 with E < 2000 reaches exactly 34 classes: all ten at W = 4, C = 6..10 at W = 8, 16 and 32, chained C = 2..10"""
    K, E = np.meshgrid(np.arange(1, 2000), np.arange(1, 2000), indexing="ij")
    cls, _ = _choose(header, K.ravel(), E.ravel())
    got = {fc.class_of(int(c)) for c in np.unique(cls)}
    assert got == fc.REACHABLE and len(got) == 34
    assert sum(1 for c in got if c[1] == 4) == 10 and sum(1 for c in got if c[1] in (8, 16, 32) and not c[2]) == 15
    assert sorted(c[0] for c in got if c[2]) == list(range(2, 11))


def test_unreachable_edges_are_the_documented_ones():
    """the shape edges a class cannot hold, as forward_cases.class_edges states them"""
    for cls in fc.REACHABLE:
        C_, W, chained = cls
        missing = set(fc.EDGES) - fc.class_edges(cls)
        want = {"strip+1"} if not (chained and C_ == 2) else set()
        if not chained:
            want |= {"E=39", "E=40", "E=41", "short-period", "one-row-strips"}
            if (W == 4 and C_ >= 5) or (W == 8 and C_ >= 9):
                want |= {"end-slot-0", "one-col-lane"}
            if C_ == 1:
                want.add("one-col-lane")
            if (C_ == 6 and W in (8, 16, 32)) or (C_ == 7 and W == 32):
                want.add("E=1")
            if C_ == 6 and W in (16, 32):
                want.add("E=2")
        else:
            if C_ < 6:
                want |= {"E=1", "E=2", "one-row-strips"}
            if C_ > 6:
                want |= {"E=39", "E=40", "E=41"}
        assert missing == want, f"class {cls}: cannot hold {sorted(missing)}, documented {sorted(want)}"
