"""The compiled reference's score_variant_thresholded with a list of methylation types (oracle/_ref/libnpref_types.so, built by
oracle/ref_types.mk) — test infrastructure for methylation-aware candidate screening.

The `ref_types` fixture is the live library where it exists, else the answers it gave to the same test when they were recorded
(tests/golden/ref_calls_methylation.pkl.xz, replayed call by call as tests/ref_calls.py does for the `ref_oracle` fixture).
Recording: run the tests with NPH_REF_TYPES_RECORD=<path> where the library is built; the calls of the tests that ran are merged
into the file at <path> (or into the committed file, if <path> does not exist yet) and written there."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

from tests import ref_calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libnpref_types.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_calls_methylation.pkl.xz")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class RefTypesOracle:
    def __init__(self):
        self.lib = C.CDLL(LIB)

    @staticmethod
    def available() -> bool:
        return os.path.exists(LIB)

    def register_reads(self, reads, ev_mean, ev_start):
        hs = np.zeros(reads.shape[0], np.int32)
        for i, r in enumerate(reads):
            o, n = int(r["event_off"]), int(r["n_events"])
            m = np.ascontiguousarray(ev_mean[o:o + n]); t = np.ascontiguousarray(ev_start[o:o + n])
            hs[i] = self.lib.npref_types_read_create(C.c_uint32(n), _p(m), _p(t), C.c_double(r["shift"]), C.c_double(r["scale"]),
                                                     C.c_double(r["drift"]), C.c_double(r["var"]), C.c_double(r["events_per_base"]))
        return hs

    def clear_reads(self):
        self.lib.npref_types_reads_clear()

    def score_variants_thresholded(self, read_handles, windows, rc, ref_seq: str, ref_position, variants, flags, threshold, types,
                                   indel_bias=1.0):
        """[score_variant_thresholded(v, Haplotype(ref), reads, flags, threshold, types).quality for v in variants], single thread"""
        n, nv = len(read_handles), len(variants)
        rh = np.ascontiguousarray(read_handles, np.int32)
        es = np.array([w[0] for w in windows], np.uint32); ee = np.array([w[1] for w in windows], np.uint32)
        rcs = np.ascontiguousarray(rc, np.uint8)
        pos = (C.c_size_t * nv)(*[v[0] for v in variants])
        refs = (C.c_char_p * nv)(*[v[1].encode() for v in variants]); alts = (C.c_char_p * nv)(*[v[2].encode() for v in variants])
        q = np.zeros(nv)
        self.lib.npref_types_score_variants_thresholded(n, _p(rh), _p(es), _p(ee), _p(rcs), ref_seq.encode(), C.c_size_t(ref_position), nv, pos,
                                                        refs, alts, C.c_uint32(flags), C.c_uint32(threshold), ",".join(types).encode(),
                                                        C.c_double(indel_bias), _p(q))
        return q


@pytest.fixture(scope="session")
def _ref_types_session():
    path = os.environ.get("NPH_REF_TYPES_RECORD")
    live = RefTypesOracle() if RefTypesOracle.available() else None
    if path and live is None:
        pytest.fail("NPH_REF_TYPES_RECORD needs oracle/_ref/libnpref_types.so")
    calls = ref_calls.load(GOLDEN)
    recorded = {}
    yield live, calls, path, recorded
    if path:
        merged = ref_calls.load(path if os.path.exists(path) else GOLDEN)
        merged.update(recorded)
        ref_calls.save(merged, path)


@pytest.fixture
def ref_types(request, _ref_types_session):
    """score_variant_thresholded with methylation types: live where oracle/_ref/libnpref_types.so exists, else recorded answers"""
    live, calls, path, recorded = _ref_types_session
    key = ref_calls.test_key(request.node)
    if path:
        recorded[key] = []
        return ref_calls.Recorder(live, recorded[key])
    if live is not None:
        return live
    if key not in calls:
        pytest.fail(f"no recorded reference answers for {key} (tests/golden/ref_calls_methylation.pkl.xz)")
    return ref_calls.Replay(key, calls[key])
