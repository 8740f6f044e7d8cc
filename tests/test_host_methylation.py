"""SURVEY.md 8(f) row N3 — call-methylation's per-read logic as staging / one launch / scatter
(nanopolish_b200/host/nph_methylation.*).  The expectation is the Python restatement of calculate_methylation_for_read
(tests/meth_restatement.py, src/basemods/nanopolish_basemods.cpp:238-457) whose windows are scored by the oracle; the
C++ side must produce the same TSV, byte for byte (src/nanopolish_call_methylation.cpp:532-550)."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import meth_restatement as mr
from tests.test_host_mirror import HOST_SO, _register, _register_reads

pytestmark = pytest.mark.gpu
K = 6


@pytest.fixture(scope="module")
def host():
    lib = C.CDLL(HOST_SO)
    lib.nphh_last_error.restype = C.c_char_p
    lib.nphh_call_methylation.restype = C.c_longlong
    return lib


def _expected_tsv(port_oracle, rs, models, reads_meta):
    lines = []
    for ridx, meta in enumerate(reads_meta):
        ref_start, pairs, rc = meta["ref_start"], meta["pairs"], meta["rc"]
        for start_position, end_position, n_motif, e1, e2, ru, rm, seq in mr.enumerate_record(
                meta["ref"], ref_start, [p[0] for p in pairs], [p[1] for p in pairs], rc, "cpg", K):
            jobs = np.zeros(2, synth.HMM_JOB_DT)
            jobs[0] = (0, ridx, 1, e1, e2, ru.shape[0], 1 if e1 <= e2 else -1, rc, 3, 0)
            jobs[1] = (ru.shape[0], ridx, 1, e1, e2, rm.shape[0], 1 if e1 <= e2 else -1, rc, 3, 0)
            sc, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, models, np.concatenate([ru, rm]).astype(np.uint32), jobs)
            ll_u, ll_m = float(sc[0]), float(sc[1])
            lines.append("%s\t%s\t%d\t%d\t%s\t%.2f\t%.2f\t%.2f\t%d\t%d\t%s\n" % (
                "chr1", "-" if meta["is_rev"] else "+", start_position, end_position, meta["name"], ll_m - ll_u, ll_m, ll_u, 1, n_motif, seq))
    return "".join(lines)


def test_call_methylation_tsv_identical(host, port_oracle):
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    rs = synth.gen_reads(6, 2500, nuc, seed=2024, cpg_keep=0.3)
    mh, ch = _register(host, nuc), _register(host, cpg)
    rh = _register_reads(host, rs, mh)
    for r in rh:
        host.nphh_read_add_model(r, b"cpg", ch)
    metas = []
    for i in range(rs.n_reads):
        codes = rs.seq_codes[i]
        nk = codes.shape[0] - K + 1
        kfe = np.minimum(rs.kmer_first_event[i], int(rs.reads[i]["n_events"]) - 1)
        ref_start = 10_000 * (i + 1)
        if i % 3 == 2:
            # reverse-strand read: the reference is the reverse complement of what the pore saw; ref k-mer p pairs with
            # read k-mer nk-1-p, so event indices fall as reference positions rise (data.rc, stride -1)
            ref = synth._CODE2DNA[(3 - codes[::-1]).astype(np.uint8)].tobytes().decode()
            pairs = [(ref_start + p, int(kfe[nk - 1 - p])) for p in range(K, nk - K)]
            rc, is_rev = 1, True
        else:
            ref = synth._CODE2DNA[codes].tobytes().decode()
            pairs = [(ref_start + p, int(kfe[p])) for p in range(K, nk - K)]
            rc, is_rev = 0, False
        metas.append(dict(ref=ref, ref_start=ref_start, pairs=pairs, rc=rc, name=f"read_{i}", is_rev=is_rev))
    want = _expected_tsv(port_oracle, rs, [nuc, cpg], metas)
    assert want.count("\n") > 60

    n = rs.n_reads
    flat = np.array([x for m in metas for pr in m["pairs"] for x in pr], np.int32)
    off = np.zeros(n + 1, np.uint64); off[1:] = np.cumsum([len(m["pairs"]) for m in metas])
    names = (C.c_char_p * n)(*[m["name"].encode() for m in metas])
    refs = (C.c_char_p * n)(*[m["ref"].encode() for m in metas])
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    buf = C.create_string_buffer(1 << 20)
    njobs = C.c_uint64()
    got = host.nphh_call_methylation(n, p(np.array(rh, np.int32)), names, p(np.array([m["is_rev"] for m in metas], np.uint8)),
                                     p(np.array([m["rc"] for m in metas], np.uint8)), p(np.array([m["ref_start"] for m in metas], np.int32)),
                                     refs, p(flat), p(off), b"chr1", C.c_double(1.0), buf, C.c_size_t(1 << 20), C.byref(njobs))
    assert got >= 0, host.nphh_last_error()
    assert njobs.value == 2 * want.count("\n")                    # two jobs per scored group, one launch for all reads
    assert buf.value.decode() == want


def test_flat_call_formats_its_rows_on_the_device(host):
    """nph::call_methylation_flat with the compact event alignment: one C call, methylation_calls.tsv bytes out, the rows formatted by
    nph_methylation_tsv — against Python's formatting of the site records of the same batch."""
    from nanopolish_b200.engine import Engine
    from tests.test_gpu_methylation import _expected_rows
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    rs = synth.gen_reads(40, 2500, nuc, seed=808, cpg_keep=0.3)
    ref, pairs, recs = synth.methylation_records(rs, model_id=1, rc_every=2)
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    params = synth.meth_params("cpg", K)
    eng = Engine(0)
    try:
        eng.model_upload(nuc); eng.model_upload(cpg)
        site_off, sites, scored = eng.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs, params)
    finally:
        eng.close()
    n = rs.n_reads
    names_py = [f"read_{i}" for i in range(n)]
    is_rev = np.ascontiguousarray(recs["rc"]).astype(np.uint8)
    want = _expected_rows(sites, site_off, recs, ref, names_py, is_rev, "chr1", K)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    cm, cs, cl = (np.ascontiguousarray(x) for x in (cpg.level_mean, cpg.level_stdv, cpg.level_log_stdv))
    host.nphh_model_create.restype = C.c_int
    mh = host.nphh_model_create(b"cpg", 6, cm.shape[0], vp(cm), vp(cs), vp(cl))
    names = (C.c_char_p * n)(*[s.encode() for s in names_py])
    host.nphh_call_methylation_flat.restype = C.c_longlong
    buf = np.zeros(len(want) + 4096, np.uint8)
    ns, se = C.c_uint64(), C.c_uint64()
    secs = np.zeros(2)
    recs2 = recs.copy()
    got = host.nphh_call_methylation_flat(vp(rs.reads), C.c_size_t(n), vp(rs.ev_mean), None, C.c_size_t(rs.ev_mean.shape[0]),
                                          vp(ref), C.c_size_t(ref.shape[0]), None, C.c_size_t(0), vp(deltas), vp(first),
                                          vp(recs2), C.c_size_t(n), mh, names, vp(is_rev), b"chr1", C.c_double(1.0),
                                          vp(buf), C.c_size_t(buf.shape[0]), C.byref(ns), C.byref(se), vp(secs))
    assert got >= 0, host.nphh_last_error()
    assert int(ns.value) == sites.shape[0] and int(se.value) == scored
    assert buf[:got].tobytes().decode() == want
    # the pair-list form of the same batch: its rows are formatted on the host, by the same row writer
    pairs_c = np.ascontiguousarray(pairs)
    buf[:] = 0
    got = host.nphh_call_methylation_flat(vp(rs.reads), C.c_size_t(n), vp(rs.ev_mean), None, C.c_size_t(rs.ev_mean.shape[0]),
                                          vp(ref), C.c_size_t(ref.shape[0]), vp(pairs_c), C.c_size_t(pairs_c.shape[0]), None, None,
                                          vp(recs2), C.c_size_t(n), mh, names, vp(is_rev), b"chr1", C.c_double(1.0),
                                          vp(buf), C.c_size_t(buf.shape[0]), C.byref(ns), C.byref(se), vp(secs))
    assert got >= 0, host.nphh_last_error()
    assert buf[:got].tobytes().decode() == want
