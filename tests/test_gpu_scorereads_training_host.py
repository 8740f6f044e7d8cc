"""ScoreReads(events_per_segment, true) end to end through the C++ host mirror (nanopolish_b200/host/nph_scorereads.*): reads
aligned by the mirror's event aligner, their segments scored and trained through nph_train_transitions_batch in one and in two
run() batches.  The per-read scores must equal those without training bit for bit, and the two strands' accumulated counts and
report() must equal the restatement (tests/transition_restatement.py, pinned to the compiled reference by
tests/test_transition_training_oracle.py) over nph_hmm_align_batch's paths of the same segments."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200.engine import Engine
from tests import eventalign_cases as EC
from tests import host_mirror as hm
from tests import transition_restatement as tr

pytestmark = pytest.mark.gpu
host = hm.fixture()


@pytest.fixture(scope="module")
def cases():
    return EC.build_cases()


def _train(host, cases, train, n_batches, max_chunk_jobs=0):
    model, rs, cs = cases
    n = len(cs)
    reads = np.array([EC.read_slot(c, rs.n_reads) for c in cs], np.int32)
    refs = (C.c_char_p * n)(*[c["fetched"].encode() for c in cs])
    offs = np.array([c["ref_pos"] for c in cs], np.int32)
    sc = np.zeros((n, 3)); counts = np.zeros((2, tr.WORDS), np.uint64); buf = C.create_string_buffer(1 << 14)
    p = hm.p
    k = host.nphh_scorereads_train(n, p(reads), refs, p(offs), EC.EPS, train, C.c_uint32(max_chunk_jobs), n_batches, p(sc), p(counts), buf,
                                   C.c_size_t(1 << 14))
    assert k >= 0, host.nphh_last_error()
    return sc, counts, buf.raw[:k].decode()


def test_score_reads_with_training(host, cases):
    model, rs, cs = cases
    EC.load_batch(host, cases)
    assert host.nphh_ea_run(C.c_double(1.0)) >= 0, host.nphh_last_error()
    plain, _, text0 = _train(host, cases, 0, 1)
    one, c1, text1 = _train(host, cases, 1, 1)
    two, c2, text2 = _train(host, cases, 1, 2, max_chunk_jobs=3)
    assert text0 == ""
    assert plain.tobytes() == one.tobytes() == two.tobytes()                 # training leaves the scores as they are
    assert c1.tobytes() == c2.tobytes() and text1 == text2                    # two batches accumulate to the one-batch counts
    # the restatement over the device's Viterbi paths of the same segments (the job list ScoreReads builds, mode 0)
    jobs, ranks, _ = EC.scorereads(host, cases, mode=0)
    slots = list(dict.fromkeys(EC.read_slot(c, rs.n_reads) for c in cs))    # the batch's read table: reads in first-use order
    jobs = jobs.copy()
    jobs["read"] = np.array(slots, np.uint32)[jobs["read"]]
    eng = Engine(0)
    try:
        eng.model_upload(model)
        paths, _ = eng.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ranks, jobs)
    finally:
        eng.close()
    want = np.zeros((2, tr.WORDS), np.uint64)
    for jo, pth in zip(jobs, paths):
        r = rs.reads[int(jo["read"])]
        rk = ranks[int(jo["rank_off"]):int(jo["rank_off"]) + int(jo["n_kmers"])]
        path = [(int(s["event_idx"]), int(s["kmer_idx"]), s["state"].decode()) for s in pth]
        tr.add_training(want[0], path, rk, lambda q, r=r: tr.scaled_mean(float(model.level_mean[q]), float(r["scale"]), float(r["shift"])))
    assert want[0, tr.SKIPS] > 0 and want[0, tr.TOTAL:].sum() > 0
    assert c1.tobytes() == want.tobytes()
    assert text1 == tr.report(want)
    host.nphh_ea_begin()
