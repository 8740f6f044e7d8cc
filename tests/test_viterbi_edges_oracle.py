"""Pin the port oracle's profile_hmm_align (oracle/np_oracle.c) to the compiled reference on every job of tests/viterbi_cases.py:
identical (event, k-mer) pairs, identical states and bit-identical l_fm, and a nonzero oracle status for exactly the jobs on
which the reference asserts.  The builders' edge claims are checked on the oracle's paths here too.

The reference's answers live in tests/golden/ref_viterbi_edges.pkl.xz, one entry per job with a fingerprint of the job's
inputs.  Where oracle/_ref/libnpref.so exists the reference is called live on every job the record does not mark as asserting;
elsewhere the record is replayed.  The reference aborts the process on an assert, so the asserting jobs are only ever run while
recording, each in a forked child: NPH_REF_VITERBI_RECORD=<path> pytest tests/test_viterbi_edges_oracle.py writes a new record."""
import hashlib
import os
import pickle
import signal

import numpy as np
import pytest

from nanopolish_b200 import synth
from oracle.oracle_py import RefOracle
from tests import ref_calls
from tests import viterbi_cases as vc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_viterbi_edges.pkl.xz")
ASSERTS = "asserts"


def _fingerprint(b, j: int, bias: float) -> str:
    jr = b.jobs[j]
    r = b.reads[int(jr["read"])]
    o, n = int(r["event_off"]), int(r["n_events"])
    h = hashlib.sha1()
    for part in (b.seqs[j], jr.tobytes(), r.tobytes(), b.ev_mean[o:o + n].tobytes(), b.ev_start_time[o:o + n].tobytes(),
                 np.float64(bias).tobytes()):
        h.update(part)
    return h.hexdigest()


def _ref_call(ref, handles, b, j, bias):
    jr = b.jobs[j]
    return ref.align(handles[int(jr["read"])], ref.builtin_model("nucleotide"), b.seqs[j], jr["event_start"], jr["event_stop"],
                     jr["rc"], jr["flags"], indel_bias=bias)


def _forked(fn):
    """fn() in a forked child: its pickled result, or ASSERTS if the child died of SIGABRT"""
    rd, wr = os.pipe()
    pid = os.fork()
    if pid == 0:
        os.close(rd)
        try:
            data = pickle.dumps(fn())
            with os.fdopen(wr, "wb") as f:
                f.write(data)
        finally:
            os._exit(0)
    os.close(wr)
    with os.fdopen(rd, "rb") as f:
        data = f.read()
    _, st = os.waitpid(pid, 0)
    if os.WIFSIGNALED(st) and os.WTERMSIG(st) == signal.SIGABRT:
        return ASSERTS
    assert os.WIFEXITED(st) and data, f"reference child ended with status {st}"
    return pickle.loads(data)


@pytest.fixture(scope="module")
def reference():
    """(live RefOracle or None, recorded answers, record path or None)"""
    path = os.environ.get("NPH_REF_VITERBI_RECORD")
    live = RefOracle() if RefOracle.available() else None
    if path and live is None:
        pytest.fail("NPH_REF_VITERBI_RECORD needs the compiled reference (oracle/_ref/libnpref.so)")
    rec = {} if path else ref_calls.load(GOLDEN)
    yield live, rec, path
    if path:
        ref_calls.save(rec, path)


@pytest.mark.parametrize("bias", [1.0, 0.9])
def test_viterbi_edges_match_reference(port_oracle, reference, bias):
    live, rec, path = reference
    model = synth.load_model("nucleotide")
    b = vc.batches(model)[bias]
    n = b.jobs.shape[0]
    if live is not None:
        live.clear_reads()
        handles = live.register_reads(b.reads, b.ev_mean, b.ev_start_time, live.builtin_model("nucleotide"))
    key = f"bias={bias}"
    if path:
        rec[key] = [(_fingerprint(b, j, bias), _forked(lambda j=j: _ref_call(live, handles, b, j, bias))) for j in range(n)]
    assert key in rec and len(rec[key]) == n, f"no recorded reference answers for {key} ({GOLDEN}); re-record"
    paths, statuses = [], []
    n_asserts = 0
    for j in range(n):
        fp, want = rec[key][j]
        assert fp == _fingerprint(b, j, bias), f"job {j}: inputs differ from the recorded ones; re-record"
        got, status = port_oracle.hmm_align(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs[j], indel_bias=bias)
        paths.append(got); statuses.append(status)
        if isinstance(want, str):
            assert want == ASSERTS
            assert status != 0 and got.shape[0] == 0, f"job {j}: the reference asserts, the oracle returned {got.shape[0]} states"
            n_asserts += 1
            continue
        if live is not None and not path:
            assert status == 0, f"job {j}: oracle status {status} where the record has a path"
            want = _ref_call(live, handles, b, j, bias)
        ek, lfm, st = want
        assert status == 0 and got.shape[0] == ek.shape[0] > 0, f"job {j}: {got.shape[0]} states (status {status}) vs {ek.shape[0]}"
        assert np.array_equal(got["event_idx"], ek[:, 0]) and np.array_equal(got["kmer_idx"], ek[:, 1]), f"job {j}: path"
        assert got["state"].tobytes() == st, f"job {j}: states"
        assert np.array_equal(got["l_fm"].view(np.uint32), lfm.view(np.uint32)), f"job {j}: l_fm"
    assert n_asserts == sum("asserts" in s.edges for s in b.spec) > 0
    vc.check_edges(b, paths, statuses)


def test_builders_reach_every_class_edge(port_oracle):
    """every class receives a job of every edge kind it can hold (the table goes to the test log)"""
    model = synth.load_model("nucleotide")
    covers = []
    for bias, b in vc.batches(model).items():
        res = [port_oracle.hmm_align(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs[j], indel_bias=bias)
               for j in range(b.jobs.shape[0])]
        covers.append(vc.check_edges(b, [r[0] for r in res], [r[1] for r in res]))
    table, merged = vc.coverage_table(covers)
    print("\n" + table)
    for C in vc.COLS:
        assert vc.CLASS_EDGES[C] <= merged[C], f"class {C} misses {sorted(vc.CLASS_EDGES[C] - merged[C])}"
    # both strands, every flag value and both biases take part
    all_specs = [s for b in vc.batches(model).values() for s in b.spec]
    assert {s.rc for s in all_specs} == {False, True} and {s.flags for s in all_specs} == {0, 1, 2, 3}


def test_trace_budget_restatement():
    """the limits include/nph.h states: one K = E window is refused from 23 046 on, and on a 132-SM H100 the resident CTAs
    are capped from K = E = 1 983 on"""
    assert vc.smallest_refused_square() == 23046
    assert vc.max_ctas([(23045, 23045)], 132) == 1 and vc.max_ctas([(23046, 23046)], 132) == 0
    assert vc.smallest_capped_square(132) == 1983
