"""Pin the port oracle's profile_hmm_align (oracle/np_oracle.c) to the compiled reference on every job of tests/viterbi_cases.py:
identical (event, k-mer) pairs, identical states and bit-identical l_fm, and a nonzero oracle status for exactly the jobs on
which the reference asserts.  The builders' edge claims are checked on the oracle's paths here too.

The reference's answers live in tests/golden/ref_viterbi_edges.pkl.xz, one row per job (a ref_calls.CaseRecord: asked live
where oracle/_ref/libnpref.so exists and compared with the record, replayed elsewhere).  The reference aborts the process on an
assert, so the jobs the oracle refuses or the builders claim it asserts on are only ever sent to it while recording, each job
in a forked child: NPH_REF_CASES_RECORD=<dir> pytest tests/test_viterbi_edges_oracle.py writes a new record to <dir>."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import ref_calls
from tests import viterbi_cases as vc

reference = ref_calls.case_fixture("ref_viterbi_edges.pkl.xz")


def _ref_call(ref, handles, b, j, bias):
    jr = b.jobs[j]
    return ref.align(handles[int(jr["read"])], ref.builtin_model("nucleotide"), b.seqs[j], jr["event_start"], jr["event_stop"],
                     jr["rc"], jr["flags"], indel_bias=bias)


@pytest.mark.parametrize("bias", [1.0, 0.9])
def test_viterbi_edges_match_reference(port_oracle, reference, bias):
    model = synth.load_model("nucleotide")
    b = vc.batches(model)[bias]
    n = b.jobs.shape[0]
    live = reference.live
    if live is not None:
        live.clear_reads()
        handles = live.register_reads(b.reads, b.ev_mean, b.ev_start_time, live.builtin_model("nucleotide"))
    paths, statuses = zip(*[port_oracle.hmm_align(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs[j],
                                                  indel_bias=bias) for j in range(n)])
    skip = {} if reference.recording else {j: ref_calls.ASSERTS for j in range(n)
                                           if statuses[j] != 0 or "asserts" in b.spec[j].edges}
    answers = reference.answers(f"bias={bias}", [vc.fingerprint(b, j, bias) for j in range(n)],
                                lambda j: _ref_call(live, handles, b, j, bias), skip=skip, fork=True)
    n_asserts = 0
    for j, want in enumerate(answers):
        got, status = paths[j], statuses[j]
        if isinstance(want, str):
            assert want == ref_calls.ASSERTS
            assert status != 0 and got.shape[0] == 0, f"job {j}: the reference asserts, the oracle returned {got.shape[0]} states"
            n_asserts += 1
            continue
        ek, lfm, st = want
        assert status == 0 and got.shape[0] == ek.shape[0] > 0, f"job {j}: {got.shape[0]} states (status {status}) vs {ek.shape[0]}"
        assert np.array_equal(got["event_idx"], ek[:, 0]) and np.array_equal(got["kmer_idx"], ek[:, 1]), f"job {j}: path"
        assert got["state"].tobytes() == st, f"job {j}: states"
        assert np.array_equal(got["l_fm"].view(np.uint32), lfm.view(np.uint32)), f"job {j}: l_fm"
    assert n_asserts == sum("asserts" in s.edges for s in b.spec) > 0
    vc.check_edges(b, list(paths), list(statuses))


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
