"""Pin the port oracle's profile_hmm_score (oracle/np_oracle.c) to the compiled reference on every job of tests/forward_cases.py
(every reachable forward class at its strip, lane, period, flag, strand, bias and outlier edges): bit-identical scores.  An event
no k-mer can emit leaves a finite score through the bad-event state.  The builders' edge claims, the coverage of every class and
the warp layouts the sub-warp classes need are checked here too.

The reference's answers live in tests/golden/ref_forward_edges.pkl.xz, one entry per job with a fingerprint of the job's inputs.
Where oracle/_ref/libnpref.so exists the reference is called live; elsewhere the record is replayed.  While recording each job
runs in a forked child, so that a job the reference aborts on would show up as such instead of ending the run:
NPH_REF_FORWARD_RECORD=<path> pytest tests/test_forward_edges_oracle.py writes a new record."""
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from oracle.oracle_py import RefOracle
from tests import forward_cases as fc
from tests import ref_calls
from tests.test_viterbi_edges_oracle import _fingerprint, _forked

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_forward_edges.pkl.xz")


@pytest.fixture(scope="module")
def reference():
    """(live RefOracle or None, recorded answers, record path or None)"""
    path = os.environ.get("NPH_REF_FORWARD_RECORD")
    live = RefOracle() if RefOracle.available() else None
    if path and live is None:
        pytest.fail("NPH_REF_FORWARD_RECORD needs the compiled reference (oracle/_ref/libnpref.so)")
    rec = {} if path else ref_calls.load(GOLDEN)
    yield live, rec, path
    if path:
        ref_calls.save(rec, path)


@pytest.fixture(scope="module")
def cases():
    return fc.batches(synth.load_model("nucleotide"))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("bias", fc.BIASES)
def test_forward_edges_match_reference(port_oracle, reference, cases, bias):
    live, rec, path = reference
    model = synth.load_model("nucleotide")
    b = cases[bias]
    n = b.jobs.shape[0]
    if live is not None:
        live.clear_reads()
        handles = live.register_reads(b.reads, b.ev_mean, b.ev_start_time, live.builtin_model("nucleotide"))
        mh = [live.builtin_model("nucleotide")]
    key = f"bias={bias}"
    if path:
        rec[key] = [(_fingerprint(b, j, bias), _forked(lambda j=j: live.score_batch(handles, b.jobs[j:j + 1], b.seqs[j:j + 1], mh,
                                                                                       indel_bias=bias)[0][0]))
                    for j in range(n)]
        assert not any(isinstance(w, str) for _, w in rec[key]), "the reference aborts on an edge job: drop it from the builder"
    assert key in rec and len(rec[key]) == n, f"no recorded reference answers for {key} ({GOLDEN}); re-record"
    for j in range(n):
        assert rec[key][j][0] == _fingerprint(b, j, bias), f"job {j}: inputs differ from the recorded ones; re-record"
    want = np.array([w for _, w in rec[key]], np.float32)
    if live is not None and not path:
        want, _ = live.score_batch(handles, b.jobs, b.seqs, mh, indel_bias=bias, threads=8)
    got, _ = port_oracle.hmm_score_batch(b.reads, b.ev_mean, b.ev_start_time, [model], b.kmer_ranks, b.jobs, indel_bias=bias,
                                         threads=8)
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, (f"{bad.size} of {n} scores differ, first jobs {bad[:5]}: {got[bad[:5]]} vs {want[bad[:5]]}; "
                           f"classes {[fc.choose_class(b.spec[j].K, b.spec[j].E)[0] for j in bad[:5]]}")


def test_builders_reach_every_class_edge(cases):
    """every reachable class receives a job of every edge it can hold (the table goes to the test log)"""
    covers = [fc.check_claims(b) for b in cases.values()]
    table, merged = fc.coverage_table(covers)
    print("\n" + table)
    for cls in fc.REACHABLE:
        assert fc.class_edges(cls) <= merged[cls], f"class {cls} misses {sorted(fc.class_edges(cls) - merged[cls])}"


@pytest.mark.parametrize("bias", fc.BIASES)
def test_sub_warp_classes_share_warps(cases, bias):
    """in each batch, every sub-warp class leaves empty groups in its last warp and has a warp whose jobs the schedule fixes that
    mixes step counts (the warp runs to its slowest group) and pre-clip with other jobs (the soft fold runs on every row)"""
    b = cases[bias]
    classes = fc.classes_of(b)
    for cls in sorted({c for c in classes if c[1] < 32}):
        G = 32 // cls[1]
        specs = [s for s, c in zip(b.spec, classes) if c == cls]
        assert len(specs) % G != 0, f"class {cls}: {len(specs)} jobs fill every warp"
        assert fc.mixed_warp(specs, G), f"class {cls}: no fixed warp mixes step counts and pre-clipping"


def test_rows_per_kmer_bound(port_oracle):
    """the long windows stay where the transitions exist: at MAX_ROWS_PER_KMER events per base every log-probability is finite,
    from about 286 on lp_mm_next is NaN"""
    for bias in fc.BIASES:
        assert np.isfinite(port_oracle.transitions(fc.MAX_ROWS_PER_KMER, bias)).all()
    assert np.isnan(port_oracle.transitions(290.0, 1.0)[3])
