"""Pin the port oracle's ABEA (npo_abea, oracle/np_oracle.c) to the compiled reference on every job of tests/abea_cases.py:
identical AlignedPairs, and an empty result exactly where the oracle's n_pairs is 0.  The builders' edge claims are checked on
the oracle's results and band history here too, and the coverage table goes to the test log.

The reference's answers live in tests/golden/ref_abea_edges.pkl.xz, one row per job: a fingerprint of the job's inputs, the
number of pairs and a hash of them (a ref_calls.CaseRecord: asked live where oracle/_ref/libnpref.so exists and compared with
the record, replayed elsewhere).  Jobs whose oracle status is NO_END_CELL never go to the reference, which walks its trace from
an unset cell there.  NPH_REF_CASES_RECORD=<dir> pytest tests/test_abea_edges_oracle.py writes a new record to <dir>, each job
in a forked child."""
import os
import re

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import abea_cases as ac
from tests import ref_calls

KERNEL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nanopolish_b200", "csrc", "abea.cu")

reference = ref_calls.case_fixture("ref_abea_edges.pkl.xz")


def _ref_answer(live, handles, b, j):
    jr = b.jobs[j]
    E = int(b.reads[int(jr["read"])]["n_events"])
    pr, n = live.abea(handles[int(jr["read"])], live.builtin_model("nucleotide"), b.seqs[j], E + int(jr["n_kmers"]) + 2)
    assert n >= 0
    return int(n), ac.pairs_hash(pr[:, 0], pr[:, 1])


def _register(live, b):
    if live is None:
        return None
    live.clear_reads()
    return live.register_reads(b.reads, b.ev_mean, b.ev_start_time, live.builtin_model("nucleotide"))


@pytest.fixture(scope="module")
def cases(port_oracle):
    model = synth.load_model("nucleotide")
    b = ac.batch(model, port_oracle)
    return model, b, ac.oracle_run(port_oracle, b, model), ac.oracle_run(port_oracle, b, model, full_cap=True)


def test_kernel_constants():
    """the band width, window, trace block and QC thresholds abea_cases.py states are abea.cu's"""
    src = open(KERNEL).read()
    assert re.search(r"constexpr int kBW = (\d+);", src).group(1) == str(ac.BAND)
    assert re.search(r"#define NPH_ABEA_TRACE_ROWS (\d+)", src).group(1) == str(ac.TRACE_BLOCK)
    assert re.search(r"const int uK = K \+ (\d+);", src).group(1) == str(ac.WINDOW)
    assert re.search(r"laneK = uK & 31, slotK = \(uK >> 5\) & 3", src)
    assert re.search(r"max_gap > (\d+)\) status", src).group(1) == str(ac.MAX_GAP)
    assert float(re.search(r"avg < (-[\d.]+)\) status", src).group(1)) == ac.MIN_AVG


def test_abea_edges_match_reference(cases, reference):
    model, b, runs, full = cases
    live = reference.live
    handles = _register(live, b)
    n = b.jobs.shape[0]
    skip = {j: None for j in range(n) if int(full[j][1]["status"]) & ac.NO_END_CELL}
    answers = reference.answers("abea_edges", [ac.fingerprint(b, j) for j in range(n)], lambda j: _ref_answer(live, handles, b, j),
                                skip=skip, fork=True)
    n_skipped = 0
    for j, want in enumerate(answers):
        pairs, res = full[j][:2]
        if int(res["status"]) & ac.NO_END_CELL:
            assert want is None and int(res["n_pairs"]) == 0
            n_skipped += 1
            continue
        wn, wh = want
        assert int(res["n_pairs"]) == wn, f"job {j}: oracle {int(res['n_pairs'])} pairs (status {int(res['status'])}), reference {wn}"
        assert ac.pairs_hash(pairs["ref_pos"], pairs["read_pos"]) == wh, f"job {j}: pairs differ from the reference's"
    assert n_skipped == sum(int(f[1]["status"]) & ac.NO_END_CELL != 0 for f in full)


def test_builders_reach_every_edge(cases, port_oracle):
    model, b, runs, full = cases
    cover = ac.check_edges(b, runs, full, port_oracle, model)
    kmods = {int(jr["n_kmers"]) % ac.WINDOW for jr, s in zip(b.jobs, b.spec) if s.family == "lane-slot"}
    print("\n" + ac.coverage_table(cover, kmods))
    assert kmods == set(range(ac.WINDOW))
    claimed = {f: set().union(*[s.edges for s in b.spec if s.family == f]) for f in ac.FAMILIES}
    for f in ac.FAMILIES:
        assert claimed[f], f"family {f} has no jobs"
        assert claimed[f] <= cover[f], f"family {f} misses {sorted(claimed[f] - cover[f])}"
    everything = set().union(*cover.values())
    for e in ("past-last-event", "no-end-cell", "diag-cross-block", "bi=2", "lead-trim-50", "tail-trim", "end-e0", "end-last",
              "end-bi<63", "end-bi=63", "end-bi=64", "end-bi=65", "gap=50", "gap=51", "low-emission", "max-gap", "low-emission+max-gap",
              "cap=n-1", "cap=n", "cap=n+1", "cap=n+31", "cap=n+32", "cap=n+33", "cap=n+1000", "cap=1", "shared-read"):
        assert e in everything, f"no job reaches {e}"
    # a job with a K >= 1000 and the stall on k-mer 0's level take part
    assert max(int(k) for k in b.jobs["n_kmers"]) >= 1000


def test_failure_records(cases):
    """the record of a failed job as include/nph.h defines it"""
    model, b, runs, full = cases
    for j in range(b.jobs.shape[0]):
        res, fres = runs[j][1], full[j][1]
        st = int(res["status"])
        if st & ac.NO_END_CELL:
            assert st == ac.NO_END_CELL and int(res["n_aligned"]) == 0 and int(res["max_gap"]) == 0
        if st & ac.PAIRS_OVERFLOW:
            assert st == ac.PAIRS_OVERFLOW
            assert int(res["n_aligned"]) == int(fres["n_aligned"]) and int(res["max_gap"]) == int(fres["max_gap"])
        if st & (ac.NO_END_CELL | ac.PAIRS_OVERFLOW):
            assert res["avg_log_emission"] == 0.0 and int(res["n_pairs"]) == 0
        else:
            assert res.tobytes() == fres.tobytes(), f"job {j}: room beyond the path changed the record"
        assert (int(res["n_pairs"]) > 0) == (st == 0)


def test_window_levels_emission(port_oracle):
    """the 2^64 builder puts |x - mu'| / sigma' in [2^64, 2^64.5): the reference's emission is finite and below -1e38 there"""
    model = synth.load_model("nucleotide")
    for rank in (0, 1000, 4095):
        x = ac.window_level(model, rank)
        mu, sd = np.float32(model.level_mean[rank]), np.float32(model.level_stdv[rank])
        a = (np.float64(x) - np.float64(mu)) / np.float64(sd)
        assert 2.0 ** 64 <= a < 2.0 ** 64.5
        em = port_oracle.lib.npo_log_normal_pdf(x, mu, sd, np.float32(np.log(model.level_stdv[rank])))
        assert np.isfinite(em) and em < -1e38


def test_mom_matches_reference(port_oracle, reference):
    """npo_mom equals the reference's estimate_scalings_using_mom bit for bit at E, K in {1, 31, 32, 33, 63, 64, 65} and on a
    21 000-event read"""
    model = synth.load_model("nucleotide")
    b = ac.mom_batch(model)
    live = reference.live
    handles = _register(live, b)
    n = b.jobs.shape[0]
    answers = reference.answers("mom", [ac.fingerprint(b, j) for j in range(n)], lambda j: tuple(
        live.mom(handles[int(b.jobs[j]["read"])], live.builtin_model("nucleotide"), b.seqs[j])[:2]))
    for j in range(n):
        got = port_oracle.mom(b.reads, b.ev_mean, model, b.kmer_ranks, b.jobs[j])
        assert np.array_equal(np.array(got).view(np.uint64), np.array(answers[j], np.float64).view(np.uint64)), f"MoM job {j}: {got} vs {answers[j]}"
