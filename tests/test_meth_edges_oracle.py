"""Pin the call-methylation restatement (tests/meth_restatement.py), scored by the port oracle, to the compiled reference's
calculate_methylation_for_read and TSV writer on every reference-parameter case of tests/meth_edge_cases.py: the same
groups, bit-identical scores and the same rows byte for byte.  The cases' edge claims are checked and printed here, and each
boundary comparison of the restatement, moved by one, must disagree with the reference on some case, which shows that the
cases sit on those boundaries.

The reference's answers live in tests/golden/ref_meth_edges.pkl.xz, one row per case: a fingerprint of the case's inputs and
the answer (a ref_calls.CaseRecord: asked live where oracle/_ref/libnpref.so exists and compared with the record, replayed
elsewhere).  NPH_REF_CASES_RECORD=<dir> pytest tests/test_meth_edges_oracle.py writes a new record to <dir>."""
import os
import re

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import meth_edge_cases as ec
from tests import ref_calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = os.path.join(ROOT, "nanopolish_b200", "csrc", "methylation.cu")
HEADER = os.path.join(ROOT, "include", "nph.h")

reference = ref_calls.case_fixture("ref_meth_edges.pkl.xz")

# (boundary, shift): every comparison the reference can reach, moved by one base each way that changes an answer
MOVED = [("separation", -1), ("separation", 1), ("sub_start", -1), ("sub_start", 1), ("max_span", -1), ("max_span", 1),
         ("event_span", -1), ("event_span", 1), ("region_start", -1), ("region_start", 1), ("region_end", -1), ("region_end", 1),
         ("substr", -1)]
# the site test q + rl <= L of the methylated copy: with the reference's parameters (min_flank == min_separation) no window
# ends on or cuts a site of another group, so this one is moved against the restatement's own answer on the cases with a wider
# flank, which the device suite compares with the device.  Moved by -1 it drops a site flush with the window's end; moved by +1
# it methylates a site cut by the window's end, reading the base past it
MOVED_OWN = [("site_fit", -1), ("site_fit", 1)]


@pytest.fixture(scope="module")
def cases():
    rs, built = ec.build(ec.all_cases())
    return rs, built, ec.models()


def _restated(port, rs, mods, b, moved=None):
    g = ec.restated(b, moved)
    return ec.answer(b, g, ec.score(port, rs, mods, b, g))


def _reference_answers(reference, rs, built):
    live = reference.live
    ref = [b for b in built if b.case.reference_case]
    handles = None
    if live is not None:
        live.clear_reads()
        for a in ec.ALPHABETS:
            live.builtin_model(a)
        handles = live.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, live.builtin_model("nucleotide"))
    return ref, reference.answers("meth_edges", [ec.fingerprint(rs, b) for b in ref], lambda i: ec.ask_reference(live, handles, rs, ref[i]))


def test_kernel_constants():
    """the warps per block, grid cap, ballot width, row chunk and window limit meth_edge_cases.py builds around are the kernels'"""
    src = open(KERNEL).read()
    assert re.search(r"constexpr int kWarps = (\d+);", src).group(1) == str(ec.WARPS)
    caps = re.findall(r"\(size_t\)ctx->sm_count \* (\d+)\)", src)
    assert len(caps) == 4 and set(caps) == {str(ec.GRID_PER_SM)}          # expand; scan and emit; fill; both row passes
    assert re.search(r"const int fgrid = .*\+ 255\) / 256", src) and "meth_fill_kernel<<<fgrid, 256" in src
    # the scan, the compact expansion and warp_first_valid step 32 bases at a time, the row writer 32 rows
    assert len(re.findall(r"base < n; base \+= (\d+)\)", src)) == 3 and set(re.findall(r"base < n; base \+= (\d+)\)", src)) == {str(ec.CHUNK)}
    assert re.search(r"base < s1; base \+= (\d+)\)", src).group(1) == str(ec.CHUNK)
    assert re.search(r"while \(hi - lo > (\d+)\)", src).group(1) == str(ec.CHUNK)
    assert re.search(r"#define NPH_METH_MAX_WINDOW (\d+)", open(HEADER).read()).group(1) == str(ec.MAX_WINDOW)


def test_every_claim_holds(cases):
    rs, built, _ = cases
    out = ec.check_claims(built) + ec.check_claims(ec.build(ec.refusal_cases())[1])
    print()
    for name, claim, ok in out:
        print(f"  {'ok ' if ok else 'NO '} {name}: {claim}")
    assert all(ok for _, _, ok in out), [n for n, _, ok in out if not ok]
    assert len({b.case.name for b in built}) == len(built)


def test_lower_bound_restatement_is_bisect():
    """warp_lower_bound's rounds, restated, equal bisect_left for every n <= 200, at the round edges and past them"""
    rng = np.random.default_rng(3)
    for n in list(range(0, 201)) + [1023, 1024, 1025, 1055, 1056, 1057, 1058, 32767, 32768, 32769]:
        vals = np.sort(rng.choice(4 * n + 8, n, replace=False)).tolist()
        for v in set(vals[:: max(1, n // 40)]) | {-1, 0, 4 * n + 9} | {x + 1 for x in vals[:: max(1, n // 40)]}:
            ec.lower_bound_trace(vals, v)
    assert ec.lower_bound_trace(list(range(32)), 5)[2] == 0 and ec.lower_bound_trace(list(range(33)), 5)[2] == 1
    assert ec.lower_bound_trace(list(range(1056)), 5)[2] == 1 and ec.lower_bound_trace(list(range(1057)), 5)[2] == 2


def test_cases_match_reference(cases, reference, port_oracle):
    rs, built, mods = cases
    ref, answers = _reference_answers(reference, rs, built)
    assert len(ref) >= 45 and {b.case.alphabet for b in ref} == set(ec.ALPHABETS)
    n_rows = 0
    for b, want in zip(ref, answers):
        got = _restated(port_oracle, rs, mods, b)
        assert got[0] == want[0], f"{b.case.name}: rows differ\n{got[0]}\n{want[0]}"
        assert ref_calls.same(got[1], want[1]), f"{b.case.name}: groups {got[1].tolist()} vs {want[1].tolist()}"
        assert ref_calls.same(got[2], want[2]), f"{b.case.name}: scores {got[2].tolist()} vs {want[2].tolist()}"
        n_rows += want[1].shape[0]
    assert n_rows > 300


@pytest.mark.parametrize("name,shift", MOVED)
def test_moved_boundary_disagrees_with_reference(cases, reference, port_oracle, name, shift):
    rs, built, mods = cases
    ref, answers = _reference_answers(reference, rs, built)
    differs = []
    for b, want in zip(ref, answers):
        got = _restated(port_oracle, rs, mods, b, {name: shift})
        if got[0] != want[0] or not ref_calls.same(got[1], want[1]) or not ref_calls.same(got[2], want[2]):
            differs.append(b.case.name)
    print(f"\n  {name} {shift:+d}: differs on {differs}")
    assert differs, f"moving {name} by {shift:+d} changes no answer of the reference"


@pytest.mark.parametrize("name,shift", MOVED_OWN)
def test_moved_boundary_disagrees_with_restatement(cases, port_oracle, name, shift):
    rs, built, mods = cases
    differs = []
    for b in built:
        if b.case.params:
            want, got = _restated(port_oracle, rs, mods, b), _restated(port_oracle, rs, mods, b, {name: shift})
            if got[0] != want[0] or not ref_calls.same(got[2], want[2]):
                differs.append(b)
    print(f"\n  {name} {shift:+d}: differs on {[b.case.name for b in differs]}")
    # every alphabet has a called window its neighbour's site is flush with (-1) or cut by (+1), on both strands.  The one
    # exception is cut cpg on the reverse strand: the window keeps only the site's C, and M and C both complement to G there
    want = {(a, rc) for a in ec.ALPHABETS for rc in (0, 1)} - ({("cpg", 1)} if shift > 0 else set())
    assert {(b.case.alphabet, b.rc) for b in differs} == want


@pytest.mark.parametrize("rev", [False, True])
def test_compact_form_step_limits(rev):
    """synth.compact_event_alignment takes event-index steps of +-32 767 and refuses +-32 768 (NPH_METH_NO_PAIR is -32 768)"""
    for step, ok in ((32767, True), (32768, False)):
        s = -step if rev else step
        pr = np.zeros(3, synth.PAIR_DT)
        pr["ref_pos"] = [100, 101, 102]
        pr["read_pos"] = np.array([40000, 40000 + s, 40000 + s + 1]) if not rev else np.array([40000, 40000 + s, 40000 + s - 1])
        rec = np.zeros(1, synth.METH_RECORD_DT)
        rec[0]["ref_len"], rec[0]["n_pairs"], rec[0]["ref_start_pos"] = 10, 3, 95
        if ok:
            d, f = synth.compact_event_alignment(rec, pr, 10)
            assert int(f[0]) == 40000 and d.tolist()[5:8] == [0, s, 1 if not rev else -1]
            assert (d == synth.METH_NO_PAIR).sum() == 7
        else:
            with pytest.raises(OverflowError):
                synth.compact_event_alignment(rec, pr, 10)
