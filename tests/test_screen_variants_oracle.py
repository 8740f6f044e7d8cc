"""The compiled reference's own screen_variants_by_score and expand_variants (src/nanopolish_call_variants.cpp:364-450, run unmodified by
oracle/variants_harness.cpp) against the restatement in tests/screen_restatement.py over the reference's profile_hmm_score: the output
list (positions, alleles, quality bits, empty INFO) on every case of tests/screen_cases.py, and expand_variants' list.  Each case
asserts the edges it was built to reach.  The reference's lists and the restated quality, read count, status and DP rows of every
candidate are kept in tests/golden/ref_screen_variants.pkl.xz for the device suite (tests/test_gpu_screen_variants.py)."""
import numpy as np
import pytest

from tests import hp_restatement as hr
from tests import screen_cases as sc
from tests import screen_restatement as scr
from tests.ref_calls import case_fixture
from tests.ref_variants import RefVariants

ref_screen = case_fixture("ref_screen_variants.pkl.xz", ref=lambda: RefVariants() if RefVariants.available() else None)


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_restatement_equals_reference(ref_screen, spec):
    c = sc.build(spec)
    live = ref_screen.live

    def ask(_):
        hs, mh = live.register(c)
        want = live.screened(c, hs)
        got = sc.ref_restated(live, c, hs, mh)
        assert scr.kept_lines(c["candidates"], got) == want, f"{spec[0]}: the restated list differs from the reference's"
        return want, [(np.float64(q), n, st, rows) for q, n, st, rows in got]

    lines, rows = ref_screen.answers(spec[0], [sc.fingerprint(c)], ask)[0]
    assert len(rows) == len(c["candidates"]) > 0
    assert lines == scr.kept_lines(c["candidates"], rows)
    _assert_edges_reached(spec[0], c, lines, rows)


def _assert_edges_reached(name, c, lines, rows):
    """each case reaches the edges it was built for (the comparison with the reference above then covers them)"""
    F = c["flank"]
    pl = sc.plan(c)
    vs = c["candidates"]
    q = [r[0] for r in rows]
    st = [r[2] for r in rows]
    assert [r[1] for r in rows] == [0 if x is None else len(x[3]) for x in pl]
    assert st == [scr.OUTSIDE if x is None else x[0] for x in pl]
    if name in ("snp_truth", "hp_truth"):
        # the truth's edits pass, the wrong ones beside them score below zero; reads on both strands
        assert len(lines) >= 3 and sum(x < 0 for x in q) >= 3
        assert any({int(c["recs"][r]["rc"]) for r, _, _ in x[3]} == {0, 1} for x in pl if x)
    if name == "hp_truth":
        assert any(len(r) > 1 for _, r, _ in vs) and any(len(a) > 1 for _, _, a in vs)        # deletions and insertions
    if name == "snp_truth_t0":
        assert lines == [] and all(x == 0.0 for x, s in zip(q, st) if s != scr.OUTSIDE)      # threshold 0: nothing is scored
    if name.startswith("edges"):
        lo, hi = c["region_start"], c["region_end"]
        cs = {(p - F, p + len(r) + F): s for (p, r, _), s in zip(vs, st)}
        assert st.count(scr.OUTSIDE) >= 2 and any(k[0] == lo and s != scr.OUTSIDE for k, s in cs.items())
        assert any(k[1] == hi and s != scr.OUTSIDE for k, s in cs.items())
        assert any(k[0] == lo - 1 for k in cs) and any(k[1] == hi + 1 for k in cs)
        na = [(v, x) for v, x, s in zip(vs, q, st) if s == scr.NOT_APPLIED]
        assert any(r.islower() for (_, r, _), _ in na) and any(r.isupper() for (_, r, _), _ in na)   # case-only and exact mismatch
        assert all(x == 0.0 for _, x in na)
        ok = [v for v, s in zip(vs, st) if s == scr.SCREENED]
        assert any(len(r) >= 3 and len(a) == 1 for _, r, a in ok) and any(len(a) >= 3 for _, _, a in ok)
        assert any(r == "" for _, r, _ in ok) and any(a == "" for _, _, a in ok) and ("", "") in [(r, a) for _, r, a in ok]
        by_pos = {}
        for p, r, _ in ok:
            by_pos.setdefault(p, set()).add(len(r))
        assert any(len(s) >= 3 for s in by_pos.values())                                    # ref lengths 1, 2, 3 at one position
        pos = [p for p, _, _ in vs]
        assert len(set(vs)) < len(vs) and pos != sorted(pos)
        if name == "edges_f30":
            assert any(x < 0 for x in q)
    if name == "sparse_t1":
        n_reads = [r[1] for r in rows]
        assert 0 in n_reads and 1 in n_reads
        # threshold 1: the early exit stops most candidates after their first read
        assert any(abs(x) >= 1 and n > 1 and rr < sum((2 * (abs(e1 - e2) + 1)) for _, e1, e2 in pl[i][3])
                   for i, (x, n, _, rr) in enumerate(rows))
    if name == "dense_f10":
        dropped = sum(len(hr.event_sequences(c["recs"], c["pairs"], p - F, p + len(r) + F, float("inf"))) - n
                      for (p, r, _), (_, n, _, _) in zip(vs, rows))
        assert dropped >= 1
    if name.startswith("meth"):
        # edits that make or break a site: the variant's set has another size than the base's
        assert sum(len(x[1]) != len(x[2]) for x in pl if x and x[3]) >= 3
        if len(c["types"]) == 2:
            assert any(len(x[1]) == 3 or len(x[2]) == 3 for x in pl if x)
    assert {s[3] for s in sc.CASES} == {3, 10, 30} and {s[4] for s in sc.CASES} == {0, sc.FLAGS}
    assert {s[5] for s in sc.CASES} == {0, 1, 25, 100, 10 ** 9} and {s[6] for s in sc.CASES} == {(), ("cpg",), ("dam", "dcm")}


def _expand_case(name):
    base = next(s for s in sc.CASES if s[0] == name)
    return sc.build(base)


@pytest.mark.parametrize("spec", sc.EXPAND, ids=[s[0] for s in sc.EXPAND])
def test_expand_equals_reference(ref_screen, spec):
    name, base, min_flank = spec
    c = _expand_case(base)
    cands = sc.expand_candidates(c)
    want = sc.expand_lines(scr.expand(sc.CONTIG, c["region_start"], c["region_ref"], cands, min_flank))

    def ask(_):
        return ref_screen.live.expanded(c["region_start"], c["region_ref"], cands, min_flank)

    got = ref_screen.answers(name, [sc.fingerprint(c) + repr((cands, min_flank))], ask)[0]
    assert got == want
    # the deletion min_flank + 1 bases from the end is extended, the one min_flank bases from it is not
    hi = c["region_end"]
    ext = {(p, len(r)) for p, r, _ in scr.expand(sc.CONTIG, c["region_start"], c["region_ref"], cands, min_flank)}
    assert (hi - 33, 3) in ext and (hi - 32, 3) not in ext
    assert len(got) > len(cands)


def test_restatement_expand_refuses_a_foreign_ref_seq():
    c = _expand_case("hp_truth")
    p = c["region_start"] + 50
    with pytest.raises(hr.RefAbort):
        scr.expand(sc.CONTIG, c["region_start"], c["region_ref"], [(p, sc._other(c["draft"][p - sc.REGION_START]) + "A", "A")], 10)
