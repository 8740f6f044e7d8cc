"""The compiled reference's own annotate_variants_with_all_support (src/common/nanopolish_variant.cpp:801-859, run unmodified by
oracle/variants_harness.cpp) against the restatement in tests/support_restatement.py over the reference's profile_hmm_score and add_logs:
the SupportFractionByBase INFO of every variant, byte for byte, on the cases of tests/support_cases.py.  Each case asserts the
edges it was built to reach.  The reference's INFO and the restated support fractions, read counts and apply_variant outcomes are
kept in tests/golden/ref_all_support.pkl.xz for the device suite (tests/test_gpu_all_support.py).  Also: the restatement refuses a
window one base past either region end, where the reference asserts."""
import numpy as np
import pytest

from tests import forward_cases as fc
from tests import hp_restatement as hr
from tests import support_cases as sc
from tests.ref_calls import case_fixture
from tests.ref_variants import RefVariants

ref_sup = case_fixture("ref_all_support.pkl.xz", ref=lambda: RefVariants() if RefVariants.available() else None)


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_restatement_equals_reference(ref_sup, spec):
    c = sc.build(spec)
    live = ref_sup.live

    def ask(_):
        hs, mh = live.register(c)
        want = live.infos(c, hs)
        got = sc.ref_restated(live, c, hs, mh)
        assert [g[3] for g in got] == want, f"{spec[0]}: the restated INFO differs from the reference's"
        return [(w, np.asarray(g[0], np.float64), g[1], g[2]) for w, g in zip(want, got)]

    rows = ref_sup.answers(spec[0], [sc.fingerprint(c)], ask)[0]
    assert len(rows) == len(c["variants"]) > 0
    for info, *_ in rows:
        assert info.startswith("SupportFractionByBase=") and info.count(",") == 3
    _assert_edges_reached(spec[0], c, rows)


def _assert_edges_reached(name, c, rows):
    """each case reaches the edges it was built for (the comparison with the reference above then covers them)"""
    F = c["flank"]
    plan = sc.plan(c)
    n_reads = [r[2] for r in rows]
    assert n_reads == [len(ev) for _, _, ev in plan]
    applied = [r[3] for r in rows]
    assert applied == [a for _, a, _ in plan]
    vs = c["variants"]
    if name in ("snp_truth", "hp_truth", "wide_f170"):
        # the truth's edits, read on both strands
        assert len(vs) >= 3 and all(applied)
        assert any({int(c["recs"][r]["rc"]) for r, _, _ in ev} == {0, 1} for _, _, ev in plan)
    if name == "hp_truth":
        assert any(len(r) > 1 for _, r, _ in vs) and any(len(a) > 1 for _, _, a in vs)      # deletions and insertions
    if name.startswith("edges"):
        pos = [p for p, _, _ in vs]
        assert c["region_start"] + F in pos and c["region_end"] - F in pos                # windows touching both region ends
        assert {r for (_, r, _), a in zip(vs, applied) if len(r) == 1 and a} == set("ACGT")
        by_len = {len(r): a for (_, r, _), a in zip(vs, applied)}
        assert by_len[4] and by_len[3] and by_len[F + 1] and not by_len[F + 2]
        assert any(r.islower() and not a for (_, r, _), a in zip(vs, applied))             # a case-only mismatch
        assert any(len(r) == 1 and r.isupper() and not a for (_, r, _), a in zip(vs, applied))
        assert any(len(a) > 1 and ap for (_, _, a), ap in zip(vs, applied))                  # an insertion, applied as a substitution
        assert len(set(vs)) < len(vs) and pos != sorted(pos)                                 # a duplicate, an unsorted list
        # a read whose alignment bounds the window at one end only (get_event_subsequences skips it)
        recs = c["recs"]
        lo, hi = recs["ref_start_pos"].astype(np.int64), recs["ref_start_pos"].astype(np.int64) + recs["ref_len"] - 1
        assert any(((lo > p - F) & (lo <= p + F) & (hi > p + F)).any() for p in pos)
    if name == "sparse_f10":
        assert 0 in n_reads and 1 in n_reads
        assert all(info == "SupportFractionByBase=-nan,-nan,-nan,-nan" for info, *_ in (r for r in rows if r[2] == 0))
    if name == "dense_f10":
        dropped = sum(len(hr.event_sequences(c["recs"], c["pairs"], p - F, p + F, float("inf"))) - n for (p, _, _), n in zip(vs, n_reads))
        assert dropped >= 1
    if name == "wide_f170":
        # every job of the case runs in the chained class, across strips
        K = 2 * F + 1 - 6 + 1
        for _, _, ev in plan:
            for _, e1, e2 in ev:
                (C, W, chained), _ = fc.choose_class(K, abs(e1 - e2) + 1)
                assert chained and K > C * W
    assert {s[3] for s in sc.CASES} == {7, 10, 30, 170} and {s[4] for s in sc.CASES} == {0, sc.FLAGS}


@pytest.mark.parametrize("spec", [s for s in sc.CASES if s[5] == "edges"], ids=[s[0] for s in sc.CASES if s[5] == "edges"])
def test_restatement_refuses_windows_past_the_region(spec):
    c = sc.build(spec)
    F = c["flank"]
    region = hr.Haplotype(c["region_start"], c["region_ref"])
    for p in (c["region_start"] + F, c["region_end"] - F):
        sc.sr.window(region, p, F)
    for p in (c["region_start"] + F - 1, c["region_end"] - F + 1, F - 1):
        with pytest.raises(hr.RefAbort):
            sc.sr.window(region, p, F)
