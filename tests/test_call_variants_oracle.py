"""The compiled reference's own call_haplotype_from_candidates (src/nanopolish_call_variants.cpp:782-880, run unmodified by
oracle/variants_harness.cpp) against the restatement in tests/call_restatement.py over the reference's profile_hmm_score: the derived
sequence and, per variant, position, alleles, quality bits, INFO and genotype on every case of tests/call_cases.py (INFO without
SupportFractionByBase, which is not restated).  Each case asserts the edges it was built to reach.  Also: the host mirror's Fisher test
against the reference's kt_fisher_exact on every table of at most 60 reads and on large and underflowing tables, and the visit orders of
the reference's Combinations generator.  The reference's answers are kept in tests/golden/ref_call_haplotype.pkl.xz for the device
suite (tests/test_gpu_call_variants.py) and for machines without the reference."""
import hashlib
import itertools

import numpy as np
import pytest

from tests import call_cases as cc
from tests import call_restatement as cr
from tests import host_mirror as hm
from tests.ref_calls import case_fixture
from tests.ref_variants import RefVariants

ref_call = case_fixture("ref_call_haplotype.pkl.xz", ref=lambda: RefVariants() if RefVariants.available() else None)

# large tables, and tables whose probabilities underflow (StrandFisherTest clamps those to 1000)
BIG_TABLES = [(500, 3, 7, 900), (2000, 1, 1, 2000), (0, 1000, 1000, 0), (1000, 0, 0, 1000), (33, 77, 121, 11), (250, 250, 250, 250),
              (4000, 2, 3, 4000), (1, 3000, 2999, 2)]


@pytest.mark.parametrize("spec", cc.CASES, ids=[s[0] for s in cc.CASES])
def test_restatement_equals_reference(ref_call, spec):
    c = cc.build(spec)
    live = ref_call.live

    def ask(_):
        hs, mh = live.register(c)
        want = live.called(c, hs)
        got = cc.ref_restated(live, c, hs, mh)
        assert got == (cc.strip_all_support(want) if c["all_support"] else want), f"{spec[0]}: the restated call differs from the reference's"
        return want

    lines = ref_call.answers(spec[0], [cc.fingerprint(c)], ask)[0]
    _assert_edges_reached(spec[0], c, lines)


def _assert_edges_reached(name, c, lines):
    """each case reaches the edges it was built for (the comparison with the reference above then covers them)"""
    calls = [l.split("\t") for l in lines[1:]]
    assert len(lines[0]) == len(c["region_ref"]) + sum(len(f[2]) - len(f[1]) for f in calls)
    groups = cr.groups(c["candidates"], cc.FLANK, cc.MIN_DISTANCE)
    if c["genotype_only"]:
        assert any(f[3] == "0" * 16 and "AlleleCount=0" in f[4] for f in calls)            # emitted with var_count 0
    if not c["genotype_only"]:
        assert all("AlleleCount=0" not in f[4] for f in calls)
    assert (";SupportFractionByBase=" in lines[-1]) == bool(c["all_support"] and calls)
    if name.startswith("truth"):
        assert len(calls) >= 3 and len({f[5] for f in calls}) >= 1
    if name.startswith("cluster"):
        sizes = [e - f for f, e, _, _ in groups]
        assert max(sizes) == 10
        if name != "cluster_p2_h1000":
            assert min(sizes) == (2 if name == "cluster_p3_h4" else 1)
    if name == "edges_p2":
        widths = [ce - cs for _, _, cs, ce in groups]
        assert 200 in widths and 201 in widths
        assert any(e - f == 1 for f, e, _, _ in groups)                                      # the group with one combination
        ps = [p for p, _, _ in c["candidates"]]
        assert any(b < a for a, b in zip(ps, ps[1:])) and len(set(c["candidates"])) < len(c["candidates"])
    if name == "sparse_p2":
        assert any("TotalReads=0" in f[4] and f[5] == "." for f in calls) and any("TotalReads=1;" in f[4] for f in calls)
    if name == "keys_p2":
        keys = sorted(n + ":0" for n in set(c["names"]))
        assert keys != [n + ":0" for n in sorted(set(c["names"]))]                             # key order is not name order
        assert c["recs"].shape[0] > len(set(int(r) for r in c["recs"]["read"]))                # a read aligned twice
    if name.endswith("_p1"):
        assert all(f[5] in ("0", "1", ".") for f in calls)
    if name == "cluster_p3_h4":
        assert all(len(f[5]) == 5 or f[5] == "." for f in calls)


def _tables(n_max):
    for a in range(n_max + 1):
        for b in range(n_max + 1 - a):
            for cc_ in range(n_max + 1 - a - b):
                for d in range(n_max + 1 - a - b - cc_):
                    yield a, b, cc_, d


def _fisher_answers(fisher):
    bits = np.array([fisher(*t) for t in _tables(60)], np.float64).view(np.uint64)
    return hashlib.sha256(bits.tobytes()).hexdigest(), [int(np.float64(fisher(*t)).view(np.uint64)) for t in BIG_TABLES]


def test_fisher_equals_reference(ref_call):
    host = hm.load()
    want = ref_call.answers("fisher", [repr((60, BIG_TABLES))], lambda _: _fisher_answers(ref_call.live.fisher))[0]
    assert _fisher_answers(host.nphh_fisher_exact) == tuple(want)
    # the restatement the device suite uses, on a sample of the tables and the large ones
    for t in list(_tables(24))[::7] + BIG_TABLES:
        assert np.float64(cr.fisher_two(*t)) == np.float64(host.nphh_fisher_exact(*t)), t


def test_combination_orders(ref_call):
    """Combinations visits r-subsets and ploidy-multisets in lexicographic order (as itertools lists them): the order the host's
    enumerator and the device's set ranks follow"""
    shapes = [(n, k, w) for n in range(1, 10) for k in range(0, 5) for w in (0, 1) if k <= n]
    want = ref_call.answers("combinations", [repr(shapes)], lambda _: [ref_call.live.combinations(n, k, w) for n, k, w in shapes])[0]
    for (n, k, w), got in zip(shapes, want):
        gen = itertools.combinations_with_replacement if w else itertools.combinations
        assert [list(x) for x in gen(range(n), k)] == got, (n, k, w)
