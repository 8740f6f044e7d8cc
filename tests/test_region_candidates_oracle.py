"""The compiled reference's own AlignmentDB::get_variants_in_region (src/alignment/nanopolish_alignment_db.cpp:259-368, run
unmodified by oracle/call_harness.cpp) against the plain-Python walk of tests/candidate_restatement.py on every case of
tests/candidate_cases.py that the reference is defined on: the kept variants' positions and, per position, the multiset of
(ref_seq, alt_seq, INFO), and the full order wherever no position repeats.  Each case asserts the edge it was built to reach; the
sort_ties case shows that the reference's order among variants at one position is not key order (std::sort's ties reach the
output).  The reference's answers are kept in tests/golden/ref_region_candidates.pkl.xz for the device suite
(tests/test_gpu_region_candidates.py) and for machines without the reference."""
import collections

import pytest

from tests import candidate_cases as cc
from tests import candidate_restatement as cr
from tests.ref_calls import case_fixture

ref_cand = case_fixture("ref_region_candidates.pkl.xz", ref=lambda: cc.RefCand() if cc.RefCand.available() else None)


def restated_lines(c):
    """the restatement's kept variants, in key order, with the reference's INFO"""
    return [(p, r, a, f"BaseCalledReadsWithVariant={n};BaseCalledFraction={cc.fmt(n / d)}")
            for p, r, a, n, d in cr.kept(cc.restated(c), c["min_frequency"], c["min_depth"])]


def by_position(lines):
    out = collections.defaultdict(collections.Counter)
    for p, *rest in lines:
        out[p][tuple(rest)] += 1
    return dict(out)


@pytest.mark.parametrize("name", cc.REF_CASES)
def test_restatement_equals_reference(ref_cand, name):
    c = cc.build(name)
    cc.claims(c, cc.restated(c))
    want = ref_cand.answers(name, [cc.fingerprint(c)], lambda _: ref_cand.live.variants(c))[0]
    got = restated_lines(c)
    assert [w[0] for w in want] == sorted(g[0] for g in got), f"{name}: positions differ"
    assert by_position(want) == by_position(got), f"{name}: the variants at some position differ"
    if len({w[0] for w in want}) == len(want):
        assert want == sorted(got, key=lambda g: g[0]), f"{name}: the order differs"
    if name == "sort_ties":
        assert len(want) > 16 and max(collections.Counter(w[0] for w in want).values()) >= 2
        key_order = sorted(got, key=lambda g: g[0])                      # stable: key order inside each position
        assert want != key_order, "sort_ties: the reference's order equals key order; the case does not reach std::sort's ties"
    if name == "deep_pile":
        assert want[0][3].endswith("BaseCalledFraction=5e-05")
    if name == "freq_float":
        assert not any(w[0] == 5060 for w in want)                       # 1/5 < 0.2f widened to double
    if name == "freq_double":
        assert any(w[0] == 5060 and w[3].endswith("BaseCalledFraction=0.2") for w in want)


def test_fraction_format():
    """cc.fmt is std::stringstream << double's default output on the fractions the cases reach"""
    assert [cc.fmt(x) for x in (1 / 3, 1.0, 5e-05, 0.2, 2 / 7)] == ["0.333333", "1", "5e-05", "0.2", "0.285714"]


@pytest.mark.parametrize("spec", cc.CALL_CASES, ids=[s[0] for s in cc.CALL_CASES])
def test_reference_region_call(ref_cand, spec):
    """the reference's default-mode region call and VCF (npref_call_region), recorded for the device suite; each case reaches its edge"""
    c = cc.build_call(spec)
    vcf = ref_cand.answers(spec[0], [cc.call_fingerprint(c)], lambda _: cc.ref_call_region(ref_cand.live.call, c))[0]
    lines = vcf.decode().splitlines()
    records = [l.split("\t") for l in lines if not l.startswith("#")]
    end = min(c["end_base"], c["contig_length"] - 1)
    assert lines[0] == "##fileformat=VCFv4.2" and lines[1] == f"##nanopolish_window=ctg:{c['start_base']}-{end}"
    assert any("ID=SupportFractionByBase" in l for l in lines) == bool(c["all_support"])
    assert records and all(r[7].split(";")[-1].startswith("RefContext=") for r in records)
    if c["snps_only"]:
        assert all(len(r[3]) == 1 and len(r[4]) == 1 for r in records)
    if c["candidates"] is None:
        assert all("BaseCalledFraction=" in r[7] for r in records)
    else:
        assert not any("BaseCalledFraction=" in r[7] for r in records)
    if spec[0].startswith("vcf_50k"):
        assert len(records) >= 20 and {r[9] for r in records} == ({"1"} if c["ploidy"] == 1 else {"0/1", "1/1"} & {r[9] for r in records} or {"1/1"})
