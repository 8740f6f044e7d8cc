"""nph_call_variant_groups_batch (csrc/call_variants.cu) and the host mirror's nph::call_haplotype_from_candidates against the compiled
reference's call_haplotype_from_candidates: on every case of tests/call_cases.py the mirror's derived sequence, and each variant's
position, alleles, quality bits, INFO bytes and genotype, equal the reference's (recorded in tests/golden/ref_call_haplotype.pkl.xz by
tests/test_call_variants_oracle.py).  Also: two random 20 kb regions at ploidy 1 and 2, and a group of 968 haplotypes at ploidy 2,
against the restatement (tests/call_restatement.py, its genotype search a numpy brute force) over nph_hmm_score_batch's scores; the
device call's counters; an empty candidate list, an empty pile-up, and every refusal by its message."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from tests import call_cases as cc
from tests import call_restatement as cr
from tests import host_mirror as hm
from tests import screen_cases as sc
from tests.ref_calls import case_answers

pytestmark = pytest.mark.gpu
GOLDEN = "ref_call_haplotype.pkl.xz"


host = hm.fixture()


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))                       # model 0
    for t in sc.ALL_TYPES:                                               # models 1, 2, 3
        e.model_upload(sc.type_models([t])[t])
    yield e
    e.close()


@pytest.mark.parametrize("spec", cc.CASES, ids=[s[0] for s in cc.CASES])
def test_mirror_equals_reference(host, spec):
    c = cc.build(spec)
    want = case_answers(GOLDEN, spec[0])[cc.fingerprint(c)]
    st, got = cc.mirror(host, c)
    assert st >= 0, host.nphh_last_error()
    assert got[0] == want[0], f"{spec[0]}: derived sequence"
    assert got[1:] == want[1:]


def _random_case(seed, ploidy, ref_len=20000):
    kind = ("snp", ref_len, 8, 1500, seed, ref_len // 150)
    c = cc.build((f"random_{seed}", kind, ploidy, 0, 64, (), 0, "truth", "plain"))
    rng = np.random.default_rng(seed)
    d = lambda p: c["draft"][p - cc.REGION_START]
    extra = [(int(p), d(int(p)), "ACGT"[(int("ACGT".index(d(int(p)))) + int(rng.integers(1, 4))) % 4])
             for p in rng.integers(cc.REGION_START + 40, cc.REGION_START + ref_len - 60, ref_len // 100)]
    c["candidates"] = sorted(c["candidates"] + extra)
    return c


@pytest.mark.parametrize("seed,ploidy", [(501, 1), (502, 2)])
def test_random_region_equals_restatement(host, eng, seed, ploidy):
    c = _random_case(seed, ploidy)
    st, got = cc.mirror(host, c)
    assert st >= 0, host.nphh_last_error()
    want = cc.restated(c, cc.hmm_scores(eng, c))
    assert got[0] == want[0]
    assert got[1:] == want[1:]
    assert len(got) > 40


def test_dam_dcm_equals_restatement(host, eng):
    """-q dam,dcm on the planted-site pile-up: sets of up to three sequences per haplotype"""
    c = cc.build(("meth_dam_dcm_p2", ("meth", 130, 10, 100, 73), 2, 1, 64, ("dam", "dcm"), 0, "meth", "plain"))
    st, got = cc.mirror(host, c)
    assert st >= 0, host.nphh_last_error()
    assert got == cc.restated(c, cc.hmm_scores(eng, c))
    assert len(got) > 3


def test_thousand_haplotypes_equal_brute_force(host, eng):
    """one group of 10 variants with max_haplotypes 1000: 968 haplotypes, 468 996 sets at ploidy 2"""
    c = cc.build(("h1000", ("snp", 700, 8, 240, 6, 10), 2, 1, 1000, (), 0, "cluster10", "plain"))
    combos = cr.combinations(c["candidates"], cr.Hap(c["region_ref"][c["candidates"][0][0] - 30 - cc.REGION_START:], c["candidates"][0][0] - 30), 1000)
    assert len(combos) == 968
    st, got = cc.mirror(host, c)
    assert st >= 0, host.nphh_last_error()
    assert got == cc.restated(c, cc.hmm_scores(eng, c))
    # and through the engine: the counters
    g, v, cnt = cc.device(eng, c)
    assert int(cnt["n_groups"]) == 1 and int(cnt["n_haplotypes"]) == 968 and int(cnt["n_sets"]) == 968 * 969 // 2
    assert int(cnt["n_set_terms"]) == int(cnt["n_sets"]) * int(g[0]["n_keys"]) and int(g[0]["n_keys"]) > 0
    assert float(cnt["forward_ms"]) > 0 and float(cnt["genotype_ms"]) > 0


def test_device_call_statuses_and_empty_inputs(eng):
    c = cc.build(cc.CASES[1])
    g, v, cnt = cc.device(eng, c)
    assert g.shape[0] > 3 and set(int(x) for x in g["status"]) <= {synth.CALL_CALLED, synth.CALL_BASE_KEPT}
    assert (g["status"] == synth.CALL_CALLED).any()
    called = g[g["status"] == synth.CALL_CALLED]
    assert (called["best_score"] - called["base_score"] >= 20).all()
    assert int(cnt["n_jobs"]) > 0 and int(cnt["n_dp_rows"]) > 0 and float(cnt["host_ms"]) >= 0
    assert v["emit"].all()                                               # genotype_all
    # no candidate: nothing to do
    p, _, h, b, cv, _, kr = cc.device_inputs(c)
    rs = c["rs"]
    deltas, first = synth.compact_event_alignment(c["recs"], c["pairs"], int(c["recs"]["ref_len"].sum()))
    g0, v0, cnt0 = eng.call_variant_groups_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(),
                                                 deltas, first, c["recs"], kr, p, np.zeros(0, synth.CALL_GROUP_DT), h, b, cv, 0)
    assert g0.shape[0] == 0 and int(cnt0["n_groups"]) == 0
    # an empty pile-up: no key, every set scores 0, the base set is kept, TotalReads 0
    ge, ve, cnte = cc.device(eng, c, recs=c["recs"][:0])
    assert (ge["n_keys"] == 0).all() and (ge["status"] == synth.CALL_BASE_KEPT).all() and (ge["base_score"] == 0).all()
    assert (ve["var_count"] == 0).all() and int(cnte["n_jobs"]) == 0


def test_refusals(eng):
    c = cc.build(cc.CASES[1])
    p, g, h, b, cv, nv, kr = cc.device_inputs(c)

    def refused(msg, **kw):
        with pytest.raises(NphError, match=msg):
            cc.device(eng, c, **kw)

    q = p.copy(); q["ploidy"] = 0
    refused("ploidy outside", params=q)
    q = p.copy(); q["ploidy"] = synth.CALL_MAX_PLOIDY + 1
    refused("ploidy outside", params=q)
    q = p.copy(); q["alignment_flags"] = 4
    refused("unknown alignment_flags", params=q)
    q = p.copy(); q["k"] = 9
    refused("k outside", params=q)
    x = g.copy(); x[0]["n_haplotypes"] = 1
    refused("fewer than 2 haplotypes", groups=x)
    q = p.copy(); q["ploidy"] = 8
    refused("fewer haplotypes than the ploidy", params=q)
    x = g.copy(); x[0]["hap_first"] = h.shape[0]
    refused("haplotypes outside", groups=x)
    x = g.copy(); x[-1]["var_first"] = nv
    refused("variants outside", groups=x)
    x = g.copy(); x[0]["calling_start"] = c["region_start"] - 1
    refused("outside the region", groups=x)
    x = g.copy(); x[0]["calling_end"] = c["region_start"] + len(c["region_ref"])
    refused("outside the region", groups=x)
    y = h.copy(); y[1]["seq_off"] = b.shape[0]
    refused("haplotype_bases", haplotypes=y)
    y = h.copy(); y[1]["var_off"] = cv.shape[0]
    refused("variant ids outside", haplotypes=y)
    y = h.copy(); y[0]["n_var"] = 1
    refused("combination 0", haplotypes=y)
    z = cv.copy(); z[0] = 99
    refused("variant id outside", cvars=z)
    r = c["recs"].copy(); r[0]["model_id"] = 1                          # a cpg model where a nucleotide model belongs
    with pytest.raises(NphError, match="not a nucleotide model"):
        cc.device(eng, c, recs=r)
    m = synth.screen_methylation(["cpg"], 6)
    with pytest.raises(NphError, match="out of range or not a model"):
        cc.device(eng, c, methylation=(m, np.full((c["recs"].shape[0], 1), 99, np.uint32)))
