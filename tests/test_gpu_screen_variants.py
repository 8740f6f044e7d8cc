"""nph_screen_variants_batch (csrc/screen_variants.cu) against the compiled reference's screen_variants_by_score: on every case of
tests/screen_cases.py the device's quality bits, read count and status per candidate equal the reference's (restated over its own
HMMs, tests/test_screen_variants_oracle.py, recorded in tests/golden/ref_screen_variants.pkl.xz), and the host mirror's
nph::screen_variants_by_score returns the reference's list.  Also: reads_per_round does not change a quality; random lists of about
2 000 candidates against the restatement over nph_hmm_score_batch's scores; the substitutions and insertions of nph_screen_edits_batch
bit for bit; the host mirror's expand_variants; an empty list, an empty pile-up and a list outside the region; every refusal."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from tests import host_mirror as hm
from tests import screen_cases as sc
from tests import screen_restatement as scr
from tests.ref_calls import case_answers

pytestmark = pytest.mark.gpu
GOLDEN = "ref_screen_variants.pkl.xz"


host = hm.fixture()


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))                       # model 0
    for t in sc.ALL_TYPES:                                               # models 1, 2, 3
        e.model_upload(sc.type_models([t])[t])
    yield e
    e.close()


def bits(v):
    return np.asarray(v, np.float64).view(np.uint64)


def _check(got, want):
    for i, (g, (q, n, st, _)) in enumerate(zip(got, want)):
        assert (int(g["n_reads"]), int(g["status"])) == (n, st), f"candidate {i}"
        assert bits(g["quality"]) == bits(q), f"candidate {i}: quality {g['quality']} vs {q}"


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_screen_equals_reference(eng, spec):
    c = sc.build(spec)
    lines, want = case_answers(GOLDEN, spec[0])[sc.fingerprint(c)]
    got, cnt = sc.device(eng, c)
    assert got.shape[0] == len(want) == len(c["candidates"])
    _check(got, want)
    assert scr.kept_lines(c["candidates"], [(float(g["quality"]), 0, int(g["status"]), 0) for g in got]) == lines
    assert int(cnt["n_candidates"]) == len(want)
    assert int(cnt["n_reference_rows"]) == sum(w[3] for w in want)
    assert int(cnt["n_jobs"]) <= int(cnt["n_jobs_without_exit"])


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_host_mirror_equals_reference(host, spec):
    c = sc.build(spec)
    lines, _ = case_answers(GOLDEN, spec[0])[sc.fingerprint(c)]
    n, got = sc.mirror(host, c)
    assert n >= 0, host.nphh_last_error()
    assert got == lines


@pytest.mark.parametrize("name", ["hp_truth", "meth_dam_dcm", "sparse_t1"])
def test_reads_per_round_does_not_change_a_quality(eng, name):
    c = sc.build(next(s for s in sc.CASES if s[0] == name))
    runs = [sc.device(eng, c, params_=sc.params(c, rpr)) for rpr in (1, 8, 1000)]
    for got, cnt in runs[1:]:
        assert np.array_equal(bits(got["quality"]), bits(runs[0][0]["quality"])) and np.array_equal(got["status"], runs[0][0]["status"])
        assert int(cnt["n_reference_rows"]) == int(runs[0][1]["n_reference_rows"])
    assert int(runs[0][1]["n_rounds"]) >= int(runs[2][1]["n_rounds"]) >= 1
    if name == "hp_truth":
        assert int(runs[0][1]["n_rounds"]) > int(runs[1][1]["n_rounds"]) > int(runs[2][1]["n_rounds"])


def random_case(seed, n=2000, flank=10, threshold=100, flags=sc.FLAGS):
    """a 20 kb pile-up at depth 10 and n random candidates: reference alleles of 0..3 draft bases (one in eight changed so that it
    does not apply), alternative alleles of 0..3 random bases, some windows past either end, in random order with repeats"""
    model = synth.load_model("nucleotide")
    draft, rs, recs, pairs, dur, deltas, first, _ = sc.suc._pileup(("snp", 20000, 10, 400, seed, 40), model)
    rng = np.random.default_rng(seed)
    lo, hi = sc.REGION_START, sc.REGION_START + len(draft) - 1
    cands = []
    for p in rng.integers(lo, hi - 2, n):
        r = draft[p - sc.REGION_START:p - sc.REGION_START + int(rng.integers(0, 4))]
        if rng.random() < 0.125:
            r = r[:-1] + sc._other(r[-1]) if r else "A"
        cands.append((int(p), r, "".join("ACGT"[x] for x in rng.integers(0, 4, int(rng.integers(0, 4))))))
    cands += cands[:50]
    c = dict(draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first, region_start=lo, region_end=hi, region_ref=draft,
             flank=flank, flags=flags, threshold=threshold, types=(), candidates=cands, truth=[])
    c["params"] = sc.params(c)
    return c


@pytest.mark.parametrize("seed,threshold,flags", [(81, 100, sc.FLAGS), (82, 25, 0)])
def test_random_list_equals_restatement(eng, seed, threshold, flags):
    c = random_case(seed, threshold=threshold, flags=flags)
    got, cnt = sc.device(eng, c)
    want = scr.screened(sc.plan(c), sc.hmm_scores(eng, c), threshold)
    _check(got, want)
    st = got["status"]
    assert (st == scr.OUTSIDE).any() and (st == scr.NOT_APPLIED).any() and (got["quality"][st == 0] < 0).any()
    assert int(cnt["n_jobs"]) < int(cnt["n_jobs_without_exit"])
    assert int(cnt["n_reference_rows"]) == sum(w[3] for w in want)
    assert int(cnt["n_windows"]) < int((st != scr.OUTSIDE).sum())                      # candidates share windows


@pytest.mark.parametrize("types", [(), ("cpg",), ("dam", "dcm")], ids=["none", "cpg", "dam_dcm"])
def test_edits_equal_the_edit_screen(eng, types):
    """a substitution or insertion at position i has the edit screen's window [i - flank, i + 1 + flank] and reads, so both calls
    give the same quality bits (with dam,dcm: sets of up to three sequences, through the edit screen's fixed rank pool and the list's
    variable one)"""
    if types:
        _, _, _, ref_chars, rs, recs, pairs = sc.methylated_pileup(list(types), 240, 10, 120, seed=91)
        draft = ref_chars.tobytes().decode()
        deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    else:
        draft, rs, recs, pairs, _, deltas, first, _ = sc.suc._pileup(("snp", 240, 12, 120, 91, 8), synth.load_model("nucleotide"))
    c = dict(draft=draft, rs=rs, recs=recs, pairs=pairs, deltas=deltas, first=first, region_start=sc.REGION_START,
             region_end=sc.REGION_START + len(draft) - 1, region_ref=draft, flank=10, flags=sc.FLAGS, threshold=100, types=types)
    c["params"] = sc.params(c, 3)
    ref = np.frombuffer(draft.encode(), np.uint8).copy()
    meth = sc.meth_arg(c)
    q, nr, _ = eng.screen_edits_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs,
                                      synth.screen_params(sc.REGION_START, 6, 10, 100, sc.FLAGS, 3), methylation=meth)
    cands, slots = [], []
    for pi in range(10, 210):
        b = draft[pi]
        for j, x in enumerate("ACGT"):
            if x != b:
                cands += [(sc.REGION_START + pi, b, x), (sc.REGION_START + pi, b, b + x)]
                slots += [(pi, 2 * j), (pi, 2 * j + 1)]
    got, _ = sc.device(eng, c, candidates=cands)
    assert (got["status"] == scr.SCREENED).all()
    for g, (pi, s) in zip(got, slots):
        assert bits(g["quality"]) == bits(q[pi, s]) and int(g["n_reads"]) == int(nr[pi]), (pi, s)


def test_host_mirror_expand_equals_reference(host):
    for name, base, min_flank in sc.EXPAND:
        c = sc.build(next(s for s in sc.CASES if s[0] == base))
        cands = sc.expand_candidates(c)
        want = case_answers(GOLDEN, name)[sc.fingerprint(c) + repr((cands, min_flank))]
        n, got = sc.host_expand(host, c, cands, min_flank)
        assert n >= 0, host.nphh_last_error()
        assert got == want
    # another contig: no extended deletion; a foreign ref_seq: the reference asserts
    n, got = sc.host_expand(host, c, [(c["region_start"] + 50, "AC", "A")], 10, var_contig="other")
    assert n >= 0 and len(got) == 5
    p = c["region_start"] + 50
    n, _ = sc.host_expand(host, c, [(p, sc._other(c["draft"][p - sc.REGION_START]) + "A", "A")], 10)
    assert n == -3 and b"not the region's" in host.nphh_last_error()


def test_empty_list_empty_pileup_and_outside(eng, host):
    c = sc.build(sc.CASES[0])
    got, cnt = sc.device(eng, c, candidates=[])
    assert got.shape == (0,) and int(cnt["n_candidates"]) == 0 and int(cnt["n_jobs"]) == 0
    n, lines = sc.mirror(host, c, candidates=[])
    assert n == 0 and lines == []
    rs = c["rs"]
    alleles, cands = sc.candidate_array(c["candidates"])
    got, cnt = eng.screen_variants_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(),
                                         c["deltas"], c["first"][:0], c["recs"][:0], c["params"], alleles, cands)
    assert (got["n_reads"] == 0).all() and (got["quality"][got["status"] != scr.OUTSIDE] == 0.0).all() and int(cnt["n_jobs"]) == 0
    F, hi = c["flank"], c["region_end"]
    got, cnt = sc.device(eng, c, candidates=[(F - 1, "A", "C"), (hi - F, "A", "C"), (hi, "", "T")])
    assert (got["status"] == scr.OUTSIDE).all() and np.isnan(got["quality"]).all() and int(cnt["n_windows"]) == 0


def _refused(eng, c, message, candidates=None, params_=None, methylation="case"):
    with pytest.raises(NphError) as ex:
        sc.device(eng, c, candidates=candidates, params_=params_, methylation=methylation)
    assert ex.value.status == -3 and message in str(ex.value), str(ex.value)


def test_refusals(eng):
    c = sc.build(sc.CASES[0])

    def params(**kw):
        p = c["params"].copy()
        for k, v in kw.items():
            p[0][k] = v
        return p
    _refused(eng, c, "not a nucleotide model of k = params.k", params_=params(k=5))
    _refused(eng, c, "k outside 1..8", params_=params(k=9))
    _refused(eng, c, "2 * flank + 1 below k", params_=params(flank=2))
    _refused(eng, c, "reads_per_round is 0", params_=params(reads_per_round=0))
    _refused(eng, c, "unknown alignment_flags", params_=params(alignment_flags=4))
    _refused(eng, c, "outside 0..INT32_MAX", candidates=[(2 ** 31 - 11, "A", "C")])
    rs = c["rs"]
    alleles, cands = sc.candidate_array([(c["region_start"] + 30, "A", "C")])
    cands[0]["alt_seq_off"] = alleles.shape[0]
    with pytest.raises(NphError) as ex:
        eng.screen_variants_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(), c["deltas"],
                                  c["first"], c["recs"], c["params"], alleles, cands)
    assert "an allele outside alleles" in str(ex.value)
    # the -q checks of nph_screen_load_methylation
    meth, ids = synth.screen_methylation(["cpg"], 6), np.ones((c["recs"].shape[0], 1), np.uint32)
    _refused(eng, c, "k != params.k", methylation=(synth.screen_methylation(["cpg"], 5), ids))
    _refused(eng, c, "out of range or not a model of that alphabet", methylation=(meth, ids * 9))
