"""nph_all_support_batch (csrc/all_support.cu) against the compiled reference's annotate_variants_with_all_support: on every case of
tests/support_cases.py the device's four support fractions, read count and apply_variant outcome per variant are bit-equal to the
reference's (restated over its own HMMs, tests/test_all_support_oracle.py, recorded in tests/golden/ref_all_support.pkl.xz), and the
host mirror's nph::annotate_variants_with_all_support (nanopolish_b200/host/nph_variants.cpp) writes the reference's INFO byte for
byte.  Also: a large random batch against the restatement over nph_hmm_score_batch's scores; an empty variant list and an empty
pile-up; every refusal, by its message."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from oracle.oracle_py import PortOracle
from tests import support_cases as sc
from tests import support_restatement as sr
from tests.ref_calls import case_answers
from tests.test_host_mirror import HOST_SO

pytestmark = pytest.mark.gpu
GOLDEN = "ref_all_support.pkl.xz"


@pytest.fixture(scope="module")
def host():
    lib = C.CDLL(HOST_SO)
    lib.nphh_last_error.restype = C.c_char_p
    return lib


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    yield e
    e.close()


def bits(v):
    return np.asarray(v, np.float64).view(np.uint64)


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_support_equals_reference(eng, spec):
    c = sc.build(spec)
    want = case_answers(GOLDEN, spec[0])[sc.fingerprint(c)]
    got, cnt = sc.device(eng, c)
    assert got.shape[0] == len(want) == len(c["variants"])
    for i, (g, (info, sup, n, applied)) in enumerate(zip(got, want)):
        assert int(g["n_reads"]) == n, f"variant {i}: read count"
        assert bool(g["applied"]) == applied, f"variant {i}: apply_variant"
        assert (bits(g["support"]) == bits(sup)).all(), f"variant {i}: support {g['support']} vs {sup}"
        assert sr.info(g["support"]) == info
    assert int(cnt["n_variants"]) == len(want) and int(cnt["n_pairs"]) == int(got["n_reads"].sum())
    assert int(cnt["n_jobs"]) == 4 * int(cnt["n_pairs"]) and int(cnt["n_dp_rows"]) >= int(cnt["n_jobs"])


@pytest.mark.parametrize("spec", sc.CASES, ids=[s[0] for s in sc.CASES])
def test_host_mirror_info_equals_reference(host, spec):
    c = sc.build(spec)
    want = case_answers(GOLDEN, spec[0])[sc.fingerprint(c)]
    n, infos = sc.mirror(host, c)
    assert n >= 0, host.nphh_last_error()
    assert infos == [w[0] for w in want]


def _hmm_scores(eng, c):
    """score_jobs of sc.restated through nph_hmm_score_batch: each haplotype's k-mer ranks on the job's strand"""
    def score(jobs, seqs):
        ranks, off = [], 0
        for j, s in enumerate(seqs):
            codes = synth.encode(s, "nucleotide")
            r = synth.dna_rc_kmer_ranks(codes, 6) if jobs[j]["rc"] else synth.kmer_ranks_from_codes(codes, 6, 4)
            jobs[j]["rank_off"], jobs[j]["n_kmers"] = off, r.shape[0]
            ranks.append(r)
            off += r.shape[0]
        rs = c["rs"]
        return eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.concatenate(ranks).astype(np.uint32), jobs)
    return score


@pytest.mark.parametrize("seed,flags", [(61, sc.FLAGS), (62, 0)])
def test_random_batch_equals_restatement(eng, seed, flags):
    c = sc.random_case(seed, flags=flags)
    got, cnt = sc.device(eng, c)
    port = PortOracle()
    want = sc.restated(c, _hmm_scores(eng, c), port.lib.npo_logsum)
    assert int(cnt["n_pairs"]) > 2000
    assert any(len(r) == 0 for _, r, _ in c["variants"]) and not all(w[2] for w in want)
    for i, (g, (sup, n, applied, _)) in enumerate(zip(got, want)):
        assert (int(g["n_reads"]), bool(g["applied"])) == (n, applied), f"variant {i}"
        assert (bits(g["support"]) == bits(sup)).all(), f"variant {i}: {g['support']} vs {sup}"


def test_empty_variant_list_and_empty_pileup(eng, host):
    c = sc.build(sc.CASES[0])
    got, cnt = sc.device(eng, c, variants=[])
    assert got.shape == (0,) and int(cnt["n_variants"]) == 0 and int(cnt["n_pairs"]) == 0
    n, infos = sc.mirror(host, c, variants=[])
    assert n == 0 and infos == []
    rs = c["rs"]
    got, cnt = eng.all_support_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(),
                                     c["deltas"], c["first"][:0], c["recs"][:0], c["params"], c["ref_seqs"], c["varr"])
    assert (got["n_reads"] == 0).all() and int(cnt["n_pairs"]) == 0
    assert (bits(got["support"]) == bits(np.full(4, -np.nan))).all()
    assert all(sr.info(g["support"]) == "SupportFractionByBase=-nan,-nan,-nan,-nan" for g in got)


def _refused(eng, c, message, variants=None, params=None):
    with pytest.raises(NphError) as ex:
        sc.device(eng, c, variants=variants, params=params)
    assert ex.value.status == -3 and message in str(ex.value), str(ex.value)


def test_refusals(eng, host):
    c = sc.build(sc.CASES[3])                                                   # edges_f30: windows touching both region ends
    F, lo, hi = c["flank"], c["region_start"], c["region_end"]
    b = c["draft"][lo + F - sc.REGION_START]
    sc.device(eng, c, variants=[(lo + F, b, "A"), (hi - F, "A", "C")])          # the edges themselves are accepted
    _refused(eng, c, "outside the region", variants=[(lo + F - 1, b, "A")])     # substr_by_reference asserts
    _refused(eng, c, "outside the region", variants=[(hi - F + 1, "A", "C")])
    _refused(eng, c, "outside the region", variants=[(F - 1, "A", "C")])       # a negative calling_start
    ref_seqs, varr = sc.variant_array([(lo + F, b, "A")])
    varr[0]["ref_seq_len"] = ref_seqs.shape[0] + 1
    with pytest.raises(NphError) as ex:
        rs = c["rs"]
        eng.all_support_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(), c["deltas"],
                              c["first"], c["recs"], c["params"], ref_seqs, varr)
    assert "ref_seq outside ref_seqs" in str(ex.value)

    def params(**kw):
        p = c["params"].copy()
        for k, v in kw.items():
            p[0][k] = v
        return p
    _refused(eng, c, "not a nucleotide model of k = 5", params=params(k=5))
    _refused(eng, c, "k outside 1..8", params=params(k=9))
    _refused(eng, c, "flank + 1 below k", params=params(flank=4))
    _refused(eng, c, "unknown alignment_flags", params=params(alignment_flags=4))
    # the host mirror: a variant on another contig (get_event_subsequences asserts), and the device's refusals
    n, _ = sc.mirror(host, c, var_contig="other")
    assert n == -3 and b"another contig" in host.nphh_last_error()
    n, _ = sc.mirror(host, c, variants=[(hi - F + 1, "A", "C")])
    assert n == -3 and b"outside the region" in host.nphh_last_error()
