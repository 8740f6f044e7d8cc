"""nph_homopolymer_likelihoods_batch (csrc/homopolymer.cu) against the compiled reference's fix_homopolymers: on every case of
tests/hp_cases.py the device's two likelihood vectors and read count per homopolymer are bit-equal to the reference's (restated
over its own HMMs, tests/test_fix_homopolymers_oracle.py, recorded in tests/golden/ref_fix_homopolymers.pkl.xz), and the call rule
applied to them gives the reference's fixed haplotype, variant for variant; so does the host mirror's nph::fix_homopolymers
(nanopolish_b200/host/nph_variants.cpp) through its C shim.  Both insertions and deletions are called, and on the long-run pile-up
the duration term makes calls the event term alone would not.  Also: a batch cut into many chunks of Viterbi states gives the same
bits as one chunk; an empty pile-up and a haplotype without homopolymers; every refusal."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from nanopolish_b200.engine import Engine
from tests import host_mirror as hm
from tests import hp_cases as hc
from tests import hp_restatement as hr
from tests.ref_calls import case_answers

pytestmark = pytest.mark.gpu
GOLDEN = "ref_fix_homopolymers.pkl.xz"


host = hm.fixture()


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    yield e
    e.close()


def bits(v):
    return np.asarray(v, np.float64).view(np.uint64)


@pytest.mark.parametrize("spec", hc.CASES, ids=[s[0] for s in hc.CASES])
def test_likelihoods_and_fixed_haplotype_equal_reference(eng, spec):
    c = hc.build(spec)
    want_text, want_vectors = case_answers(GOLDEN, spec[0])[hc.fingerprint(c)]
    liks, cnt = hc.device(eng, c)
    got = hc.vectors_of(liks)
    assert len(got) == len(want_vectors) == len(c["wins"]) > 0
    for i, ((n, e, d), (wn, we, wd)) in enumerate(zip(got, want_vectors)):
        assert n == wn, f"window {i}: TotalReads"
        assert (bits(e) == bits(we)).all(), f"window {i}: event likelihoods {e} vs {we}"
        assert (bits(d) == bits(wd)).all(), f"window {i}: duration likelihoods {d} vs {wd}"
    assert int(cnt["n_pairs"]) == int(liks["scored_reads"].sum()) > 0 and int(cnt["n_jobs"]) == 7 * int(cnt["n_pairs"])
    fixed = hr.fix_homopolymers(c["hap"], c["wins"], got)
    assert hr.fixed_text(fixed, len(c["variants"])) == want_text
    if spec[0] == "long_runs":
        assert sum(hr.duration_decides(w, e, d) for w, (_, e, d) in zip(c["wins"], got)) >= 1
    calls = [l.split("\t") for l in want_text.split("\n")[1:] if l]
    if spec[0] in ("plain", "long_runs"):
        assert any(len(a) > len(r) for _, r, a, _, _ in calls) and any(len(a) < len(r) for _, r, a, _, _ in calls)


@pytest.mark.parametrize("spec", hc.CASES, ids=[s[0] for s in hc.CASES])
def test_host_mirror_fixed_haplotype_equals_reference(host, spec):
    c = hc.build(spec)
    want_text, _ = case_answers(GOLDEN, spec[0])[hc.fingerprint(c)]
    assert hc.mirror(host, c) == want_text


def test_many_chunks_equal_one(eng):
    c = hc.build(hc.CASES[0])
    one, cnt1 = hc.device(eng, c)
    many, cnt = hc.device(eng, c, max_chunk_pairs=7)
    assert int(cnt1["n_chunks"]) == 1 and int(cnt["n_chunks"]) == -(-int(cnt["n_pairs"]) // 7) > 1
    assert one.tobytes() == many.tobytes()


def test_empty_pileup_and_no_homopolymers(eng):
    c = hc.build(hc.CASES[0])
    none = c["recs"][:0]
    liks, cnt = eng.homopolymer_likelihoods_batch(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, c["dur"],
                                                  np.frombuffer(c["draft"].encode(), np.uint8).copy(), c["deltas"], c["first"][:0], none,
                                                  c["params"], c["seqs"], c["warr"])
    assert (liks["total_reads"] == 0).all() and (liks["scored_reads"] == 0).all() and int(cnt["n_pairs"]) == 0
    assert (liks["event_lik"] == 0).all() and (liks["duration_lik"] == 0).all()
    # with every read gone the scores are all 0: the argmax is L = 3 with score 0 < 10, nothing is called
    assert hr.fix_homopolymers(c["hap"], c["wins"], hc.vectors_of(liks)).seq == c["hap"].seq
    hap = hr.Haplotype(hc.REGION_START, "ACGT" * 100)
    assert hr.windows(hap, hc.REGION_START, hc.REGION_START + 399, 30) == []
    liks, cnt = eng.homopolymer_likelihoods_batch(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, c["dur"],
                                                  np.frombuffer(c["draft"].encode(), np.uint8).copy(), c["deltas"], c["first"], c["recs"],
                                                  c["params"], np.zeros(1, np.uint8), np.zeros(0, synth.HP_WINDOW_DT))
    assert liks.shape == (0,) and int(cnt["n_windows"]) == 0


def _refused(eng, c, warr=None, params=None, seqs=None):
    with pytest.raises(NphError) as ex:
        eng.homopolymer_likelihoods_batch(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, c["dur"],
                                          np.frombuffer(c["draft"].encode(), np.uint8).copy(), c["deltas"], c["first"], c["recs"],
                                          c["params"] if params is None else params, c["seqs"] if seqs is None else seqs,
                                          c["warr"] if warr is None else warr)
    assert ex.value.status == -3


def test_refusals(eng):
    c = hc.build(hc.CASES[0])
    w0 = c["warr"]

    def edit(field, value, i=0):
        w = w0.copy()
        w[i][field] = value
        return w

    _refused(eng, c, warr=edit("k", 5))                                        # the reference asserts a 6-mer model
    _refused(eng, c, warr=edit("hp_length", 2))
    _refused(eng, c, warr=edit("hp_length", 10))
    _refused(eng, c, warr=edit("edit_offset", int(w0[0]["seq_len"]) - int(w0[0]["hp_length"]) + 1))   # erase / insert outside
    _refused(eng, c, warr=edit("k0", int(w0[0]["seq_len"]) - int(w0[0]["hp_length"]) - 6))          # slot k0 + L + 1 past the k-mers
    _refused(eng, c, warr=edit("seq_len", int(c["seqs"].shape[0]) + 1))                            # outside calling_seqs
    _refused(eng, c, warr=edit("ref_calling_start", hc.REGION_START - 1))                          # outside the region
    _refused(eng, c, warr=edit("ref_calling_end", c["region_end"] + 1))
    _refused(eng, c, warr=edit("ref_calling_end", int(w0[0]["ref_calling_start"]) - 1))
    p = c["params"].copy()
    p[0]["min_flanking_sequence"] = 6
    _refused(eng, c, params=p)
    # the edges themselves are accepted
    w = edit("k0", int(w0[0]["seq_len"]) - int(w0[0]["hp_length"]) - 7)
    w[0]["edit_offset"] = int(w0[0]["seq_len"]) - int(w0[0]["hp_length"])
    w[0]["ref_calling_end"] = c["region_end"]
    liks, _ = eng.homopolymer_likelihoods_batch(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, c["dur"],
                                                np.frombuffer(c["draft"].encode(), np.uint8).copy(), c["deltas"], c["first"], c["recs"],
                                                c["params"], c["seqs"], w)
    assert liks.shape[0] == w.shape[0]
