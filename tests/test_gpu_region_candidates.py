"""nph_region_candidates_batch (csrc/region_candidates.cu) and the host mirror's nph::get_variants_in_region against the reference's
AlignmentDB::get_variants_in_region: on every case of tests/candidate_cases.py the device's distinct variants, counts and depths equal
the plain-Python walk of tests/candidate_restatement.py (records entirely before start included), and the mirror's ordered list,
INFO bytes included, equals the compiled reference's (recorded in tests/golden/ref_region_candidates.pkl.xz by
tests/test_region_candidates_oracle.py).  Also: the call's counters, a first output capacity that is too small, every refusal, and
the sizes of the new ABI structs."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NPH_ERR_INVALID, NphError
from nanopolish_b200.engine import Engine
from tests import candidate_cases as cc
from tests import host_mirror as hm
from tests.ref_calls import case_answers

pytestmark = pytest.mark.gpu
GOLDEN = "ref_region_candidates.pkl.xz"
NPH_ERR_UNSUPPORTED = -6
host = hm.fixture()


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def cases():
    return {n: cc.build(n) for n in cc.CASES}


def device(eng, c, **kw):
    seq, deltas, recs = synth.seq_records(c["bases"], c["aligned"])
    return eng.region_candidates_batch(c["region_ref"], c["region_start"], seq if seq.shape[0] else np.zeros(1, np.uint8),
                                       deltas if deltas.shape[0] else np.zeros(1, np.int16), recs, c["start"], c["stop"], **kw), seq


def distinct_of(c, out, seq):
    got = {}
    for v in out:
        p, o = int(v["ref_position"]), int(v["alt_off"])
        key = (p, c["region_ref"][p - c["region_start"]:p - c["region_start"] + int(v["ref_len"])], bytes(seq[o:o + int(v["alt_len"])]).decode("latin-1"))
        assert key not in got, f"{c['name']}: {key} appears twice"
        got[key] = (int(v["count"]), int(v["depth"]))
    return got


@pytest.mark.parametrize("name", cc.CASES)
def test_device_equals_restatement(eng, cases, name):
    c = cases[name]
    (out, cnt), seq = device(eng, c)
    want = cc.restated(c)
    assert distinct_of(c, out, seq) == want
    assert int(cnt["n_records"]) == len(c["bases"]) and int(cnt["n_variants"]) == len(want)
    assert int(cnt["n_instances"]) == sum(n for n, _ in want.values())
    assert np.all(np.diff(out["ref_position"]) >= 0)


@pytest.mark.parametrize("name", cc.REF_CASES)
def test_mirror_equals_reference(host, cases, name):
    c = cases[name]
    want = case_answers(GOLDEN, name)[cc.fingerprint(c)]
    counts = np.zeros(1, synth.CANDIDATE_COUNTS_DT)
    n, got = cc.mirror(host, c, counts)
    assert n >= 0, host.nphh_last_error()
    assert got == want
    assert int(counts[0]["n_records"]) == len(c["bases"])


def test_counters_and_retry(eng, cases):
    c = cases["region_50k"]
    (out, cnt), _ = device(eng, c, cap=1)                                # a first cap of 1: the call says how many, and is retried
    (out2, cnt2), _ = device(eng, c)
    assert out.tobytes() == out2.tobytes()
    assert int(cnt["n_pairs"]) > 50 * 40_000 and cnt["kernel_ms"] > 0
    walked = 0
    for a in c["aligned"]:
        r = a[:, 0]
        walked += int(np.count_nonzero((r >= c["start"]) & (r < c["stop"])))
    assert int(cnt["n_pairs"]) == walked


def test_empty_inputs(eng):
    ref = "ACGT" * 20
    recs = np.zeros(0, synth.SEQ_RECORD_DT)
    out, cnt = eng.region_candidates_batch(ref, 100, np.zeros(1, np.uint8), np.zeros(1, np.int16), recs, 110, 170)
    assert out.shape[0] == 0 and int(cnt["n_instances"]) == 0


def _refused(eng, ref, rs, seq, deltas, recs, start, stop):
    with pytest.raises(NphError) as e:
        eng.region_candidates_batch(ref, rs, seq, deltas, recs, start, stop)
    return e.value


def test_refusals(eng, host):
    ref = "ACGTTGCA" * 20
    b, a, _ = cc.rec(ref, 1000, 1010, [("M", 30), ("X", 1), ("M", 30)])
    seq, deltas, recs = synth.seq_records([b], [a])
    assert "stop < start" in str(_refused(eng, ref, 1000, seq, deltas, recs, 1050, 1049))
    for s0, s1 in ((999, 1050), (1000, 1160), (1100, 1160)):
        assert "not inside" in str(_refused(eng, ref, 1000, seq, deltas, recs, s0, s1))
    eng.region_candidates_batch(ref, 1000, seq, deltas, recs, 1000, 1159)                 # the whole region is fine
    bad = recs.copy(); bad[0]["seq_len"] = len(b) - 1                                     # the last read position leaves the bases
    assert "read positions" in str(_refused(eng, ref, 1000, seq, deltas, bad, 1000, 1100))
    bad = recs.copy(); bad[0]["first_read_pos"] = -1
    assert "read positions" in str(_refused(eng, ref, 1000, seq, deltas, bad, 1000, 1100))
    d2 = deltas.copy(); d2[5] = 0                                                         # a read position that does not increase
    assert "read positions" in str(_refused(eng, ref, 1000, seq, d2, recs, 1000, 1100))
    bad = recs.copy(); bad[0]["seq_off"] = 1                                              # the bases leave their array
    assert "leave their arrays" in str(_refused(eng, ref, 1000, seq, deltas, bad, 1000, 1100))
    bad = recs.copy(); bad[0]["map_len"] += 1
    assert "leave their arrays" in str(_refused(eng, ref, 1000, seq, deltas, bad, 1000, 1100))
    # the mirror: an insertion of 32 767 bases fits the compact form, one of 32 768 does not; pairs that do not increase are refused
    c = dict(region_start=1000, region_ref=ref, rc=[0], start=1000, stop=1150, min_frequency=0.0, min_depth=0)
    for ins, status in ((32_766, 0), (32_767, NPH_ERR_UNSUPPORTED)):
        b, a, _ = cc.rec(ref, 1000, 1010, [("M", 30), ("I", "A" * ins), ("M", 30)])
        n, got = cc.mirror(host, dict(c, bases=[b], aligned=[a]))
        assert (n >= 0) if status == 0 else (n == status), host.nphh_last_error()
        if status == 0:
            assert [(g[0], len(g[2])) for g in got] == [(1039, ins + 1)]
    b, a, _ = cc.rec(ref, 1000, 1010, [("M", 30)])
    a = a[[0, 2, 1, 3]]
    assert cc.mirror(host, dict(c, bases=[b], aligned=[a]))[0] == NPH_ERR_INVALID
    assert cc.mirror(host, dict(c, bases=[b], aligned=[cc.rec(ref, 1000, 1010, [("M", 30)])[1]], start=1100, stop=1099))[0] == NPH_ERR_INVALID


def test_abi_sizes():
    assert synth.SEQ_RECORD_DT.itemsize == 32 and synth.REGION_CANDIDATE_DT.itemsize == 32 and synth.CANDIDATE_COUNTS_DT.itemsize == 40
    assert synth.SEQ_RECORD_DT.fields["first_read_pos"][1] == 28 and synth.REGION_CANDIDATE_DT.fields["alt_off"][1] == 24


@pytest.mark.parametrize("spec", cc.CALL_CASES, ids=[s[0] for s in cc.CALL_CASES])
def test_region_call_vcf_equals_reference(host, spec):
    c = cc.build_call(spec)
    want = case_answers(GOLDEN, spec[0])[cc.call_fingerprint(c)]
    n, got = cc.call_region(host, c)
    assert n >= 0, host.nphh_last_error()
    assert got == want


def test_region_call_refusals(host):
    c = cc.build_call(cc.CALL_CASES[2])
    for kw in (dict(start_base=c["end_base"] + 1), dict(start_base=c["contig_length"] - 39, end_base=c["contig_length"] + 5),
               dict(region_start=c["region_start"] + 1, region_ref=c["region_ref"][1:])):
        n, _ = cc.call_region(host, dict(c, **kw))
        assert n == NPH_ERR_INVALID, kw
    n, _ = cc.call_region(host, dict(c, candidates="ctg\t5100\n"))                  # read_vcf asserts on an empty REF
    assert n == NPH_ERR_INVALID
