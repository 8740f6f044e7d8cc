"""Methylation-aware candidate screening on the device (`variants -q ...`) — nph_screen_edits_batch_methylation /
nph_screen_load_methylation (csrc/variants.cu) against the restatement (tests/var_meth_restatement.py, pinned to the compiled reference
in tests/test_variants_methylation_oracle.py) and against the compiled reference itself."""
import math

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from tests import var_meth_restatement as vmr
from tests import var_restatement as vr
from tests.ref_types import _ref_types_session, ref_types  # noqa: F401  (fixtures)
from tests.screen_cases import N_AT, TYPE_LISTS, methylated_pileup, type_models, with_n

pytestmark = pytest.mark.gpu
K = 6
REGION = 5000
ALL_TYPES = ("cpg", "dam", "dcm")
NPH_ERR_INVALID, NPH_ERR_STATE, NPH_ERR_UNSUPPORTED = -3, -5, -6


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))                       # model 0
    for name, m in type_models(ALL_TYPES).items():                      # models 1, 2, 3
        e.model_upload(m)
    yield e
    e.close()


def meth_arg(types, n_records):
    ids = np.array([[1 + ALL_TYPES.index(t) for t in types]] * n_records, np.uint32).reshape(n_records, len(types))
    return synth.screen_methylation(types, K), ids


def run(eng, types, ref_chars, rs, recs, pairs, threshold, flags, rpr):
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    params = synth.screen_params(REGION, K, 10, threshold, flags, rpr)
    q, nr, scored = eng.screen_edits_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref_chars, deltas, first, recs, params, indel_bias=0.9,
                                           methylation=meth_arg(types, recs.shape[0]))
    return q, nr, scored, eng.screen_counts(), (deltas, first, params)


def same(a, b):
    return np.float64(a).tobytes() == np.float64(b).tobytes() or (math.isnan(a) and math.isnan(b))


@pytest.mark.parametrize("types", TYPE_LISTS, ids=[",".join(t) for t in TYPE_LISTS])
def test_every_position_and_counter_equals_restatement(eng, port_oracle, types):
    threshold, flags, rpr = 40, 3, 3
    nuc, tm, ref, ref_chars, rs, recs, pairs = methylated_pileup(types, 130, 10, 100, seed=71 + len(types))
    q, nr, scored, cnt, (deltas, first, params) = run(eng, types, ref_chars, rs, recs, pairs, threshold, flags, rpr)
    ref_s = ref_chars.tobytes().decode()
    n_pos = ref.shape[0] - 1
    models = [nuc] + [tm[t] for t in types]
    got = vmr.position_scores(port_oracle, rs, models, types, ref_s, REGION, [REGION + p for p in range(n_pos)], recs, pairs, 10, flags, 0.9, K)
    jobs = rows = no_exit = rounds = 0
    ref_rows = np.zeros(n_pos, np.uint64)
    differ = two_alts = 0
    for pi, g in enumerate(got):
        if g is None:
            assert np.isnan(q[pi]).all(), pi
            continue
        cands, seqs, sets, scores = g
        want, rrows = vmr.accumulate(cands, seqs, sets, scores, threshold)
        for c in range(9):
            assert same(float(q[pi, c]), want[c]), (pi, c, q[pi], want)
        assert int(nr[pi]) == len(seqs)
        ref_rows[pi] = rrows
        j, ev, rd, ne = vmr.device_accounting(cands, seqs, sets, scores, threshold, rpr)
        jobs += j; rows += ev; no_exit += ne; rounds = max(rounds, rd)
        if seqs:
            differ += sum(len(s) != len(sets[0]) for s in sets[1:])
            two_alts += sum(len(s) == 3 for s in sets)
    assert scored == cnt["scored_events"] == rows
    assert cnt["jobs"] == jobs and cnt["jobs_without_exit"] == no_exit and cnt["rounds"] == rounds
    assert cnt["reference_events"] == int(ref_rows.sum())
    # the data exercises the feature: edits change the set size, both types meet in one window, and the early exit saves work
    assert differ >= 20, differ
    if len(types) == 2:
        assert two_alts >= 1
    assert rounds >= 2 and cnt["jobs"] < cnt["jobs_without_exit"]
    # the staged form, with the reference rows per position
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.screen_load(ref_chars, deltas, first, recs, params, indel_bias=0.9, methylation=meth_arg(types, recs.shape[0]))
    eng.screen_run()
    q2, nr2, rows2 = eng.screen_fetch(with_reference_rows=True)
    assert np.array_equal(q.view(np.uint64), q2.view(np.uint64)) and np.array_equal(nr, nr2)
    assert np.array_equal(rows2, ref_rows) and eng.screen_counts() == cnt


@pytest.mark.parametrize("types", TYPE_LISTS, ids=[",".join(t) for t in TYPE_LISTS])
def test_windows_with_n_and_compiled_reference(eng, port_oracle, ref_types, types):
    nuc, tm, ref, ref_chars, rs, recs, pairs = methylated_pileup(types, 110, 8, 90, seed=31 + len(types))
    chars = with_n(ref_chars)
    q, nr, scored, cnt, _ = run(eng, types, chars, rs, recs, pairs, 40, 0, 4)
    ref_s = chars.tobytes().decode()
    models = [nuc] + [tm[t] for t in types]
    # positions whose base or left neighbour is N: the nucleotide path's own (pre-existing) candidate rule, not compared here
    pos = [REGION + p for p in range(1, len(ref_s) - 1) if ref_s[p] != "N" and ref_s[p - 1] != "N"]
    got = vmr.position_scores(port_oracle, rs, models, types, ref_s, REGION, pos, recs, pairs, 10, 0, 0.9, K)
    near_n = 0
    for i, g in zip(pos, got):
        pi = i - REGION
        if g is None:
            assert np.isnan(q[pi]).all()
            continue
        want, _ = vmr.accumulate(g[0], g[1], g[2], g[3], 40)
        for c in range(9):
            assert same(float(q[pi, c]), want[c]), (pi, c, q[pi], want)
        near_n += any(abs(pi - n) <= 10 for n in N_AT)
    assert near_n >= 10
    # a sample straight through the compiled reference's score_variant_thresholded with these types
    ref_types.clear_reads()
    rh = ref_types.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time)
    for pi in (24, 40, 66, 80):
        i = REGION + pi
        cs, ce = i - 10, i + 11
        seqs = vr.event_sequences(recs, pairs, cs, ce)
        cands = vr.candidates(ref_s, pi)
        v = ref_types.score_variants_thresholded([rh[r] for r, _, _ in seqs], [(e1, e2) for _, e1, e2 in seqs],
                                             np.array([recs[r]["rc"] for r, _, _ in seqs], np.uint8), ref_s[cs - REGION:ce - REGION + 1], cs,
                                             [(REGION + off, rseq, aseq) for _, off, rseq, aseq in cands], 0, 40, types, indel_bias=0.9)
        for (slot, _, _, _), x in zip(cands, v):
            assert same(float(q[pi, slot]), float(x)), (pi, slot)
    ref_types.clear_reads()


def test_no_types_equals_nucleotide_screening(eng):
    nuc = synth.load_model("nucleotide")
    ref, rs, recs, pairs = synth.gen_pileup(150, 12, 110, nuc, seed=13, region_start=REGION, n_true_variants=3)
    ref_chars = synth._CODE2DNA[ref]
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    params = synth.screen_params(REGION, K, 10, 40, 3, 4)
    args = (rs.reads, rs.ev_mean, rs.ev_start_time, ref_chars, deltas, first, recs, params)
    q1, nr1, s1 = eng.screen_edits_batch(*args, indel_bias=0.9)
    c1 = eng.screen_counts()
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.screen_load(ref_chars, deltas, first, recs, params, indel_bias=0.9)
    eng.screen_run()
    _, _, rows1 = eng.screen_fetch(with_reference_rows=True)
    none = (synth.screen_methylation([], K), np.zeros((recs.shape[0], 0), np.uint32))
    q2, nr2, s2 = eng.screen_edits_batch(*args, indel_bias=0.9, methylation=none)
    c2 = eng.screen_counts()
    eng.screen_load(ref_chars, deltas, first, recs, params, indel_bias=0.9, methylation=none)
    eng.screen_run()
    _, _, rows2 = eng.screen_fetch(with_reference_rows=True)
    assert np.array_equal(q1.view(np.uint64), q2.view(np.uint64)) and np.array_equal(nr1, nr2) and s1 == s2
    assert c1 == c2 and c1["rounds"] >= 2 and np.array_equal(rows1, rows2)


def test_refusals_leave_run_in_state_error(eng):
    nuc, tm, ref, ref_chars, rs, recs, pairs = methylated_pileup(["dam"], 90, 6, 80, seed=5)
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    params = synth.screen_params(REGION, K, 10, 40, 0, 4)
    n = recs.shape[0]
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)

    def refused(meth, ids, status):
        eng.screen_load(ref_chars, deltas, first, recs, params)                # a good load first: the refusal must undo it
        with pytest.raises(NphError) as e:
            eng.screen_load(ref_chars, deltas, first, recs, params, methylation=(meth, ids))
        assert e.value.status == status
        assert eng.lib.nph_screen_run(eng.ctx) == NPH_ERR_STATE

    m, ids = meth_arg(["dam"], n)
    too_many = synth.screen_methylation(["dam"], K)
    too_many[0]["n_types"] = 5
    refused(too_many, np.full((n, 5), 2, np.uint32), NPH_ERR_INVALID)
    bad_symbol = m.copy()
    bad_symbol[0]["alphabets"][0]["complements"] = b"TGCXA"
    refused(bad_symbol, ids, NPH_ERR_INVALID)
    overlapping = m.copy()
    a = overlapping[0]["alphabets"][0]
    a["site_len"], a["sites"][0], a["sites_methylated"][0], a["sites_methylated_complement"][0] = 2, b"AA", b"MA", b"TM"
    refused(overlapping, ids, NPH_ERR_UNSUPPORTED)
    other_k = synth.screen_methylation(["dam"], 5)
    refused(other_k, ids, NPH_ERR_INVALID)
    refused(m, np.full((n, 1), 9, np.uint32), NPH_ERR_INVALID)              # no such model
    refused(m, np.full((n, 1), 0, np.uint32), NPH_ERR_INVALID)              # the nucleotide model is not a dam model
    # and a good load still runs
    eng.screen_load(ref_chars, deltas, first, recs, params, methylation=(m, ids))
    eng.screen_run()
