"""The restatement of methylation-aware candidate screening (tests/var_meth_restatement.py) against the compiled reference's own
score_variant_thresholded with opt::methylation_types, on methylated pile-ups: every type list, early exit on and off, both
alignment-flag settings, forward and reverse reads, edits that create or destroy recognition sites, and windows with an N."""
import numpy as np
import pytest

from tests import var_meth_restatement as vmr
from tests.ref_types import _ref_types_session, ref_types  # noqa: F401  (fixtures)
from tests.screen_cases import N_AT, TYPE_LISTS, methylated_pileup, with_n

K = 6
REGION = 5000


def changes_sets(sets):
    return any(len(s) != len(sets[0]) for s in sets[1:])


@pytest.mark.parametrize("types", TYPE_LISTS, ids=[",".join(t) for t in TYPE_LISTS])
@pytest.mark.parametrize("threshold,flags", [(40, 0), (40, 3), (10 ** 6, 0), (10 ** 6, 3)])
def test_restatement_equals_reference(port_oracle, ref_types, types, threshold, flags):
    nuc, tm, ref, ref_chars, rs, recs, pairs = methylated_pileup(types, 110, 8, 90, seed=31 + len(types))
    ref_s = with_n(ref_chars).tobytes().decode()
    models = [nuc] + [tm[t] for t in types]
    # screenable positions whose base and left neighbour are not N
    cand_pos = [REGION + p for p in range(11, len(ref_s) - 11) if ref_s[p] != "N" and ref_s[p - 1] != "N"]
    got = vmr.position_scores(port_oracle, rs, models, types, ref_s, REGION, cand_pos, recs, pairs, 10, flags, 0.9, K)
    site_change = [i for i, g in zip(cand_pos, got) if g is not None and g[1] and changes_sets(g[2])]
    n_flank = [i for i, g in zip(cand_pos, got) if g is not None and g[1] and any(abs(i - (REGION + n)) <= 10 for n in N_AT)]
    assert len(site_change) >= 3 and len(n_flank) >= 2
    picked = sorted(set(site_change[::max(1, len(site_change) // 4)][:4] + n_flank[:2]))
    ref_types.clear_reads()
    rh = ref_types.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time)
    rcs = {int(recs[r]["rc"]) for i, g in zip(cand_pos, got) if i in picked for r, _, _ in g[1]}
    assert rcs == {0, 1}                                              # forward and reverse reads in the sample
    for i in picked:
        cands, seqs, sets, scores = got[cand_pos.index(i)]
        want, _ = vmr.accumulate(cands, seqs, sets, scores, threshold)
        cs, ce = i - 10, i + 11
        q = ref_types.score_variants_thresholded([rh[r] for r, _, _ in seqs], [(e1, e2) for _, e1, e2 in seqs],
                                             np.array([recs[r]["rc"] for r, _, _ in seqs], np.uint8), ref_s[cs - REGION:ce - REGION + 1],
                                             cs, [(REGION + off, rseq, aseq) for _, off, rseq, aseq in cands], flags, threshold, types,
                                             indel_bias=0.9)
        for (slot, _, _, _), v in zip(cands, q):
            assert np.float64(want[slot]).tobytes() == np.float64(v).tobytes(), (i, slot, want[slot], v)
    ref_types.clear_reads()


def test_score_set_fold_equals_host_combine():
    """the numpy fold against nph_score_set_combine (host code: the shared fold of exact_math.cuh), including -inf and large gaps"""
    import ctypes as C
    from nanopolish_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 5):
        s = rng.normal(-300.0, 6.0, (400, n)).astype(np.float32)
        s[::7, -1] = -np.inf
        s[::11, 0] -= 40.0
        out = np.zeros(400, np.float32)
        assert lib.nph_score_set_combine(s.ctypes.data_as(C.c_void_p), 400, n, out.ctypes.data_as(C.c_void_p)) == 0
        want = np.array([vmr.score_set(row) for row in s], np.float32)
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), n
