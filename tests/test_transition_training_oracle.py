"""The compiled reference's model_score with --train-transitions (src/nanopolish_scorereads.cpp:116-203, run unmodified by
oracle/scorereads_harness.cpp), then TransitionParameters::train() and print(), against the restatement in
tests/transition_restatement.py over the reference's own profile_hmm_score and profile_hmm_align: the per-read score, every
training count and the skip-bin histogram, the trained probabilities and print()'s bytes.  Each case asserts the edges it was built
for.  The reference's answers are kept in tests/golden/ref_transitions_edges.pkl.xz for the device suite
(tests/test_gpu_transition_training.py)."""
import numpy as np
import pytest

from tests import transition_restatement as tr
from tests import tt_cases as tc
from tests.ref_calls import case_fixture

ref_tt = case_fixture("ref_transitions_edges.pkl.xz", ref=lambda: tc.RefTT() if tc.RefTT.available() else None)


@pytest.mark.parametrize("spec", tc.CASES, ids=[s[0] for s in tc.CASES])
def test_restatement_equals_reference(ref_tt, spec):
    c = tc.build(spec)
    live = ref_tt.live
    state = {}

    def ask(_):
        want = live.model_score(c)
        trace = []
        score, counts, paths = live.restated(c, trace)
        prior = live.prior_r9() if c["prior"] else None
        assert score == want[0], f"{spec[0]}: model_score's score differs from the restatement's"
        assert np.array_equal(counts, want[1]), f"{spec[0]}: training counts differ"
        assert tr.train(counts, prior) == list(want[2]), f"{spec[0]}: trained probabilities differ"
        assert want[3] == "".join(f"skip_probabilities[{b}] = {p:.3f};\n" for b, p in enumerate(want[2]))
        state.update(trace=trace, paths=paths, prior=prior)
        return want[0], want[1], want[2], want[3], (np.zeros(0) if prior is None else prior)

    score, counts, probs, text, prior = ref_tt.answers(spec[0], [tc.fingerprint(c)], ask)[0]
    if ref_tt.live is None:
        return                                               # replay: the record's own checks ran when it was recorded
    _assert_edges_reached(spec[0], c, state["trace"], state["paths"], counts, score)


def _assert_edges_reached(name, c, trace, paths, counts, score):
    obs = [t for t in trace if t[0] == "obs"]
    lens = {len(p) for p in paths}
    prevs = {t[6] for t in obs if t[5] == "K"}
    if name in ("plain", "rc", "drift", "prior", "stalled", "wide_scale"):
        assert counts[tr.SKIPS] > 0 and counts[tr.MATCHES] > 0
        # K after M (to = from + 1) and after K; the interior limits pi = 6 and size - 6 hold observations, pi = 5 and size - 5 not
        if name == "plain":
            assert {"M", "K", "B"} <= prevs
        interior = {t[1] for t in trace if t[0] == "interior"}
        assert 6 in interior and 5 not in interior
        assert any(len(p) - 6 in interior and len(p) - 5 not in interior for p in paths)
        assert any(p[i][2] == "B" and p[i + 1][2] == "B" for p in paths for i in range(len(p) - 1))     # B runs
    if name == "short_paths":
        assert lens == {4} and counts.sum() == 0                      # paths of <= 5 states record nothing
    if name == "short_paths4":
        assert {5, 6} <= lens
        assert counts[:18].sum() > 0                                  # a 6-state path records its transitions, once each
    if name == "wide_scale":
        assert any(t[4] == 29 and t[7] >= 15.0 for t in obs)          # clamped to the last bin
    if name == "stalled":
        _, skipped = tr.segments(c["align"], c["contig"], 0, c["eps"], tc.K)
        assert skipped                                                # fetched_len <= k: not scored, not trained
    if name == "no_segment":
        assert score == 1.0 and counts.sum() == 0


def test_report_bytes(ref_tt):
    """the report of two strands: the reference's print() bytes per strand behind its header line"""
    specs = [tc.CASES[0], tc.CASES[1]]
    rows = []
    for spec in specs:
        c = tc.build(spec)
        rows.append(ref_tt.answers(spec[0], [tc.fingerprint(c)], lambda _: None if ref_tt.live is None else
                                   (lambda w: (w[0], w[1], w[2], w[3], np.zeros(0)))(ref_tt.live.model_score(c)))[0])
    text = tr.report([rows[0][1], rows[1][1]])
    assert text == "".join(f"Transition parameters for {s}\n" + rows[s][3] for s in range(2))


def test_host_mirror_training(ref_tt):
    """nph::TransitionTraining (nanopolish_b200/host/nph_scorereads.cpp) on the recorded counts: train() with either prior equals
    the reference's trained probabilities, and report() equals its stderr for two strands"""
    import ctypes as C
    from tests import host_mirror as hm
    lib = hm.load()
    p = hm.p
    rows = {}
    for spec in (tc.CASES[0], tc.CASES[1], tc.CASES[3]):
        c = tc.build(spec)
        rows[spec[0]] = ref_tt.answers(spec[0], [tc.fingerprint(c)], lambda _: (lambda w: (w[0], w[1], w[2], w[3], (
            ref_tt.live.prior_r9() if c["prior"] else np.zeros(0))))(ref_tt.live.model_score(c)))[0]
    for a, b in (("plain", "rc"), ("prior", "plain")):
        two = np.ascontiguousarray(np.stack([rows[a][1], rows[b][1]]), np.uint64)
        prior = rows[a][4] if rows[a][4].shape[0] else np.zeros(tr.BINS)
        probs = np.zeros(tr.BINS); buf = C.create_string_buffer(1 << 14)
        n = lib.nphh_transition_training(p(two), 0, p(prior), p(probs), buf, C.c_size_t(1 << 14))
        assert n > 0
        assert probs.tobytes() == np.asarray(rows[a][2], np.float64).tobytes()
        if a == "plain":
            assert buf.raw[:n].decode() == "Transition parameters for 0\n" + rows[a][3] + "Transition parameters for 1\n" + rows[b][3]
