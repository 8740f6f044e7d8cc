"""The compiled reference's own fix_homopolymers (src/nanopolish_call_variants.cpp:541-780, run unmodified by oracle/variants_harness.cpp)
against the restatement in tests/hp_restatement.py over the reference's profile_hmm_score / profile_hmm_align: the fixed sequence
and every variant it adds (position, REF / ALT, the bits of its quality, INFO), on pile-ups whose truth differs from the draft by
homopolymer insertions and deletions, reads of both strands, a haplotype with inserted and substituted bases in the calling
flanks that leave the range as it is, bases without a reference position exactly at the calling-range ends (the range moves),
min_flanking_sequence at its least (7), durations so short that sum_duration stays below MIN_DURATION, long runs where the duration
term makes calls the event term alone would not, and every edge of the scan, the event windows and the call rule reached on both
sides (each case asserts the edges it was built for).  The reference's answers, and the restated likelihood vectors, are kept in
tests/golden/ref_fix_homopolymers.pkl.xz for the device suite (tests/test_gpu_fix_homopolymers.py).  Also the host mirror's
Haplotype::substr_by_reference and enclosing range (nanopolish_b200/host/nph_variants.cpp) against the reference's own."""
import ctypes as C

import numpy as np
import pytest

from tests import hp_cases as hc
from tests import hp_restatement as hr
from tests.ref_calls import case_fixture
from tests.ref_variants import RefVariants
from tests.test_host_mirror import HOST_SO

ref_hp = case_fixture("ref_fix_homopolymers.pkl.xz", ref=lambda: RefVariants() if RefVariants.available() else None)


@pytest.mark.parametrize("spec", hc.CASES, ids=[s[0] for s in hc.CASES])
def test_restatement_equals_reference(ref_hp, spec):
    c = hc.build(spec)
    live = ref_hp.live

    def ask(_):
        hs, mh = live.register(c)
        want = live.fixed(c, hs)
        vectors, got = hc.ref_restated(live, c, hs, mh)
        assert got == want, f"{spec[0]}: the restatement's fixed haplotype differs from the reference's"
        # the vectors as float64 arrays: recorded and compared by their bits (NaN included)
        return want, [(n, np.array(e, np.float64), np.array(d, np.float64)) for n, e, d in vectors]

    want, vectors = ref_hp.answers(spec[0], [hc.fingerprint(c)], ask)[0]
    assert len(vectors) == len(c["wins"])
    # every case calls something; the plain pile-up calls both insertions and deletions
    calls = [l.split("\t") for l in want.split("\n")[1:] if l]
    assert calls
    if spec[0] in ("plain", "long_runs"):
        assert any(len(a) > len(r) for _, r, a, _, _ in calls) and any(len(a) < len(r) for _, r, a, _, _ in calls)
    if spec[0] == "long_runs":
        assert sum(hr.duration_decides(w, e, d) for w, (_, e, d) in zip(c["wins"], vectors)) >= 1
    _assert_edges_reached(spec[0], c, vectors)


def _assert_edges_reached(name, c, vectors):
    """each case reaches the edges it was built for (the comparison with the reference above then covers them)"""
    F = c["min_flank"]
    trace = []
    hr.fix_homopolymers(c["hap"], c["wins"], vectors, trace)
    scan = set(c["scan_trace"])
    has = lambda test, outcome, value=None, length=None: any(t[0] == test and t[1] == outcome and (value is None or t[2] == value) and
                                                            (length is None or t[3] == length) for t in scan)
    seqs, dropped = hc.event_edges(c)
    spans = {abs(e1 - e2) for s in seqs for _, e1, e2 in s}
    if name == "moved":
        # the enclosing range moved: k0, the edit offset and the calling sequence come from the moved start
        moved = [w for w in c["wins"] if w["edit_offset"] != F and len(w["calling"]) != 2 * F + w["hp_length"] + 1]
        assert len(moved) >= 3 and {w["edit_offset"] for w in moved} >= {F + 1, F + 2}
        assert any(t[0] == "tries" and t[1] >= 1 and t[2] for t in trace)      # the first base tried has no reference position
    if name == "edges_out":
        assert has("length", False, length=2) and has("length", False, length=10)
        assert has("flank_lo", False, -1) and has("flank_hi", False, 0) and has("region_lo", False, -1) and has("region_hi", False, 0)
    if name == "edges_in":
        assert has("length", True, length=3) and has("length", True, length=9)
        assert has("flank_lo", True, 0) and has("npos", True) and has("flank_hi", True, -1)
        assert has("region_lo", True, 0) and has("region_hi", True, -1)
        assert sum(dropped) >= 1                                                  # the event/bp ratio test drops a read
        calls = [t for t in trace if t[0] == "call"]
        assert any(t[1] == hr.NPOS and t[2] != t[2] for t in calls)              # call npos, quality NaN, kept
    if name.startswith("edges"):
        assert has("last_run", True)
        assert 9 in spans and 10 in spans                                        # 10 events (skipped) and 11 events (scored)
        for s, (n, _, _) in zip(seqs, vectors):
            assert n == len(s)
    if name == "short_durations":
        assert all(d == 0.0 for _, _, ds in vectors for d in ds) and any(n for n, _, _ in vectors)     # sum_duration <= MIN_DURATION


def test_call_rule_edges():
    """the mirror's call rule (nph::homopolymer_call) against the restatement's on crafted vectors: quality exactly 10 and one ulp
    below, NaN scores, nothing above -inf (call npos), +inf, and ties (the first length wins)"""
    host = C.CDLL(HOST_SO)
    below = float(np.nextafter(10.0, 0.0))
    nan, inf = float("nan"), float("inf")
    cases = [
        (4, [0.0, 0.0, 10.0, 0.0, 0.0, 0.0, 0.0], [0.0] * 7),       # quality exactly 10: kept
        (4, [0.0, 0.0, below, 0.0, 0.0, 0.0, 0.0], [0.0] * 7),      # one ulp below: not kept
        (5, [1.0] * 7, [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 11.0]),       # an insertion of 4 bases
        (9, [30.0] + [0.0] * 6, [0.0] * 7),                         # a deletion of 6 bases
        (3, [nan] * 7, [0.0] * 7),                                  # every score NaN: call npos, quality NaN, kept
        (6, [-inf] * 7, [0.0] * 7),                                 # nothing beats -inf: call npos, quality NaN
        (3, [0.0] * 7, [0.0, inf, 0.0, 0.0, 0.0, 0.0, 0.0]),        # +inf
        (7, [5.0, 20.0, 20.0, 0.0, 0.0, 0.0, 0.0], [0.0] * 7),      # a tie: the first length wins
        (4, [0.0] * 7, [0.0] * 7),                                  # all equal: quality 0
    ]
    for hp, e, d in cases:
        call, q, sd = C.c_uint64(), C.c_double(), C.c_int()
        ea, da = np.array(e, np.float64), np.array(d, np.float64)
        kept = host.nphh_homopolymer_call(ea.ctypes.data_as(C.c_void_p), da.ctypes.data_as(C.c_void_p), C.c_uint32(hp), C.byref(call),
                                          C.byref(q), C.byref(sd))
        w_call, w_q, w_sd, w_kept = hr.call_rule(hp, e, d)
        assert (call.value, sd.value, bool(kept)) == (w_call, w_sd, w_kept), (hp, e, d)
        assert np.float64(q.value).tobytes() == np.float64(w_q).tobytes() or (q.value != q.value and w_q != w_q)
    assert hr.call_rule(4, cases[0][1], cases[0][2])[3] and not hr.call_rule(4, cases[1][1], cases[1][2])[3]
    assert hr.call_rule(3, cases[4][1], cases[4][2])[:1] == (hr.NPOS,) and hr.call_rule(3, cases[4][1], cases[4][2])[2] == -4

def _range_cases():
    """haplotypes with insertions, deletions and substitutions, and substr_by_reference / enclosing-range queries the reference
    answers without an assert (the restatement decides which)"""
    rng = np.random.default_rng(12)
    out = []
    for h in range(6):
        ref = "".join("ACGT"[x] for x in rng.integers(0, 4, 80))
        hap = hr.Haplotype(hc.REGION_START, ref)
        variants = []
        for off in sorted(rng.choice(np.arange(2, 76), 10, replace=False)):
            kind = int(rng.integers(3))
            r = ref[off:off + (2 if kind == 1 else 1)]
            a = r + "ACGT"[int(rng.integers(4))] if kind == 0 else (r[0] if kind == 1 else "ACGT"[("ACGT".index(r) + 1) % 4])
            if hap.apply_variant(hc.REGION_START + int(off), r, a):
                variants.append((int(off), r, a))
        for _ in range(40):
            s = hc.REGION_START + int(rng.integers(0, 81)); e = s + int(rng.integers(0, 12))
            lo = int(rng.integers(0, len(hap.seq))); hi = min(len(hap.seq) + 1, lo + int(rng.integers(0, 12)))
            try:
                sub = hap.substr_by_reference(s, e)
            except hr.RefAbort:
                continue
            enc = hap.enclosing(lo, hi)
            want = (sub.ref_position, sub.seq, tuple(enc) if enc else (-1, -1, -1, -1))
            out.append((ref, variants, s, e, lo, hi, want))
    return out


def test_mirror_haplotype_ranges_equal_reference(ref_hp):
    host = C.CDLL(HOST_SO)
    cases = _range_cases()
    assert len(cases) > 150
    fps = [repr(x[:6]) for x in cases]
    want = ref_hp.answers("haplotype_ranges", fps, lambda i: hc.ranges(ref_hp.live.lib, "npref_haplotype_ranges", *cases[i][:6]))
    for (ref, variants, s, e, lo, hi, restated), w in zip(cases, want):
        assert w == restated
        assert hc.ranges(host, "nphh_haplotype_ranges", ref, variants, s, e, lo, hi) == w
