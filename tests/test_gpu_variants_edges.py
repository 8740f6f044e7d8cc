"""Device candidate screening (csrc/variants.cu, nph_screen_edits_batch) where tests/test_gpu_variants.py does not reach:
  * a region of 2,199 positions: nine var_bounds blocks of 256 positions and three scan blocks of 1,024, records that run past
    both ends of the region, and the same records in shuffled order;
  * gapped event alignments: deleted reference bases (NO_PAIR entries inside a record), insertions (event-index jumps), windows
    that start or end inside a gap or lie wholly inside one, and the 20 events-per-base cut at 419 / 420 events over 21 bases;
  * more than 256 records on one block (several passes of the ordered append), and more than 2,048 (the block's shared-memory
    list overflows and the kernel walks every record);
  * flank 30 (63-base insertion windows), flank 3, flank 2 with a 5-mer model (one-k-mer deletion windows), the refused settings;
  * thresholds 0 and 1, and rounds larger than every position's depth.
Every quality (NaN where the reference generates no candidate), every position's event-sequence count and reference DP rows, and
the number of rounds equal tests/var_restatement.py scored by the port oracle.  The tests without the gpu mark check that the
builders really produce these edges."""
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from tests import var_restatement as vr
from tests.eventalign_cases import five_mer_model
from tests.meth_restatement import find_by_ref_bounds

K = 6
R0 = 5000
VAR_BLOCK, LIST_CAP, SCAN_BLOCK = 256, 2048, 1024          # kBlock, kListCap, kScanBlock of csrc/variants.cu
NPH_ERR_INVALID, NPH_ERR_STATE, NPH_ERR_UNSUPPORTED = -3, -5, -6
THREADS = os.cpu_count() or 1


class Pile:
    """One screening input: reads, the region's reference bases, event-alignment records in the order the caller passes them."""

    def __init__(self, rs, model, ref_codes, region_start, recs, pairs, flags=0, indel_bias=1.0, model_id=0):
        self.rs, self.model, self.region_start, self.flags, self.indel_bias = rs, model, region_start, flags, indel_bias
        self.ref_chars = synth._CODE2DNA[ref_codes]
        self.ref = self.ref_chars.tobytes().decode()
        self.recs, self.pairs = recs.copy(), pairs
        self.recs["model_id"] = model_id
        n_total = int((recs["ref_off"].astype(np.int64) + recs["ref_len"]).max())
        self.deltas, self.first = synth.compact_event_alignment(self.recs, pairs, n_total)

    @property
    def n_pos(self):
        return len(self.ref) - 1

    def reordered(self, order):
        return Pile(self.rs, self.model, synth.encode(self.ref, "nucleotide"), self.region_start, self.recs[order], self.pairs, self.flags,
                    self.indel_bias, int(self.recs["model_id"][0]))


def _repack(recs, pair_lists):
    """records with new pair lists (same order), and the concatenated PAIR_DT array"""
    recs = recs.copy()
    off = 0
    for r, pr in enumerate(pair_lists):
        recs[r]["pair_off"], recs[r]["n_pairs"] = off, pr.shape[0]
        off += pr.shape[0]
    return recs, np.concatenate(pair_lists) if pair_lists else np.zeros(0, synth.PAIR_DT)


def _scores(port_oracle, pile, flank=10, k=K):
    return vr.position_scores(port_oracle, pile.rs, pile.model, pile.ref, pile.region_start,
                              range(pile.region_start, pile.region_start + pile.n_pos), pile.recs, pile.pairs, flank, pile.flags,
                              pile.indel_bias, k, threads=THREADS)


# ---- pile-up builders ------------------------------------------------------------------------------------------------------

def multi_block_pile():
    """2,200 reference bases (2,199 positions) cut from the middle of a 2,500-base pile-up, ~20x of 400-base reads: records start
    before the region and end after it."""
    nuc = synth.load_model("nucleotide")
    ref, rs, recs, pairs = synth.gen_pileup(2500, 20, 400, nuc, seed=31, region_start=R0, n_true_variants=6)
    lo = 150
    return Pile(rs, nuc, ref[lo:lo + 2200], R0 + lo, recs, pairs, flags=3, indel_bias=0.9)


def _ratio_edit(pr, ref_start, n_events, span):
    """Shift the events of a forward record so that the first window [cs, cs + 21] that has entries at both ends spans exactly
    `span` events (an insertion at cs + 21); events past the read's end are dropped.  -> (pairs, window centre i)"""
    rp, ev = pr["ref_pos"], pr["read_pos"]
    at = {int(p): j for j, p in enumerate(rp)}
    cs = next(int(p) for p in rp if p >= ref_start + 8 and int(p) + 21 in at)
    ce = cs + 21
    assert ev[at[cs]] + span < n_events
    pr = pr.copy()
    pr["read_pos"][at[ce]:] += span - (ev[at[ce]] - ev[at[cs]])
    return pr[pr["read_pos"] < n_events], cs + 10


def gapped_pile():
    """A 600-base pile-up of 300-base reads whose event alignments are edited before compaction.  -> (pile, edits):
    ("del", record, first ref position, length): deleted reference bases, NO_PAIR entries inside the record;
    ("ins", record, ref position, J): an insertion, every later event index J further along the read's strand;
    ("long", record, first ref position, 30): a gap longer than a window;
    ("ratio", record, position i, span): the window of position i spans `span` events (419: kept, 420: dropped)."""
    nuc = synth.load_model("nucleotide")
    ref, rs, recs, pairs = synth.gen_pileup(600, 16, 300, nuc, seed=47, region_start=R0, n_true_variants=3)
    rng = np.random.default_rng(2024)
    n_ev = rs.reads["n_events"].astype(np.int64)
    fwd = [r for r in range(recs.shape[0]) if recs[r]["rc"] == 0]
    rev = [r for r in range(recs.shape[0]) if recs[r]["rc"] == 1]
    ratio = {fwd[1]: 419, fwd[4]: 420}
    long_gap = {fwd[2], rev[2]}
    edits, lists = [], []
    for r, R in enumerate(recs):
        pr = pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])].copy()
        if r in ratio:
            pr, i = _ratio_edit(pr, int(R["ref_start_pos"]), n_ev[r], ratio[r])
            edits.append(("ratio", r, i, ratio[r]))
            lists.append(pr)
            continue
        n = pr.shape[0]
        keep = np.ones(n, bool)
        if r % 3 != 2:
            for _ in range(2):
                L = 1 + sum(e[0] == "del" for e in edits) % 15           # every length 1..15 in turn
                at = int(rng.integers(25, n - 40))
                keep[at:at + L] = False
                edits.append(("del", r, int(pr["ref_pos"][at]), L))
        if r % 3 != 0:
            at, J = int(rng.integers(25, n - 40)), int(rng.integers(12, 41))
            pr["read_pos"][at:] += -J if R["rc"] else J
            edits.append(("ins", r, int(pr["ref_pos"][at]), J))
        if r % 4 == 3:
            keep[:int(rng.integers(1, 16))] = False
            keep[n - int(rng.integers(1, 16)):] = False
        if r in long_gap:
            keep[n // 2:n // 2 + 30] = False
            edits.append(("long", r, int(pr["ref_pos"][n // 2]), 30))
        keep &= (pr["read_pos"] >= 0) & (pr["read_pos"] < n_ev[r])
        lists.append(pr[keep])
    recs, pairs = _repack(recs, lists)
    return Pile(rs, nuc, ref, R0, recs, pairs), edits


def crowded_piles(n_fill=2200, seed=53):
    """~350 records of 60 bases over 300 reference bases (all on the first var_bounds block), and the same with n_fill filler records
    spread among them: ref_len 40 on the first block, no aligned event, so they bound no window.  -> (plain, filled)"""
    nuc = synth.load_model("nucleotide")
    ref, rs, recs, pairs = synth.gen_pileup(300, 70, 60, nuc, seed=seed, region_start=R0, n_true_variants=2)
    plain = Pile(rs, nuc, ref, R0, recs, pairs)
    rng = np.random.default_rng(seed)
    fill = np.zeros(n_fill, synth.METH_RECORD_DT)
    fill["read"] = rng.integers(0, recs.shape[0], n_fill)
    fill["rc"] = recs["rc"][fill["read"]]
    fill["ref_len"] = 40
    fill["ref_off"] = int((recs["ref_off"].astype(np.int64) + recs["ref_len"]).max()) + 40 * np.arange(n_fill)
    fill["pair_off"] = pairs.shape[0]
    fill["ref_start_pos"] = R0 + rng.integers(-30, 220, n_fill)
    # the real records keep their order; the fillers take random places among them
    is_fill = np.zeros(recs.shape[0] + n_fill, bool)
    is_fill[rng.choice(is_fill.shape[0], n_fill, replace=False)] = True
    both = np.zeros(is_fill.shape[0], synth.METH_RECORD_DT)
    both[~is_fill], both[is_fill] = recs, fill
    return plain, Pile(rs, nuc, ref, R0, both, pairs)


EDGE_SETTINGS = [(30, 6), (3, 6), (2, 5)]          # (flank, k)


def edge_pile(flank, k):
    """a small pile-up for a window of 2 flank + 2 bases; reads long enough to hold ~90 windows of flank 30"""
    model = synth.load_model("nucleotide") if k == 6 else five_mer_model()
    assert model.k == k
    n_ref, read_bases = (220, 170) if flank == 30 else (150, 110)
    ref, rs, recs, pairs = synth.gen_pileup(n_ref, 14, read_bases, model, seed=61 + flank, region_start=R0, n_true_variants=2)
    return Pile(rs, model, ref, R0, recs, pairs, flags=3 if flank == 3 else 0, indel_bias=0.9, model_id=0 if k == 6 else 1)


def block_overlaps(pile, block, flank=10):
    """records whose extent meets the windows of var_bounds block `block` (the kernel's lo / hi)"""
    p0 = block * VAR_BLOCK
    lo = pile.region_start + p0 - flank
    hi = pile.region_start + min(p0 + VAR_BLOCK - 1, pile.n_pos - 1) + 1 + flank
    st = pile.recs["ref_start_pos"].astype(np.int64)
    return (pile.recs["ref_len"] > 0) & (st <= hi) & (st + pile.recs["ref_len"] - 1 >= lo)


# ---- expectations and the device run -------------------------------------------------------------------------------------------

def expected(scores, threshold, rpr):
    """-> (qualities f8[n_pos, 9], event sequences per position, reference DP rows per position, rounds): a position takes reads_per_round
    event sequences a round until its last candidate has left the threshold or its sequences run out"""
    n = len(scores)
    q = np.full((n, 9), np.nan)
    nr, rows = np.zeros(n, np.int64), np.zeros(n, np.int64)
    rounds = 0
    for pi, got in enumerate(scores):
        if got is None:
            continue
        cands, seqs, sc = got
        qq, rows[pi], used = vr.accumulate(cands, seqs, sc, threshold)
        q[pi], nr[pi] = qq, len(seqs)
        if seqs:
            rounds = max(rounds, max(1, -(-used // rpr)))
    return q, nr, rows, rounds


def screen(eng, pile, threshold, rpr, flank=10, k=K):
    params = synth.screen_params(pile.region_start, k, flank, threshold, pile.flags, rpr)
    eng.reads_load(pile.rs.reads, pile.rs.ev_mean, pile.rs.ev_start_time)
    eng.screen_load(pile.ref_chars, pile.deltas, pile.first, pile.recs, params, indel_bias=pile.indel_bias)
    eng.screen_run()
    q, nr, rows = eng.screen_fetch(with_reference_rows=True)
    return q, nr, rows, eng.screen_counts()


def assert_screen(got, want):
    q, nr, rows, cnt = got
    wq, wnr, wrows, wrounds = want
    assert q.shape == wq.shape
    nan = np.isnan(wq)
    bad = np.argwhere(np.isnan(q) != nan)
    assert bad.size == 0, f"NaN slots differ at (position, slot) {bad[:8].tolist()}"
    bad = np.argwhere(~nan & (q.view(np.uint64) != wq.view(np.uint64)))
    assert bad.size == 0, f"{bad.shape[0]} qualities differ, first {[(p, s, q[p, s], wq[p, s]) for p, s in bad[:4].tolist()]}"
    bad = np.flatnonzero(nr.astype(np.int64) != wnr)
    assert bad.size == 0, f"event sequences differ at positions {bad[:8].tolist()}: {nr[bad[:8]].tolist()} vs {wnr[bad[:8]].tolist()}"
    bad = np.flatnonzero(rows.astype(np.int64) != wrows)
    assert bad.size == 0, f"reference rows differ at positions {bad[:8].tolist()}: {rows[bad[:8]].tolist()} vs {wrows[bad[:8]].tolist()}"
    assert cnt["rounds"] == wrounds
    assert cnt["reference_events"] == int(wrows.sum())


def exited(want, threshold):
    q = want[0]
    return int((~np.isnan(q) & (np.abs(np.nan_to_num(q)) >= threshold)).sum())


# ---- fixtures --------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    assert e.model_upload(synth.load_model("nucleotide")) == 0
    assert e.model_upload(five_mer_model()) == 1
    yield e
    e.close()


@pytest.fixture(scope="module")
def multi_block(port_oracle):
    pile = multi_block_pile()
    return pile, _scores(port_oracle, pile)


@pytest.fixture(scope="module")
def gapped(port_oracle):
    pile, _ = gapped_pile()
    return pile, _scores(port_oracle, pile)


@pytest.fixture(scope="module")
def edges(port_oracle):
    out = {}
    for flank, k in EDGE_SETTINGS:
        pile = edge_pile(flank, k)
        out[flank, k] = pile, _scores(port_oracle, pile, flank, k)
    return out


# ---- device tests ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("shuffled", [False, True])
def test_multi_block_region(eng, multi_block, shuffled):
    pile, scores = multi_block
    if shuffled:
        # the device walks the records in the caller's order: the expectations follow the shuffled array
        order = np.random.default_rng(9).permutation(pile.recs.shape[0])
        new_of_old = np.argsort(order)
        pile = pile.reordered(order)
        lists = vr.pair_lists(pile.recs, pile.pairs)
        moved = []
        for pi, got in enumerate(scores):
            if got is None:
                moved.append(None)
                continue
            cands, seqs, sc = got
            j = sorted(range(len(seqs)), key=lambda t: new_of_old[seqs[t][0]])
            seqs = [(int(new_of_old[seqs[t][0]]), seqs[t][1], seqs[t][2]) for t in j]
            i = pile.region_start + pi
            assert seqs == vr.event_sequences(pile.recs, pile.pairs, i - 10, i + 11, lists), pi
            moved.append((cands, seqs, sc[j]))
        scores = moved
    assert pile.n_pos == 2199
    for threshold, rpr in ((100, 8), (30, 1)):
        want = expected(scores, threshold, rpr)
        assert exited(want, threshold) > 2000 and want[3] >= 3
        assert_screen(screen(eng, pile, threshold, rpr), want)


@pytest.mark.gpu
@pytest.mark.parametrize("threshold,rpr", [(100, 4), (30, 2)])
def test_gapped_alignments(eng, gapped, threshold, rpr):
    pile, scores = gapped
    want = expected(scores, threshold, rpr)
    assert exited(want, threshold) > 500
    assert_screen(screen(eng, pile, threshold, rpr), want)


@pytest.mark.gpu
def test_crowded_block(eng, port_oracle):
    plain, filled = crowded_piles()
    want = expected(_scores(port_oracle, plain), 60, 4)
    assert exited(want, 60) > 500
    got_plain = screen(eng, plain, 60, 4)
    assert_screen(got_plain, want)
    got_filled = screen(eng, filled, 60, 4)
    assert_screen(got_filled, want)
    assert np.array_equal(got_plain[0].view(np.uint64), got_filled[0].view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("flank,k", EDGE_SETTINGS)
def test_window_edges(eng, edges, flank, k):
    pile, scores = edges[flank, k]
    want = expected(scores, 50, 3)
    assert exited(want, 50) > 100 and want[1].sum() > 0
    assert_screen(screen(eng, pile, 50, 3, flank, k), want)


@pytest.mark.gpu
def test_refused_settings_leave_the_context_usable(eng, edges):
    pile, scores = edges[3, 6]
    want = expected(scores, 50, 3)
    rs = pile.rs
    for flank, k, rpr, status in ((31, 6, 3, NPH_ERR_UNSUPPORTED), (2, 6, 3, NPH_ERR_INVALID), (3, 6, 0, NPH_ERR_INVALID)):
        params = synth.screen_params(pile.region_start, k, flank, 50, pile.flags, rpr)
        with pytest.raises(NphError) as e:
            eng.screen_edits_batch(rs.reads, rs.ev_mean, rs.ev_start_time, pile.ref_chars, pile.deltas, pile.first, pile.recs, params,
                                   indel_bias=pile.indel_bias)
        assert e.value.status == status, (flank, k, rpr)
        with pytest.raises(NphError) as e:
            eng.screen_run()
        assert e.value.status == NPH_ERR_STATE
        assert_screen(screen(eng, pile, 50, 3, 3, 6), want)


@pytest.mark.gpu
def test_threshold_edges(eng, gapped):
    pile, scores = gapped
    # threshold 0: no candidate is ever inside it; every position with event sequences takes one round and scores nothing
    want = expected(scores, 0, 4)
    q = want[0]
    assert want[3] == 1 and (want[2] == 0).all() and (q[~np.isnan(q)] == 0.0).all() and want[1].sum() > 0
    assert_screen(screen(eng, pile, 0, 4), want)
    # threshold 1: nearly every candidate leaves after its first event sequence
    first_step = []
    for got in scores:
        if got is not None and got[1]:
            sc = got[2]
            first_step += [abs(float(sc[0, c]) - float(sc[0, 0])) >= 1 for c in range(1, sc.shape[1])]
    assert len(first_step) > 3000 and sum(first_step) > 0.9 * len(first_step)
    assert_screen(screen(eng, pile, 1, 2), expected(scores, 1, 2))
    # reads_per_round above every position's depth: one round
    depth = max(len(got[1]) for got in scores if got)
    want = expected(scores, 100, depth + 1)
    assert want[3] == 1
    assert_screen(screen(eng, pile, 100, depth + 1), want)


# ---- the builders' edges (no GPU) ------------------------------------------------------------------------------------------------

def _compact_bounds(pile, r, cs, ce):
    """the window's (e1, e2) read off the compact form (event deltas per reference base, first event), the way var_bounds_kernel
    reads it, or None"""
    R = pile.recs[r]
    n, st = int(R["ref_len"]), int(R["ref_start_pos"])
    d = pile.deltas[int(R["ref_off"]):int(R["ref_off"]) + n].astype(np.int64)
    valid = np.flatnonzero(d != synth.METH_NO_PAIR)
    if valid.size == 0:
        return None
    ev = int(pile.first[r]) + np.cumsum(d[valid])
    os_, oe = cs - st, ce - st
    a, b = np.searchsorted(valid, max(os_, 0)), np.searchsorted(valid, max(oe, 0))
    if a == valid.size or b == valid.size or not (valid[a] <= os_ or a > 0):
        return None
    return int(ev[a]), int(ev[b])


def _gaps(pile, r):
    """interior runs of NO_PAIR in record r's compact deltas: [(first ref position, length)]"""
    R = pile.recs[r]
    d = pile.deltas[int(R["ref_off"]):int(R["ref_off"]) + int(R["ref_len"])]
    valid = np.flatnonzero(d != synth.METH_NO_PAIR)
    return [(int(R["ref_start_pos"]) + int(a) + 1, int(b - a - 1)) for a, b in zip(valid[:-1], valid[1:]) if b - a > 1]


def test_gapped_builder_reaches_its_edges():
    pile, edits = gapped_pile()
    recs = pile.recs
    # deleted reference bases are NO_PAIR runs inside their record, on both strands, lengths 1..15
    gaps = {r: _gaps(pile, r) for r in range(recs.shape[0])}
    dels = [e for e in edits if e[0] == "del"]
    for _, r, p, L in dels:
        assert any(g <= p and p + L <= g + n for g, n in gaps[r]), (r, p, L)
    assert {int(recs[r]["rc"]) for _, r, _, _ in dels} == {0, 1}
    assert {L for *_, L in dels} >= {1, 15} and len({L for *_, L in dels}) >= 10
    # insertions are event-index steps of at least J, forward steps up and reverse steps down
    ins = [e for e in edits if e[0] == "ins"]
    assert {int(recs[r]["rc"]) for _, r, _, _ in ins} == {0, 1}
    for _, r, p, J in ins:
        R = recs[r]
        d = pile.deltas[int(R["ref_off"]) + p - int(R["ref_start_pos"]):int(R["ref_off"]) + int(R["ref_len"])]
        step = int(d[d != synth.METH_NO_PAIR][0])
        assert (step <= -J) if R["rc"] else (step >= J), (r, p, J, step)
    # every window: the compact form bounds what the pair form bounds
    lists = vr.pair_lists(recs, pile.pairs)
    in_gap_start = in_gap_end = whole = 0
    for i in range(R0 + 10, R0 + pile.n_pos - 11):
        cs, ce = i - 10, i + 11
        seqs = vr.event_sequences(recs, pile.pairs, cs, ce, lists)
        compact = []
        for r in range(recs.shape[0]):
            b = _compact_bounds(pile, r, cs, ce)
            if b is not None and abs(b[0] - b[1]) / 21 < 20:
                compact.append((r, b[0], b[1]))
        assert compact == seqs, i
        for r, e1, e2 in seqs:
            in_gap_start += any(g <= cs < g + n for g, n in gaps[r])
            in_gap_end += any(g <= ce < g + n for g, n in gaps[r])
            whole += e1 == e2
    assert in_gap_start > 50 and in_gap_end > 50 and whole >= 2
    # a record with no entry inside some window it spans
    for _, r, p, n in (e for e in edits if e[0] == "long"):
        assert any(g <= p and p + n <= g + m for g, m in gaps[r]), (r, p)
        assert find_by_ref_bounds(*lists[r], p + 2, p + 23) is not None
    # the 20 events-per-base cut: 419 events over 21 bases are kept, 420 are not
    ratio = {span: (r, i) for kind, r, i, span in edits if kind == "ratio"}
    assert set(ratio) == {419, 420}
    for span, (r, i) in ratio.items():
        assert recs[r]["rc"] == 0 and R0 + 10 <= i < R0 + pile.n_pos - 11
        e1, e2 = find_by_ref_bounds(*lists[r], i - 10, i + 11)
        assert e2 - e1 == span
        assert any(s[0] == r for s in vr.event_sequences(recs, pile.pairs, i - 10, i + 11, lists)) == (span == 419)


def test_multi_block_builder_reaches_its_edges():
    pile = multi_block_pile()
    assert pile.n_pos == 2199
    assert -(-pile.n_pos // VAR_BLOCK) == 9
    assert -(-pile.n_pos // SCAN_BLOCK) == 3 and pile.n_pos % SCAN_BLOCK != 0
    st = pile.recs["ref_start_pos"].astype(np.int64)
    end = st + pile.recs["ref_len"] - 1
    lists = vr.pair_lists(pile.recs, pile.pairs)
    region_end = pile.region_start + pile.n_pos
    # records that start before the region and bound windows inside it, and records that end after it
    left = [r for r in np.flatnonzero(st < pile.region_start) if lists[r][0] and lists[r][0][-1] > pile.region_start + 30]
    right = [r for r in np.flatnonzero(end > region_end) if lists[r][0] and lists[r][0][0] < region_end - 30]
    assert len(left) >= 2 and len(right) >= 2
    assert (pile.recs["rc"] == 1).sum() == pile.recs.shape[0] // 2


def test_crowded_builder_reaches_its_edges():
    plain, filled = crowded_piles()
    assert block_overlaps(plain, 0).sum() > VAR_BLOCK
    assert block_overlaps(filled, 0).sum() > LIST_CAP
    # the fillers have no aligned event, and the real records keep their order with fillers on both sides of them
    fill = filled.recs["ref_len"] == 40
    assert (filled.recs["n_pairs"][fill] == 0).all() and (filled.recs["ref_len"] > 0).all()
    assert np.array_equal(filled.recs[~fill], plain.recs)
    assert np.flatnonzero(fill).min() < np.flatnonzero(~fill).max() and np.flatnonzero(~fill).min() < np.flatnonzero(fill).max()


def test_edge_piles_reach_their_windows():
    for flank, k in EDGE_SETTINGS:
        pile = edge_pile(flank, k)
        lists = vr.pair_lists(pile.recs, pile.pairs)
        i = pile.region_start + pile.n_pos // 2
        assert pile.model.k == pile.rs.k == k
        assert len(vr.event_sequences(pile.recs, pile.pairs, i - flank, i + 1 + flank, lists)) >= 3
