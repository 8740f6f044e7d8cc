"""call-methylation's device front end (csrc/methylation.cu) on every edge case of tests/meth_edge_cases.py, and its grid-stride
loops on batches larger than one pass of the grid.

Every call runs three ways, which must return bit-identical site records: the pair form, the compact form (int16 deltas
rebuilt by meth_expand_kernel) and the staged load / run / fetch.  Cases with the reference's parameters are compared with the
compiled reference's recorded answers (tests/golden/ref_meth_edges.pkl.xz): groups, scores as doubles and the TSV rows the
device writes.  The others are compared with the restatement scored by the port oracle: scores bit for bit and the scored-event
count."""
import numpy as np
import pytest
import torch

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from tests import meth_edge_cases as ec
from tests import meth_restatement as mr
from tests import ref_calls

pytestmark = pytest.mark.gpu
NPH_ERR_INVALID, NPH_ERR_UNSUPPORTED = -3, -6
SUB_BATCH = 3000


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    for m in ec.models():
        e.model_upload(m)
    yield e
    e.close()


def _params(case):
    kw = case.kw
    return synth.meth_params(case.alphabet, ec.K, **kw)


def _three_forms(eng, rs, ref, pairs, recs, params, compact=True):
    """(site_off, sites, scored events) of the pair form, after checking the compact and staged forms give the same (compact
    False: records cut short of their pair lists, which the compact form cannot carry)"""
    off, sites, scored = eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, pairs, recs, params)
    if compact:
        deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
        c = eng.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs, params)
        assert np.array_equal(off, c[0]) and sites.tobytes() == c[1].tobytes() and scored == c[2], "compact form differs"
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.methylation_load(ref, pairs, recs, params)
    eng.methylation_run()
    s_off, s_sites = eng.methylation_fetch()
    n = sites.shape[0]
    assert np.array_equal(off, s_off) and s_sites[:n].tobytes() == sites.tobytes(), "staged form differs"
    assert eng.methylation_counts()[2] == scored
    return off, sites, scored


def _tsv(eng, built):
    return eng.methylation_tsv("chr1", [b.inputs["name"] for b in built], np.array([b.rc for b in built], np.uint8)).decode()


def test_edge_cases(eng, port_oracle):
    rs, built = ec.build(ec.all_cases())
    mods = ec.models()
    rec = ref_calls.case_answers("ref_meth_edges.pkl.xz", "meth_edges")
    calls = {}
    for b in built:
        calls.setdefault(b.case.group, []).append(b)
    n_ref = n_own = 0
    for group in calls.values():
        ref, pairs, recs = ec.records(group)
        off, sites, scored = _three_forms(eng, rs, ref, pairs, recs, _params(group[0].case), compact=group[0].case.cut is None)
        want_tsv, want_events = [], 0
        for j, b in enumerate(group):
            s = sites[int(off[j]):int(off[j + 1])]
            assert (s["record"] == j).all()
            g = ec.restated(b)
            want_events += sum(2 * (abs(x[4] - x[3]) + 1) for x in g)
            if b.case.reference_case:
                tsv, ws, wl = rec[ec.fingerprint(rs, b)]
                assert s.shape[0] == ws.shape[0], f"{b.case.name}: {s.shape[0]} groups, the reference {ws.shape[0]}"
                got = np.stack([s["start_position"], s["end_position"], s["n_motif"].astype(np.int32)], 1) if s.shape[0] else np.zeros((0, 3))
                assert np.array_equal(got, ws[:, :3]), f"{b.case.name}: groups differ from the reference's"
                assert np.array_equal(s["ll_unmethylated"].astype(np.float64), wl[:, 0]), f"{b.case.name}: ll_unmethylated"
                assert np.array_equal(s["ll_methylated"].astype(np.float64), wl[:, 1]), f"{b.case.name}: ll_methylated"
                want_tsv.append(tsv)
                n_ref += 1
            else:
                ll = ec.score(port_oracle, rs, mods, b, g)
                assert [(int(x["start_position"]), int(x["end_position"]), int(x["n_motif"])) for x in s] == [x[:3] for x in g], b.case.name
                assert np.array_equal(s["ll_unmethylated"].view(np.uint32), ll[:, 0].view(np.uint32)), f"{b.case.name}: ll_unmethylated"
                assert np.array_equal(s["ll_methylated"].view(np.uint32), ll[:, 1].view(np.uint32)), f"{b.case.name}: ll_methylated"
                want_tsv.append(ec.tsv(b, g, ll))
                n_own += 1
        assert scored == want_events, f"{group[0].case.group}: scored events"
        assert _tsv(eng, group) == "".join(want_tsv)
    assert n_ref >= 45 and n_own >= 10


def test_window_shorter_than_k_is_refused(eng):
    """a window cut to k - 1 bases refuses the whole call, one-shot or staged, and names its record; cut to k it is called
    (test_edge_cases)"""
    ok, bad = ec.refusal_cases()
    rs, built = ec.build([ok, bad])
    ref, pairs, recs = ec.records(built)
    j = 1                                  # the refused record follows one that is called
    with pytest.raises(NphError) as ex:
        eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, pairs, recs, _params(bad))
    assert ex.value.status == NPH_ERR_INVALID and f"methylation record {j}:" in str(ex.value)
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.methylation_load(ref, pairs, recs, _params(bad))
    with pytest.raises(NphError) as ex:
        eng.methylation_run()
    assert ex.value.status == NPH_ERR_INVALID and f"methylation record {j}:" in str(ex.value)


def test_window_limit(eng):
    """max_span + 2 * min_flank + 1 == NPH_METH_MAX_WINDOW + 1 is unsupported (one less is test_edge_cases' 1 024-base window)"""
    rs, built = ec.build([c for c in ec.all_cases() if c.name == "window=1024"])
    ref, pairs, recs = ec.records(built)
    p = synth.meth_params("cpg", ec.K, max_span=ec.MAX_WINDOW - 20)
    with pytest.raises(NphError) as ex:
        eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, pairs, recs, p)
    assert ex.value.status == NPH_ERR_UNSUPPORTED


# ---------------------------------------------------------------- grid-stride loops
def _stride_batch(n_records, seed=5):
    """n_records short all-M records (200 to 400 bases) drawn from 40 templates: cpg sites 11 apart, templates without sites,
    every 7th record without an event alignment (all NPH_METH_NO_PAIR in the compact form), every 3rd on the reverse strand"""
    nuc = synth.load_model("nucleotide")
    rng = np.random.default_rng(seed)
    n_t = 40
    per = -(-n_records // n_t)
    sets = []
    for t in range(n_t):
        n = int(rng.integers(200, 401)) if t % 2 else int(rng.integers(300, 401))
        sites = [] if t % 10 == 3 else list(range(21 + t % 5, n - 14, 11))
        s = ec.plant(n, sites, seed=100 + t)
        sets.append(synth.gen_reads_from_sequence(synth.encode(s, "nucleotide"), per, nuc, seed=seed * 1000 + t * per))
    rs = ec.concat(sets)
    order = rng.permutation(rs.n_reads)[:n_records]
    rs = synth.ReadSet(rs.reads[order].copy(), rs.ev_mean, rs.ev_start_time, [rs.seq_codes[i] for i in order], [rs.ev_kmer[i] for i in order],
                       [rs.kmer_first_event[i] for i in order], ec.K)
    ref, pairs, recs = synth.methylation_records(rs, model_id=ec.MODEL_ID["cpg"], rc_every=3)
    recs = recs.copy()
    recs["n_pairs"][::7] = 0
    return rs, ref, pairs, recs


def _sub_batches(eng, rs, ref, pairs, recs, params, compact):
    sites, tsv = [], []
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0]) if compact else (None, None)
    for a in range(0, recs.shape[0], SUB_BATCH):
        r = recs[a:a + SUB_BATCH]
        if compact:
            off, s, _ = eng.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first[a:a + SUB_BATCH], r, params)
        else:
            off, s, _ = eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, pairs, r, params)
        s = s.copy(); s["record"] += a
        sites.append(s)
        tsv.append(eng.methylation_tsv("chr20", [f"r{i}" for i in range(a, a + r.shape[0])], (np.arange(a, a + r.shape[0]) % 2).astype(np.uint8)))
    return np.concatenate(sites), b"".join(tsv)


@pytest.fixture(scope="module")
def stride_batch():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    W = sm * ec.GRID_PER_SM * ec.WARPS
    return sm, W, _stride_batch(2 * W + 1)


@pytest.mark.parametrize("which", ["W+1", "2W+1"])
def test_grid_stride_loops(eng, port_oracle, stride_batch, which):
    """W = multi_processor_count * 64 warps is one pass of the grid of every kernel: W + 1 and 2W + 1 records make warps take a
    second and a third record (the per-warp shared window of meth_emit_kernel, the per-record state of the scan), and more than
    sm_count * 2 048 sites make meth_fill_kernel's threads take a second site.  The big call must equal sub-batches of at most
    3 000 records, and a sample of records the restatement scored by the port oracle."""
    sm, W, (rs, ref, pairs, recs) = stride_batch
    n = W + 1 if which == "W+1" else 2 * W + 1
    recs = recs[:n]
    params = synth.meth_params("cpg", ec.K)
    off, sites, scored = _three_forms(eng, rs, ref, pairs, recs, params)
    names = [f"r{i}" for i in range(n)]
    tsv = eng.methylation_tsv("chr20", names, (np.arange(n) % 2).astype(np.uint8))
    if which == "2W+1":
        assert sites.shape[0] > sm * ec.GRID_PER_SM * 256
    assert (np.diff(off)[::7] == 0).all() and (np.diff(off) == 0).sum() > n // 7
    for compact in (False, True):
        s2, t2 = _sub_batches(eng, rs, ref, pairs, recs, params, compact)
        assert s2.tobytes() == sites.tobytes(), f"sub-batches (compact={compact}) differ"
        assert t2 == tsv
    # a seeded sample against the restatement and the port oracle (records past the first pass of the grid included)
    pick = np.sort(np.random.default_rng(n).choice(n, 200, replace=False))
    pick[-1] = n - 1
    sub = recs[pick]
    rows, jobs, ranks = mr.enumerate_batch(ref, pairs, sub, "cpg", ec.K)
    scores, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ec.models(), ranks, jobs)
    got = np.concatenate([sites[int(off[i]):int(off[i + 1])] for i in pick])
    assert got.shape[0] == len(rows) > 1000
    assert [(int(x["start_position"]), int(x["end_position"]), int(x["n_motif"]), int(x["record"])) for x in got] == \
        [(r[1], r[2], r[3], int(pick[r[0]])) for r in rows]
    assert np.array_equal(got["ll_unmethylated"].view(np.uint32), scores[0::2].view(np.uint32))
    assert np.array_equal(got["ll_methylated"].view(np.uint32), scores[1::2].view(np.uint32))
