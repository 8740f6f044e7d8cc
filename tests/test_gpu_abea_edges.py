"""The CUDA adaptive banded event aligner (abea_kernel) against the port oracle on every edge job of tests/abea_cases.py: the
pairs [0, n_pairs) exactly, all five result fields exactly (avg_log_emission by its bits), and the pairs against the compiled
reference's recorded answers (tests/golden/ref_abea_edges.pkl.xz).  Also: slot bounds on the device buffer, scheduling with
one, sm_count + 1 and more than 20 x sm_count jobs, the staged path, and the method-of-moments kernel at its staging edges."""
import numpy as np
import pytest
import torch

from nanopolish_b200 import synth
from tests import abea_cases as ac
from tests import ref_calls

pytestmark = pytest.mark.gpu
NPH_ERR_INVALID = -3


@pytest.fixture(scope="module")
def nuc(engine):
    m = synth.load_model("nucleotide")
    return m, engine.model_upload(m)


def _compare(b, pairs_g, res_g, model, port, what):
    po, ro, _ = port.abea_batch(b.reads, b.ev_mean, b.ev_start_time, model, b.kmer_ranks, b.jobs, b.pairs_total, threads=8)
    for j in range(b.jobs.shape[0]):
        o, n = int(b.jobs[j]["pairs_off"]), int(ro[j]["n_pairs"])
        assert res_g[j].tobytes() == ro[j].tobytes(), f"{what} job {j} (K={int(b.jobs[j]['n_kmers'])}): record {res_g[j]} vs oracle {ro[j]}"
        assert np.array_equal(pairs_g[o:o + n], po[o:o + n]), f"{what} job {j}: pairs differ"
    return po, ro


def test_edge_jobs_match_oracle_and_reference(engine, nuc, port_oracle):
    model, mid = nuc
    b = ac.batch(model, port_oracle, levels=False)
    pairs, res = engine.abea_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, b.jobs, mid, b.pairs_total)
    _compare(b, pairs, res, model, port_oracle, "edge")
    rec = ref_calls.case_answers("ref_abea_edges.pkl.xz", "abea_edges")
    n_ref = 0
    for j in range(b.jobs.shape[0]):
        want = rec[ac.fingerprint(b, j)]
        if int(res[j]["status"]) == 0:
            o, n = int(b.jobs[j]["pairs_off"]), int(res[j]["n_pairs"])
            assert want is not None and want[0] == n and ac.pairs_hash(pairs["ref_pos"][o:o + n], pairs["read_pos"][o:o + n]) == want[1], \
                f"job {j}: pairs differ from the reference's"
            n_ref += 1
    assert n_ref > 150
    st = res["status"]
    assert (st == ac.PAIRS_OVERFLOW).sum() >= 2 and ((st & ac.LOW_EMISSION) != 0).any() and ((st & ac.MAX_GAP_BIT) != 0).any()


def test_slot_bounds_on_device(engine, nuc, port_oracle):
    """a batch whose slots tile pairs_total, then the same jobs with gaps of that size between smaller slots: the gaps keep the
    first run's values (the kernel writes nothing outside a slot).  The first run is staged, the second one-shot."""
    model, mid = nuc
    G = 37
    jobs = ac.capacity_jobs() + ac.backtrack_jobs() + ac.trim_jobs()
    b2 = ac.make_batch(jobs, model, gap=G, port=port_oracle)
    b1 = ac.make_batch(jobs, model, gap=0, port=port_oracle)
    b1.jobs["pairs_cap"] = b2.jobs["pairs_cap"] + G
    b1.jobs["pairs_off"] = b2.jobs["pairs_off"]
    b1.pairs_total = b2.pairs_total
    assert int(b1.jobs["pairs_off"][-1] + b1.jobs["pairs_cap"][-1]) == b1.pairs_total
    engine.reads_load(b1.reads, b1.ev_mean, b1.ev_start_time)
    engine.abea_jobs_load(b1.kmer_ranks, b1.jobs, mid, b1.pairs_total)
    engine.abea_run()
    p1, r1 = engine.abea_fetch()
    _compare(b1, p1, r1, model, port_oracle, "tiled")
    p2, r2 = engine.abea_batch(b2.reads, b2.ev_mean, b2.ev_start_time, b2.kmer_ranks, b2.jobs, mid, b2.pairs_total)
    _compare(b2, p2, r2, model, port_oracle, "gapped")
    for j in range(b2.jobs.shape[0]):
        g0 = int(b2.jobs[j]["pairs_off"] + b2.jobs[j]["pairs_cap"])
        assert p2[g0:g0 + G].tobytes() == p1[g0:g0 + G].tobytes(), f"job {j} wrote past its slot"
    # the staged path on the gapped jobs gives the one-shot call's answer
    engine.reads_load(b2.reads, b2.ev_mean, b2.ev_start_time)
    engine.abea_jobs_load(b2.kmer_ranks, b2.jobs, mid, b2.pairs_total)
    engine.abea_run()
    p3, r3 = engine.abea_fetch()
    assert r3.tobytes() == r2.tobytes() and p3.tobytes() == p2.tobytes()


@pytest.mark.parametrize("which", ["one", "sm+1", "20sm+1"])
def test_scheduling(engine, nuc, port_oracle, which):
    """one job; sm_count + 1 jobs (two active warps per CTA); more than 20 x sm_count jobs mixing long and tiny reads and equal
    band counts, so warps take further jobs on scratch they used before"""
    model, mid = nuc
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = {"one": 1, "sm+1": sm + 1, "20sm+1": 20 * sm + 1}[which]
    b = ac.make_batch(ac.scheduling_jobs(n, seed=10 + n), model)
    pairs, res = engine.abea_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, b.jobs, mid, b.pairs_total)
    _compare(b, pairs, res, model, port_oracle, which)


def test_mom_edges_bit_exact(engine, nuc, port_oracle):
    model, mid = nuc
    b = ac.mom_batch(model)
    got = engine.mom_batch(b.reads, b.ev_mean, b.kmer_ranks, b.jobs, mid)
    rec = ref_calls.case_answers("ref_abea_edges.pkl.xz", "mom")
    for j in range(b.jobs.shape[0]):
        want = np.array(port_oracle.mom(b.reads, b.ev_mean, model, b.kmer_ranks, b.jobs[j]))
        assert got[j].view(np.uint64).tolist() == want.view(np.uint64).tolist(), f"MoM job {j}: {got[j]} vs {want}"
        assert got[j].tolist() == list(rec[ac.fingerprint(b, j)])


@pytest.mark.parametrize("level", ac.LEVELS)
def test_out_of_range_levels(engine, nuc, port_oracle, level):
    """one level outside the pA range mid-read and one in the first 20 events.  Levels beyond NPH_ABEA_MAX_LEVEL (2048) or NaN
    are refused (include/nph.h): at +-inf the kernel's Gaussian was NaN where the reference's is -inf, and in the 2^64 window
    it was -inf where the reference's is finite.  Every level the device takes is compared, 2048 itself included."""
    from nanopolish_b200._lib import NphError
    model, mid = nuc
    b = ac.make_batch([j for j in ac.level_jobs() if j.levels[0][1] == level], model)
    if not ac.in_domain(b.ev_mean):
        assert level not in ("max",)
        with pytest.raises(NphError) as ex:
            engine.abea_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, b.jobs, mid, b.pairs_total)
        assert ex.value.status == NPH_ERR_INVALID
        engine.reads_load(b.reads, b.ev_mean, b.ev_start_time)
        with pytest.raises(NphError) as ex:
            engine.abea_jobs_load(b.kmer_ranks, b.jobs, mid, b.pairs_total)
        assert ex.value.status == NPH_ERR_INVALID
        return
    assert level == "max"
    pairs, res = engine.abea_batch(b.reads, b.ev_mean, b.ev_start_time, b.kmer_ranks, b.jobs, mid, b.pairs_total)
    _compare(b, pairs, res, model, port_oracle, level)


def _raw_jobs(signals, seqs, k, sample_rate=4000.0):
    jobs = np.zeros(len(signals), synth.RAW_JOB_DT)
    ranks = []
    soff = roff = 0
    for i, (x, c) in enumerate(zip(signals, seqs)):
        rk = synth.kmer_ranks_from_codes(c, k, 4)
        jobs[i] = (soff, roff, x.shape[0], rk.shape[0], sample_rate)
        ranks.append(rk)
        soff += x.shape[0]
        roff += rk.shape[0]
    return np.concatenate(signals), np.concatenate(ranks).astype(np.uint32), jobs


@pytest.mark.parametrize("where,value,refused", [("none", 0.0, False), ("slice", np.nan, True), ("slice", np.inf, True),
                                                 ("slice", 2049.0, True), ("unused", -2049.0, True), ("unused", 2048.0, False)])
def test_raw_prologue_sample_domain(engine, nuc, where, value, refused):
    """nph_load_from_raw_batch refuses a raw buffer with a sample outside +-NPH_ABEA_MAX_LEVEL or NaN, inside a job's slice or
    in samples no job reads, before any step runs; 2048 itself is taken"""
    from nanopolish_b200._lib import NphError
    model, mid = nuc
    raw, rr, seqs = synth.gen_raw(2, 6000, model, seed=901, return_seqs=True)
    signals = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])].copy() for r in rr]
    flat, ranks, jobs = _raw_jobs(signals, seqs, model.k)
    flat = np.concatenate([flat, np.full(16, 90.0, np.float32)])          # samples after every job's slice
    if where == "slice":
        flat[int(jobs[1]["sample_off"]) + 3000] = value
    elif where == "unused":
        flat[-5] = value
    if refused:
        with pytest.raises(NphError) as ex:
            engine.load_from_raw_batch(flat, ranks, jobs, mid, synth.event_params(False))
        assert ex.value.status == NPH_ERR_INVALID
    else:
        off = engine.load_from_raw_batch(flat, ranks, jobs, mid, synth.event_params(False))[0]
        assert int(off[-1]) > 0
