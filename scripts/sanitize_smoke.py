"""Small instances of every kernel for compute-sanitizer (memcheck / racecheck / synccheck / initcheck).
Usage (GPU box): compute-sanitizer --tool memcheck python scripts/sanitize_smoke.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from nanopolish_b200 import synth
from nanopolish_b200.engine import Engine

nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
eng = Engine(0)
mid, cid = eng.model_upload(nuc), eng.model_upload(cpg)
rs = synth.gen_reads(6, 1500, nuc, seed=1, drift=True, cpg_keep=0.3)
# forward: scorereads segments (W=32 single strip), wide jobs (chained strips), methylation windows (W<32)
j1 = synth.scorereads_jobs(rs, 250, model_id=mid, rc_every=2)
a = eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, j1.kmer_ranks, j1.jobs)
j2 = synth.scorereads_jobs(rs, 700, model_id=mid)
b = eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, j2.kmer_ranks, j2.jobs)
j3 = synth.methylation_jobs(rs, model_id=cid)
c = eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, j3.kmer_ranks, j3.jobs)
# one-shot pipelined path needs >= 2^20 events and drift 0
rs2 = synth.gen_reads(300, 3600, nuc, seed=2)
j4 = synth.scorereads_jobs(rs2, 500, model_id=mid)
d = eng.hmm_score_batch(rs2.reads, rs2.ev_mean, rs2.ev_start_time, j4.kmer_ranks, j4.jobs)
# viterbi
v, _ = eng.hmm_align_batch(rs.reads, rs.ev_mean, rs.ev_start_time, j1.kmer_ranks, j1.jobs)
# abea + mom
rs3 = synth.gen_reads(5, 1200, nuc, seed=3, rng_scalings=False)
aj, ar, total = synth.abea_jobs(rs3)
pairs, res = eng.abea_batch(rs3.reads, rs3.ev_mean, rs3.ev_start_time, ar, aj, mid, total)
mom = eng.mom_batch(rs3.reads, rs3.ev_mean, ar, aj, mid)
assert np.isfinite(a).all() and np.isfinite(b).all() and np.isfinite(c).all() and np.isfinite(d).all()
assert all(x.shape[0] > 0 for x in v) and (res["n_pairs"] > 0).all()
print("sanitize smoke ok", a.shape, b.shape, c.shape, d.shape, len(v), res["n_pairs"])
# raw-read prologue: trim, event detection (fast path + fallback), calibration, and the fused call
raw, rr, seqs = synth.gen_raw(3, 6000, nuc, seed=9, return_seqs=True)
sig = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])] for r in rr]
sig.append(np.full(900, 70.0, np.float32)); seqs.append(seqs[0][:80])
flat = np.concatenate(sig)
jobs = np.zeros(len(sig), synth.RAW_JOB_DT); rk = []
so = ro = 0
for i, (x, c) in enumerate(zip(sig, seqs)):
    r_ = synth.kmer_ranks_from_codes(c, nuc.k, 4); jobs[i] = (so, ro, x.shape[0], r_.shape[0], 4000.0); rk.append(r_); so += x.shape[0]; ro += r_.shape[0]
ranks = np.concatenate(rk).astype(np.uint32)
rng = eng.trim_raw_batch(raw, rr)
evs = eng.detect_events_batch(raw, rr, synth.event_params(False))
out = eng.load_from_raw_batch(flat, ranks, jobs, mid, synth.event_params(False))
b2e, cal = eng.recalibrate_batch(rs3.reads, rs3.ev_mean, ar, aj, mid, pairs, res)
print("prologue ok", [int(c) for c in out[6]["status"]], int(out[0][-1]))
# eventalign chain kernel (one warp per read walks its windows) and the RNA branch of the fused prologue
rs4 = synth.gen_reads(5, 1200, nuc, seed=4, drift=True)
eng.reads_load(rs4.reads, rs4.ev_mean, rs4.ev_start_time)
pr, mp, rf, rrc, ch = synth.eventalign_chains(rs4, mid)
recs, resu = eng.eventalign_chain(pr, mp, rf, rrc, ch)
assert (resu["status"] == 0).all() and (resu["n_records"] > 1000).all()
prm = synth.event_params(True)
out_rna = eng.load_from_raw_batch(flat, ranks, jobs, mid, prm)
print("eventalign chain ok", [int(x) for x in resu["n_windows"]], "rna prologue", [int(c) for c in out_rna[6]["status"]])
# round 2: base-code jobs (ranks formed by the scheduler's pre-pass), call-methylation enumerated on the device (pair and compact forms),
# variant screening rounds, and the fused event detector with 1 / 2 / 4 warps per read and the repair path (no warm-up)
e = eng.hmm_score_batch_seq(rs.reads, rs.ev_mean, rs.ev_start_time, j1.seq_codes, j1.code_jobs)
assert np.array_equal(e.view(np.uint32), a.view(np.uint32))
ref_b, prs, recs = synth.methylation_records(rs, model_id=cid, rc_every=3)
mp = synth.meth_params("cpg", 6)
so1, sites1, sc1 = eng.methylation_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref_b, prs, recs, mp)
dl, fe = synth.compact_event_alignment(recs, prs, int(recs["ref_len"].sum()))
so2, sites2, sc2 = eng.methylation_batch_compact(rs.reads, rs.ev_mean, rs.ev_start_time, ref_b, dl, fe, recs, mp)
assert sites1.shape[0] > 0 and sites1.tobytes() == sites2.tobytes()
pref, prs_, precs, ppairs = synth.gen_pileup(150, 10, 110, nuc, seed=5, region_start=5000, n_true_variants=2)
pdl, pfe = synth.compact_event_alignment(precs, ppairs, int(precs["ref_len"].sum()))
q, nr, scored = eng.screen_edits_batch(prs_.reads, prs_.ev_mean, prs_.ev_start_time, synth._CODE2DNA[pref], pdl, pfe, precs,
                                       synth.screen_params(5000, 6, 10, 30, 0, 4), indel_bias=0.9)
assert np.isfinite(q[20:100]).any() and scored > 0
for env in ({"NPH_EVENTS_WPR": "1"}, {"NPH_EVENTS_WPR": "2"}, {"NPH_EVENTS_WPR": "4"}, {"NPH_EVENTS_WPR": "2", "NPH_EVENTS_WARMUP": "0"}):
    os.environ.update(env)
    ev2 = eng.detect_events_batch(raw, rr, synth.event_params(False))
    assert all(x.tobytes() == y.tobytes() for x, y in zip(evs, ev2))
    for k_ in env: del os.environ[k_]
print("round-2 kernels ok", sites1.shape[0], int(np.isfinite(q).sum()), [x.shape[0] for x in evs])
# the region calls of `variants` over one window-read walk: fix-homopolymers, all-support and list screening
from tests import hp_cases as hc, screen_cases as scc, support_cases as suc
_, hcnt = hc.device(eng, hc.build(hc.CASES[1]))
_, ucnt = suc.device(eng, suc.build(suc.CASES[0]))
_, lcnt = scc.device(eng, scc.build(scc.CASES[1]))
assert int(hcnt["n_pairs"]) > 0 and int(ucnt["n_pairs"]) > 0 and int(lcnt["n_jobs"]) > 0
print("region calls ok", int(hcnt["n_pairs"]), int(ucnt["n_pairs"]), int(lcnt["n_jobs"]))
# call_haplotype_from_candidates' scores and genotype search: groups of two candidates at ploidy 2
from tests import call_cases as ccs
cg, _, ccnt = ccs.device(eng, ccs.build(ccs.CASES[1]))
assert int(ccnt["n_jobs"]) > 0 and (cg["n_keys"] > 0).any()
print("variant groups ok", int(ccnt["n_groups"]), int(ccnt["n_jobs"]), int(ccnt["n_sets"]))
eng.close()
