"""`nanopolish scorereads` — model_score (src/nanopolish_scorereads.cpp:116-203) as a batch generator over
profile_hmm_score (nanopolish_b200/host/nph_scorereads.*): the segments it cuts out of a read's event alignment, and the
per-read score = sum(segment scores) / sum(events).  The enumeration is checked on the CPU (the event alignments come
from the C++ cursors fed by the plain-C Viterbi), the scores on the GPU against the oracle's profile_hmm_score.

Pin status: profile_hmm_score and align_read_to_ref are pinned to the compiled reference (tests/test_oracle_vs_ref.py); model_score's own
segment cutting and normalisation are checked against a restatement of nanopolish_scorereads.cpp:116-203 only (scorereads' main() reads
fast5 files, which the harness cannot supply)."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from oracle import eventalign_py as EP
from tests import eventalign_cases as EC
from tests import host_mirror as hm

host = hm.fixture()


@pytest.fixture(scope="module")
def cases():
    return EC.build_cases()


def _expected_segments(cs, restated, rs):
    """model_score's loop, restated: per read the list of (event_start, event_stop, stride, rc, ranks)"""
    out = []
    for c, (al, _) in zip(cs, restated):
        segs = []
        for start in range(EC.EPS, len(al) - EC.EPS, EC.EPS):
            a0, a1 = al[start], al[start + EC.EPS]
            seg = c["fetched"][a0.ref_position - c["ref_pos"]:a1.ref_position - c["ref_pos"] + 1]
            if len(seg) <= EC.K:
                continue
            codes = synth.encode(EP.disambiguate(seg), "nucleotide")
            rc = bool(al[0].rc)
            ranks = synth.dna_rc_kmer_ranks(codes, EC.K) if rc else synth.kmer_ranks_from_codes(codes, EC.K, 4)
            segs.append((a0.event_idx, a1.event_idx, 1 if a0.event_idx <= a1.event_idx else -1, int(rc), ranks.astype(np.uint32)))
        out.append(segs)
    return out


def _restate(cases, port_oracle):
    model, rs, cs = cases
    out = []
    for c in cs:
        al = EP.align_read_to_ref(c["read"], c["contig_name"], c["fetched"], c["ref_pos"], c["flag"], c["cigar"], c["read_idx"],
                                  EC.port_align_fn(port_oracle, rs, model, EC.read_slot(c, rs.n_reads)), *c["region"])
        out.append((al, 0))
    return out


def _check_jobs(jobs, ranks, want):
    flat = [s for segs in want for s in segs]
    assert jobs.shape[0] == len(flat) > 10
    for jb, (e0, e1, stride, rc, rk) in zip(jobs, flat):
        assert (int(jb["event_start"]), int(jb["event_stop"]), int(jb["stride"]), int(jb["rc"]), int(jb["flags"])) == (e0, e1, stride, rc, 0)
        assert np.array_equal(ranks[int(jb["rank_off"]):int(jb["rank_off"]) + int(jb["n_kmers"])], rk)


def test_model_score_segments_on_cpu(host, cases, port_oracle):
    model, rs, cs = cases
    restated = _restate(cases, port_oracle)
    EC.load_batch(host, cases)
    EC.drive_rounds(host, cs, rs, model, port_oracle)
    jobs, ranks, _ = EC.scorereads(host, cases, mode=0)
    _check_jobs(jobs, ranks, _expected_segments(cs, restated, rs))
    host.nphh_ea_begin()


@pytest.mark.gpu
def test_model_score_on_device(host, cases, port_oracle):
    model, rs, cs = cases
    restated = _restate(cases, port_oracle)
    EC.load_batch(host, cases)
    assert host.nphh_ea_run(C.c_double(1.0)) >= 0, host.nphh_last_error()
    jobs, ranks, sc = EC.scorereads(host, cases, mode=1)
    want = _expected_segments(cs, restated, rs)
    _check_jobs(jobs, ranks, want)
    # per-read score from the oracle's profile_hmm_score of the same segments (float scores summed in double, in order)
    for i, (c, segs) in enumerate(zip(cs, want)):
        slot = EC.read_slot(c, rs.n_reads)
        total, nev = 0.0, 0
        for e0, e1, stride, rc, rk in segs:
            jb = np.zeros(1, synth.HMM_JOB_DT)
            jb[0] = (0, slot, 0, e0, e1, rk.shape[0], stride, rc, 0, 0)
            v, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [model], rk, jb)
            total += float(v[0]); nev += abs(e0 - e1) + 1
        assert sc[i][1] == nev and sc[i][2] == len(segs)
        assert sc[i][0] == (total / nev if nev else 1.0)
    host.nphh_ea_begin()
