"""The C++ host mirror of the reference call surface (nanopolish_b200/host/): Alphabet known answers
copied from the reference's own unit test expectations (src/test/nanopolish_test.cpp:27-237),
randomised agreement with the compiled reference, and — on the GPU — profile_hmm_score /
profile_hmm_score_set / adaptive_banded_simple_event_align called exactly like a nanopolish caller."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import host_mirror as hm

OPS = {"reverse_complement": 0, "methylate": 1, "unmethylate": 2, "disambiguate": 3}
host = hm.fixture()


def _op(lib, alphabet, op, s):
    out = C.create_string_buffer(len(s) + 16)
    n = lib.nphh_alphabet_op(alphabet.encode(), OPS[op], s.encode(), out)
    assert n >= 0, lib.nphh_last_error()
    return out.raw[:n].decode()


KNOWN = [
    ("cpg", "methylate", "C", "C"), ("cpg", "methylate", "CG", "MG"), ("cpg", "methylate", "GC", "GC"),
    ("cpg", "methylate", "CGCG", "MGMG"), ("cpg", "methylate", "AAGCGT", "AAGMGT"), ("cpg", "methylate", "CGGCGT", "MGGMGT"),
    ("cpg", "methylate", "CGCGC", "MGMGC"),
    ("cpg", "unmethylate", "C", "C"), ("cpg", "unmethylate", "M", "C"), ("cpg", "unmethylate", "MG", "CG"), ("cpg", "unmethylate", "MT", "MT"),
    ("cpg", "disambiguate", "", ""), ("cpg", "disambiguate", "M", "M"), ("cpg", "disambiguate", "MT", "AT"),
    ("cpg", "disambiguate", "MG", "MG"), ("cpg", "disambiguate", "AMG", "AMG"), ("cpg", "disambiguate", "CAM", "CAM"),
    ("cpg", "reverse_complement", "M", "G"), ("cpg", "reverse_complement", "C", "G"), ("cpg", "reverse_complement", "MG", "MG"),
    ("cpg", "reverse_complement", "CG", "CG"), ("cpg", "reverse_complement", "AM", "GT"), ("cpg", "reverse_complement", "AMG", "MGT"),
    ("cpg", "reverse_complement", "AAAMG", "MGTTT"), ("cpg", "reverse_complement", "MGMG", "MGMG"),
    ("cpg", "reverse_complement", "MGAMG", "MGTMG"),
    ("dam", "methylate", "GAT", "GAT"), ("dam", "methylate", "GATC", "GMTC"), ("dam", "methylate", "GATCGATC", "GMTCGMTC"),
    ("dam", "methylate", "GMTCGATC", "GMTCGMTC"),
    ("dam", "unmethylate", "M", "A"), ("dam", "unmethylate", "MTC", "ATC"), ("dam", "unmethylate", "GMTCGM", "GATCGA"),
    ("dam", "unmethylate", "MA", "MA"), ("dam", "unmethylate", "CM", "CM"),
    ("dam", "disambiguate", "GMTC", "GMTC"), ("dam", "disambiguate", "GMA", "GAA"), ("dam", "disambiguate", "MT", "MT"),
    ("dam", "reverse_complement", "M", "T"), ("dam", "reverse_complement", "GM", "TC"), ("dam", "reverse_complement", "GMT", "MTC"),
    ("dam", "reverse_complement", "GMTC", "GMTC"), ("dam", "reverse_complement", "MTC", "GMT"), ("dam", "reverse_complement", "GAT", "ATC"),
    ("dcm", "methylate", "CCAGG", "CMAGG"), ("dcm", "methylate", "CCTGG", "CMTGG"), ("dcm", "methylate", "CCAG", "CCAG"),
    ("dcm", "methylate", "CCAGGCCTGG", "CMAGGCMTGG"), ("dcm", "methylate", "CCAGGCCTG", "CMAGGCCTG"),
    ("dcm", "unmethylate", "M", "C"), ("dcm", "unmethylate", "MAGG", "CAGG"), ("dcm", "unmethylate", "MTG", "CTG"),
]


@pytest.mark.parametrize("alphabet,op,inp,want", KNOWN)
def test_alphabet_known_answers(host, alphabet, op, inp, want):
    assert _op(host, alphabet, op, inp) == want


def test_ranks_and_lexicographic_order(host):
    assert host.nphh_kmer_rank(b"nucleotide", b"GATGA", 5) == 568          # "string functions" test
    for a, bases in (("nucleotide", "ACGT"), ("cpg", "ACGMT")):
        kmer = bases[0] * 3
        out = C.create_string_buffer(8)
        n = len(bases) ** 3
        for i in range(n - 1):
            host.nphh_lexicographic_next(a.encode(), kmer.encode(), out)
            nxt = out.value.decode()
            assert host.nphh_kmer_rank(a.encode(), nxt.encode(), 3) - host.nphh_kmer_rank(a.encode(), kmer.encode(), 3) == 1
            kmer = nxt
        assert kmer == bases[-1] * 3


def test_alphabet_ops_match_compiled_reference(host, ref_oracle):
    rng = np.random.default_rng(12)
    for alphabet, motif, meth in (("cpg", "CG", "MG"), ("gpc", "GC", "GM"), ("dam", "GATC", "GMTC"), ("dcm", "CCAGG", "CMAGG")):
        for _ in range(150):
            n = int(rng.integers(1, 40))
            s = "".join(rng.choice(list("ACGT"), n))
            for _ in range(int(rng.integers(0, 3))):         # plant (possibly overlapping / truncated) motifs
                p = int(rng.integers(0, n))
                s = (s[:p] + motif + s[p:])[:n + 3]
            m = _op(host, alphabet, "methylate", s)
            assert m == ref_oracle.alphabet_op(alphabet, 1, s.encode()).decode()
            for op, code in (("reverse_complement", 0), ("unmethylate", 2), ("disambiguate", 3)):
                for x in (s, m):
                    assert _op(host, alphabet, op, x) == ref_oracle.alphabet_op(alphabet, code, x.encode()).decode(), (alphabet, op, x)


def test_kmer_ranks_match_compiled_reference(host, ref_oracle):
    rng = np.random.default_rng(5)
    hn, hc = ref_oracle.builtin_model("nucleotide"), ref_oracle.builtin_model("cpg")
    for _ in range(60):
        n = int(rng.integers(6, 80))
        s = "".join(rng.choice(list("ACGT"), n))
        for rc in (0, 1):
            out = np.zeros(n, np.uint32)
            k = host.nphh_kmer_ranks(b"nucleotide", s.encode(), 6, rc, out.ctypes.data_as(C.c_void_p))
            assert np.array_equal(out[:k], ref_oracle.kmer_ranks(hn, s.encode(), bool(rc)))
            m = _op(host, "cpg", "methylate", s)
            k = host.nphh_kmer_ranks(b"cpg", m.encode(), 6, rc, out.ctypes.data_as(C.c_void_p))
            assert np.array_equal(out[:k], ref_oracle.kmer_ranks(hc, m.encode(), bool(rc)))


def test_rolling_ranks_equal_get_kmer_rank(host):
    """HmmBatch::add fills the ranks by one rolling pass; they must be HMMInputSequence::get_kmer_rank's, both strands,
    plain and methylation alphabets (the rc strand of a methylated sequence is not a per-base complement)."""
    rng = np.random.default_rng(12)
    for alphabet, sym in (("nucleotide", "ACGT"), ("cpg", "ACGT")):
        for rep in range(20):
            seq = "".join(sym[c] for c in rng.integers(0, 4, int(rng.integers(6, 260))))
            if alphabet == "cpg" and rep % 2:
                seq = seq.replace("CG", "MG")
            for rc in (0, 1):
                assert host.nphh_kmer_ranks_rolling_check(alphabet.encode(), seq.encode(), 6, rc) == 0, (alphabet, seq, rc)
    assert host.nphh_kmer_ranks_rolling_check(b"nucleotide", b"ACG", 6, 0) == 0


# ---- GPU: the reference's free functions through the mirror -----------------------------------
@pytest.mark.gpu
def test_profile_hmm_score_like_a_caller(host, port_oracle):
    nuc = synth.load_model("nucleotide")
    rs = synth.gen_reads(3, 900, nuc, seed=61, drift=True)
    jobs = synth.scorereads_jobs(rs, 200, rc_every=2, keep_seqs=True)
    want, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc], jobs.kmer_ranks, jobs.jobs)
    mh = hm.register_model(host, nuc)
    rh = hm.register_reads(host, rs, mh)
    host.nphh_set_indel_bias(C.c_double(1.0))
    # one call per job, exactly the reference's signature
    for j in range(min(4, jobs.jobs.shape[0])):
        jb = jobs.jobs[j]
        out = C.c_float()
        rc = host.nphh_profile_hmm_score(rh[int(jb["read"])], mh, jobs.seqs[j], int(jb["event_start"]), int(jb["event_stop"]),
                                         int(jb["rc"]), int(jb["flags"]), C.byref(out))
        assert rc == 0, host.nphh_last_error()
        assert np.float32(out.value).view(np.uint32) == want[j].view(np.uint32)
    # one HmmBatch for all of them
    n = jobs.jobs.shape[0]
    buf = b"".join(jobs.seqs)
    off = np.zeros(n + 1, np.uint64); off[1:] = np.cumsum([len(s) for s in jobs.seqs])
    got = np.zeros(n, np.float32)
    p = hm.p
    reads = np.ascontiguousarray(np.array(rh, np.int32)[jobs.jobs["read"]])
    models = np.full(n, mh, np.int32)
    rc = host.nphh_profile_hmm_score_many(C.c_size_t(n), p(reads), p(models), C.c_char_p(buf), p(off),
                                          p(np.ascontiguousarray(jobs.jobs["event_start"])), p(np.ascontiguousarray(jobs.jobs["event_stop"])),
                                          p(np.ascontiguousarray(jobs.jobs["rc"])), p(np.ascontiguousarray(jobs.jobs["flags"].astype(np.uint32))), p(got))
    assert rc == 0, host.nphh_last_error()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # rc / stride mismatch is rejected where the reference asserts
    out = C.c_float()
    jb = jobs.jobs[0]
    assert host.nphh_profile_hmm_score(rh[0], mh, jobs.seqs[0], int(jb["event_stop"]), int(jb["event_start"]), 0, 0, C.byref(out)) != 0


@pytest.mark.gpu
def test_profile_hmm_score_set_like_a_caller(host, port_oracle):
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    rs = synth.gen_reads(2, 600, nuc, seed=88, cpg_keep=0.4)
    mj = synth.methylation_jobs(rs, model_id=1, keep_seqs=True, max_groups_per_read=3)
    mh, ch = hm.register_model(host, nuc), hm.register_model(host, cpg)
    rh = hm.register_reads(host, rs, mh)
    for r in rh:
        host.nphh_read_add_model(r, b"cpg", ch)
    for g in range(mj.jobs.shape[0] // 2):
        ju = mj.jobs[2 * g]
        useq = mj.seqs[2 * g]            # unmethylated bases (ACGT only): valid in the nucleotide alphabet too
        mseq = mj.seqs[2 * g + 1]
        # oracle: score(nucleotide seq, nucleotide model) (+) score(methylated seq, cpg model), each - log 2
        k = 6
        jobs = np.zeros(2, synth.HMM_JOB_DT)
        r_u = synth.kmer_ranks_from_codes(synth.encode(useq, "nucleotide"), k, 4)
        r_m = synth.kmer_ranks_from_codes(synth.encode(mseq, "cpg"), k, 5)
        jobs[0] = (0, ju["read"], 0, ju["event_start"], ju["event_stop"], r_u.shape[0], 1, 0, ju["flags"], 0)
        jobs[1] = (r_u.shape[0], ju["read"], 1, ju["event_start"], ju["event_stop"], r_m.shape[0], 1, 0, ju["flags"], 0)
        ranks = np.concatenate([r_u, r_m]).astype(np.uint32)
        sc, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [nuc, cpg], ranks, jobs)
        want = np.float32(port_oracle.score_set_combine(sc))
        out = C.c_float()
        seqs = (C.c_char_p * 2)(useq, mseq)
        alphs = (C.c_char_p * 2)(b"nucleotide", b"cpg")
        rc = host.nphh_profile_hmm_score_set(rh[int(ju["read"])], mh, 2, seqs, alphs, int(ju["event_start"]), int(ju["event_stop"]),
                                             0, int(ju["flags"]), C.byref(out))
        assert rc == 0, host.nphh_last_error()
        assert np.float32(out.value).view(np.uint32) == want.view(np.uint32)


@pytest.mark.gpu
def test_abea_and_mom_like_a_caller(host, port_oracle):
    nuc = synth.load_model("nucleotide")
    rs = synth.gen_reads(2, 700, nuc, seed=17, rng_scalings=False)
    jobs, ranks, total = synth.abea_jobs(rs)
    po, ro, _ = port_oracle.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, nuc, ranks, jobs, total)
    mh = hm.register_model(host, nuc)
    rh = hm.register_reads(host, rs, mh)
    for i in range(rs.n_reads):
        seq = synth._CODE2DNA[rs.seq_codes[i]].tobytes()
        cap = int(jobs[i]["pairs_cap"])
        pairs = np.zeros((cap, 2), np.int32)
        n = host.nphh_abea(rh[i], mh, seq, pairs.ctypes.data_as(C.c_void_p), C.c_size_t(cap))
        assert n == int(ro[i]["n_pairs"]) and n > 0
        w = po[int(jobs[i]["pairs_off"]):int(jobs[i]["pairs_off"]) + n]
        assert np.array_equal(pairs[:n, 0], w["ref_pos"]) and np.array_equal(pairs[:n, 1], w["read_pos"])
        out = np.zeros(4)
        assert host.nphh_mom(rh[i], mh, seq, out.ctypes.data_as(C.c_void_p)) == 0
        sh, sc = port_oracle.mom(rs.reads, rs.ev_mean, nuc, ranks, jobs[i])
        assert out[0] == sh and out[1] == sc and out[2] == 0.0 and out[3] == 1.0


@pytest.mark.gpu
def test_load_from_raw_like_a_caller(host, port_oracle):
    """nph::load_from_raw over a batch (raw samples + basecalls in, SquiggleReads out) against the same chain through
    the oracle: identical events, bit-identical scalings, identical base_to_event_map and the same reads dropped."""
    from oracle.prep_chain import oracle_chain
    nuc = synth.load_model("nucleotide")
    raw, rr, seqs = synth.gen_raw(4, 24000, nuc, seed=901, return_seqs=True)
    signals = [raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])] for r in rr]
    g = np.random.default_rng(11)                                                  # homopolymer runs: < 200 'M' events, calibration refuses
    codes = np.concatenate([np.concatenate([g.integers(0, 4, 8, dtype=np.uint8), np.full(20, g.integers(0, 4), np.uint8)]) for _ in range(14)])
    ranks = synth.kmer_ranks_from_codes(codes, nuc.k, 4)
    dwell = np.maximum(1, g.geometric(1.0 / 9.0, ranks.shape[0]))
    signals.append((np.repeat(nuc.level_mean[ranks], dwell) + 1.2 * np.repeat(nuc.level_stdv[ranks], dwell) * g.standard_normal(int(dwell.sum()))).astype(np.float32))
    seqs.append(codes)
    short, _, sq = synth.gen_raw(1, 2400, nuc, seed=77, return_seqs=True)          # too short once trimmed: alignment fails
    signals.append(short); seqs.append(sq[0])
    signals.append(np.full(5000, 101.0, np.float32)); seqs.append(seqs[0][:400])   # flat: nothing survives the trim
    noise = np.random.default_rng(5).uniform(60, 130, 20000).astype(np.float32)    # no sequence signal at all
    signals.append(noise); seqs.append(seqs[1][:2000])
    n = len(signals)
    want = oracle_chain(port_oracle, nuc, signals, seqs)
    mh = hm.register_model(host, nuc)
    soff = np.zeros(n + 1, np.uint64); soff[1:] = np.cumsum([s.shape[0] for s in signals])
    qoff = np.zeros(n + 1, np.uint64); qoff[1:] = np.cumsum([c.shape[0] for c in seqs])
    seqbuf = b"".join(synth._CODE2DNA[c].tobytes() for c in seqs)
    eoff = np.zeros(n, np.uint64); eoff[1:] = np.cumsum([s.shape[0] // 2 + 8 for s in signals])[:-1]
    room = int(eoff[-1]) + signals[-1].shape[0] // 2 + 8
    n_events = np.zeros(n, np.uint32); scal = np.zeros((n, 5)); stats = np.zeros(5, np.uint64)
    mean = np.zeros(room, np.float32); stdv = np.zeros(room, np.float32); start = np.zeros(room, np.float64); dur = np.zeros(room, np.float32)
    b2e = np.full((int(qoff[-1]), 2), -7, np.int32)
    flat = np.concatenate(signals)
    p = hm.p
    host.nphh_set_load_flags(2)                                 # SRF_LOAD_RAW_SAMPLES: keep the trimmed samples on every read
    try:
        rc = host.nphh_load_from_raw(mh, n, p(flat), p(soff), seqbuf, p(qoff), C.c_double(4000.0), p(n_events), p(scal), p(eoff), p(mean), p(stdv),
                                     p(start), p(dur), p(b2e), p(stats))
    finally:
        host.nphh_set_load_flags(0)
    assert rc >= 0, host.nphh_last_error()
    for i in range(n):                                          # samples[i] = rt.raw[rt.start + i] (squiggle_read.cpp:251-258)
        s0, s1 = want[i]["range"]
        assert host.nphh_read_num_samples(rc + i) == s1 - s0
        if s1 > s0:
            assert host.nphh_read_sample(rc + i, C.c_size_t(0)) == signals[i][s0] and host.nphh_read_sample(rc + i, C.c_size_t(s1 - s0 - 1)) == signals[i][s1 - 1]
    dropped = 0
    for i in range(n):
        w = want[i]
        if w["events"] is None:
            assert n_events[i] == 0
            continue
        keep = w["n_pairs"] > 0 and int(w["cal"]["status"]) == 0
        dropped += not keep
        if not keep:
            assert n_events[i] == 0
        else:
            ev = w["events"]; o = int(eoff[i])
            assert n_events[i] == ev.shape[0]
            assert np.array_equal(mean[o:o + ev.shape[0]], ev["mean"]) and np.array_equal(stdv[o:o + ev.shape[0]], ev["stdv"])
            assert np.array_equal(dur[o:o + ev.shape[0]], w["duration"]) and np.array_equal(start[o:o + ev.shape[0]], w["start_time"])
        if w["n_pairs"] > 0:
            c = w["cal"]
            exp = (c["shift"], c["scale"], c["drift"], c["var"]) if not int(c["status"]) & 2 else (w["mom"][0], w["mom"][1], 0.0, 1.0)
            assert tuple(scal[i][:4]) == tuple(float(v) for v in exp) and scal[i][4] == c["events_per_base"]
            nk = seqs[i].shape[0] - nuc.k + 1
            got = b2e[int(qoff[i]):int(qoff[i]) + nk]
            assert np.array_equal(got[:, 0], w["b2e"]["start"]) and np.array_equal(got[:, 1], w["b2e"]["stop"])
        else:
            assert tuple(scal[i][:2]) == w["mom"] and scal[i][4] == 0.0
    assert [int(v) for v in stats] == [n, 1, stats[2], stats[3], stats[4]] and int(stats[2] + stats[3] + stats[4]) == dropped
    assert (n_events[:4] > 2000).all() and (n_events[4:] == 0).all()
    assert int(want[4]["cal"]["status"]) == 2 and want[5]["n_pairs"] == 0 and want[6]["events"] is None and [int(v) for v in stats[1:4]] == [1, 2, 1]


@pytest.mark.gpu
def test_load_from_raw_direct_rna_like_a_caller(host, port_oracle):
    """The RNA branch through nph::load_from_raw: basecalls with U, a 5-mer u_to_t_rna model, RNA detector parameters,
    events turned around to 5'->3' (src/nanopolish_squiggle_read.cpp:192-213,262-265) — vs the chain through the oracle."""
    from oracle.prep_chain import oracle_chain
    m6 = synth.load_model("nucleotide")
    sd5 = m6.level_stdv.reshape(1024, 4).mean(1)
    rna = synth.PoreModel("derived.u_to_t_rna.5mer", 5, "nucleotide", m6.level_mean.reshape(1024, 4).mean(1), sd5, np.log(sd5))
    raw, rr, seqs = synth.gen_raw(3, 50000, rna, seed=431, mean_dwell=40.0, return_seqs=True)
    signals = [np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])][::-1]) for r in rr]
    n = len(signals)
    want = oracle_chain(port_oracle, rna, signals, seqs, sample_rate=3012.0, rna=True)
    mean5, sd = np.ascontiguousarray(rna.level_mean), np.ascontiguousarray(rna.level_stdv)
    lsd = np.ascontiguousarray(rna.level_log_stdv)
    p = hm.p
    mh = host.nphh_model_create(b"u_to_t_rna", 5, 1024, p(mean5), p(sd), p(lsd))
    assert mh >= 0, host.nphh_last_error()
    soff = np.zeros(n + 1, np.uint64); soff[1:] = np.cumsum([s.shape[0] for s in signals])
    qoff = np.zeros(n + 1, np.uint64); qoff[1:] = np.cumsum([c.shape[0] for c in seqs])
    seqbuf = b"".join(synth._CODE2DNA[c].tobytes() for c in seqs).replace(b"T", b"U")        # what an RNA basecaller writes
    eoff = np.zeros(n, np.uint64); eoff[1:] = np.cumsum([s.shape[0] // 2 + 8 for s in signals])[:-1]
    room = int(eoff[-1]) + signals[-1].shape[0] // 2 + 8
    n_events = np.zeros(n, np.uint32); scal = np.zeros((n, 5)); stats = np.zeros(5, np.uint64)
    mean = np.zeros(room, np.float32); stdv = np.zeros(room, np.float32); start = np.zeros(room, np.float64); dur = np.zeros(room, np.float32)
    b2e = np.full((int(qoff[-1]), 2), -7, np.int32)
    flat = np.concatenate(signals)
    host.nphh_set_rna(1)
    try:
        rc = host.nphh_load_from_raw(mh, n, p(flat), p(soff), seqbuf, p(qoff), C.c_double(3012.0), p(n_events), p(scal), p(eoff), p(mean), p(stdv),
                                     p(start), p(dur), p(b2e), p(stats))
    finally:
        host.nphh_set_rna(0)
    assert rc >= 0, host.nphh_last_error()
    for i in range(n):
        w = want[i]
        assert w["n_pairs"] > 0 and int(w["cal"]["status"]) == 0
        ev = w["events"]; o = int(eoff[i])
        assert n_events[i] == ev.shape[0]
        assert np.array_equal(mean[o:o + ev.shape[0]], ev["mean"]) and np.array_equal(start[o:o + ev.shape[0]], w["start_time"])
        c = w["cal"]
        assert tuple(scal[i]) == (c["shift"], c["scale"], c["drift"], c["var"], c["events_per_base"])
        nk = seqs[i].shape[0] - 5 + 1
        got = b2e[int(qoff[i]):int(qoff[i]) + nk]
        assert np.array_equal(got[:, 0], w["b2e"]["start"]) and np.array_equal(got[:, 1], w["b2e"]["stop"])
    assert [int(v) for v in stats] == [n, 0, 0, 0, 0]
