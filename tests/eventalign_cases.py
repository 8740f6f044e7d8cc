"""Synthetic eventalign inputs shared by the oracle, host-logic and GPU tests (SURVEY.md 8f N1): reads as
load_from_raw leaves them (events, scalings, basecalled sequence, base-to-event map) plus what the reference pulls
from the BAM record and the FASTA (position, flag, CIGAR, contig).  Seeded; no file access.  Also the ways the host
mirror's EventAligner and ScoreReads take them: load_batch, drive_rounds and scorereads."""
import ctypes as C

import numpy as np

from nanopolish_b200 import synth
from oracle import eventalign_py as EP
from tests import host_mirror as hm

K = 6
EPS = 200          # events per segment of scorereads (the reference uses 500 on whole reads; the test reads have ~1 500 events)
_DNA = "ACGT"


def _edit_script(read_seq: str, rng, soft_clip: int, with_skip: bool):
    """Walk the (reference-oriented) read and derive a reference + CIGAR: matches with a few substitutions, short
    insertions and deletions, optionally one reference skip (two BAM segments), a leading soft clip."""
    ops, ref = [], []
    i = 0
    if soft_clip:
        ops.append((soft_clip, "S")); i = soft_clip
    n = len(read_seq)
    block = 0
    while i < n:
        m = int(min(n - i, rng.integers(120, 320)))
        seg = list(read_seq[i:i + m])
        for j in rng.choice(m, size=max(1, m // 90), replace=False):      # substitutions stay inside an M block
            seg[j] = _DNA[(_DNA.index(seg[j]) + int(rng.integers(1, 4))) % 4]
        ref += seg; ops.append((m, "M")); i += m
        if i >= n:
            break
        kind = block % 3
        if kind == 0:                                                      # bases in the read that the reference lacks
            ins = int(min(n - i - 1, rng.integers(1, 5)))
            if ins > 0:
                ops.append((ins, "I")); i += ins
        elif kind == 1:                                                    # reference bases the read lacks
            d = int(rng.integers(1, 6))
            ref += [_DNA[c] for c in rng.integers(0, 4, d)]; ops.append((d, "D"))
        elif with_skip and not any(o == "N" for _, o in ops):
            s = int(rng.integers(20, 40))
            ref += [_DNA[c] for c in rng.integers(0, 4, s)]; ops.append((s, "N"))
        block += 1
    return "".join(ref), ops


def five_mer_model():
    """a 5-mer table with correlated neighbouring levels: the 6-mer table averaged over its last base"""
    m6 = synth.load_model("nucleotide")
    sd5 = m6.level_stdv.reshape(1024, 4).mean(1)
    return synth.PoreModel("derived.nucleotide.5mer", 5, "nucleotide", m6.level_mean.reshape(1024, 4).mean(1), sd5, np.log(sd5))


def build_cases(n_reads=4, n_events=1500, seed=77, model=None):
    model = model or synth.load_model("nucleotide")
    K = model.k
    rs = synth.gen_reads(n_reads, n_events, model, seed=seed, drift=True)
    cases = []
    for i in range(rs.n_reads):
        rng = np.random.default_rng(seed * 1000 + i)
        codes = rs.seq_codes[i]
        read_sequence = synth._CODE2DNA[codes].tobytes().decode()
        nk = len(read_sequence) - K + 1
        o, E = int(rs.reads[i]["event_off"]), int(rs.reads[i]["n_events"])
        which = rs.ev_kmer[i]
        first = np.searchsorted(which, np.arange(nk), side="left")
        last = np.searchsorted(which, np.arange(nk), side="right") - 1
        has = last >= first
        b2e_start = np.where(has, first, -1).astype(np.int32)
        b2e_stop = np.where(has, last, -1).astype(np.int32)
        reverse = i % 2 == 1
        oriented = EP.reverse_complement(read_sequence) if reverse else read_sequence
        ref_core, ops = _edit_script(oriented, rng, soft_clip=15 if i % 3 == 0 else 0, with_skip=(i % 4 == 2))
        left = "".join(_DNA[c] for c in rng.integers(0, 4, 40 + 7 * i))
        right = "".join(_DNA[c] for c in rng.integers(0, 4, 90))
        contig = list(left + ref_core + right)
        # soft-masked stretch and one ambiguity code: align_read_to_ref upper-cases and disambiguates
        a = len(left) + 200
        contig[a:a + 60] = [c.lower() for c in contig[a:a + 60]]
        contig[len(left) + 333] = "R"
        contig = "".join(contig)
        ref_pos = len(left)
        rlen = sum(n for n, op in ops if op in "MDN=X")
        fetched = contig[ref_pos:min(ref_pos + rlen + 1, len(contig))]      # faidx_fetch_seq(pos, bam_endpos): end inclusive
        stdv = rng.uniform(0.5, 3.0, E).astype(np.float32)
        duration = (rng.integers(3, 40, E) / 4000.0).astype(np.float32)
        rd = rs.reads[i]
        ear = EP.EARead(name=f"read_{i}", read_sequence=read_sequence, b2e_start=b2e_start, mean=rs.ev_mean[o:o + E],
                        stdv=stdv, duration=duration, start_time=rs.ev_start_time[o:o + E], shift=float(rd["shift"]),
                        scale=float(rd["scale"]), drift=float(rd["drift"]), var=float(rd["var"]), model=model, k=K)
        cases.append(dict(read=ear, b2e_stop=b2e_stop, contig=contig, contig_name="chr_test", ref_pos=ref_pos,
                          flag=EP.BAM_FREVERSE if reverse else 0, mapq=60 - i, cigar=EP.pack_cigar(ops), fetched=fetched,
                          read_idx=i, region=(-1, -1)))
    # one unmapped record and one restricted to a reference window
    if cases:
        c = dict(cases[0]); c["flag"] = EP.BAM_FUNMAP; c["read_idx"] = len(cases); cases.append(c)
        c = dict(cases[1 if len(cases) > 1 else 0]); c["region"] = (c["ref_pos"] + 300, c["ref_pos"] + 900); c["read_idx"] = len(cases); cases.append(c)
    return model, rs, cases


def read_slot(case, n_synth_reads):
    """index of the synthetic read a case is built on"""
    return int(case["read"].name.split("_")[1])


def port_align_fn(port_oracle, rs, model, slot, indel_bias=1.0):
    """profile_hmm_align through the plain-C oracle for read `slot` of rs."""
    K = model.k

    def fn(fwd, rc_seq, e0, e1, stride, rc):
        assert EP.reverse_complement(fwd) == rc_seq
        codes = synth.encode(fwd, "nucleotide")
        ranks = (synth.dna_rc_kmer_ranks(codes, K) if rc else synth.kmer_ranks_from_codes(codes, K, 4)).astype(np.uint32)
        jb = np.zeros(1, synth.HMM_JOB_DT)
        jb[0] = (0, slot, 0, e0, e1, ranks.shape[0], stride, int(rc), 0, 0)
        st, status = port_oracle.hmm_align(rs.reads, rs.ev_mean, rs.ev_start_time, [model], ranks, jb[0], indel_bias=indel_bias)
        return [(int(s["event_idx"]), int(s["kmer_idx"]), s["state"].decode()) for s in st]
    return fn


def raw_samples(slot):
    """stand-in for the trimmed raw samples SRF_LOAD_RAW_SAMPLES keeps: enough of them to cover every event's time span"""
    return np.random.default_rng(900 + slot).normal(90.0, 12.0, 420_000).astype(np.float32)


def load_batch(host, cases, samples_of=raw_samples):
    """clear the mirror, register the model and reads, give each case's read its eventalign data and its samples (samples_of(slot), at
    4 kHz; none where that is None), and queue every case in a new EventAligner batch"""
    model, rs, cs = cases
    host.nphh_clear()
    mh = hm.register_model(host, model)
    rh = hm.register_reads(host, rs, mh)
    host.nphh_ea_begin()
    for c in cs:
        slot, r = read_slot(c, rs.n_reads), c["read"]
        a, b = np.ascontiguousarray(r.b2e_start, np.int32), np.ascontiguousarray(c["b2e_stop"], np.int32)
        assert host.nphh_read_set_eventalign(rh[slot], r.name.encode(), r.read_sequence.encode(), hm.p(a), hm.p(b), C.c_size_t(a.shape[0]),
                                             hm.p(np.ascontiguousarray(r.stdv)), hm.p(np.ascontiguousarray(r.duration))) == 0
        smp = samples_of(slot)
        if smp is not None:
            assert host.nphh_read_set_samples(rh[slot], hm.p(smp), C.c_size_t(smp.shape[0]), C.c_double(4000.0)) == 0
        idx = host.nphh_ea_add_read(rh[slot], c["contig_name"].encode(), c["ref_pos"], c["flag"], c["mapq"], hm.p(c["cigar"]),
                                    int(c["cigar"].shape[0]), c["fetched"].encode(), c["read_idx"], c["region"][0], c["region"][1])
        assert idx == c["read_idx"], host.nphh_last_error()


def drive_rounds(host, cs, rs, model, port_oracle):
    """pull every round's jobs out of the C++ cursors and feed back the plain-C Viterbi's paths"""
    jobs = np.zeros(max(len(cs), 1), synth.HMM_JOB_DT)
    ranks = np.zeros(len(cs) * 400 + 400, np.uint32)
    n_ranks = C.c_uint64()
    rounds = 0
    while True:
        n = host.nphh_ea_next_round(hm.p(jobs), C.c_size_t(jobs.shape[0]), hm.p(ranks), C.c_size_t(ranks.shape[0]), C.byref(n_ranks))
        assert n >= 0, host.nphh_last_error()
        if n == 0:
            return rounds
        paths, off = [], [0]
        for j in range(n):
            jb = jobs[j].copy()
            jb["read"] = read_slot(cs[int(jb["read"])], rs.n_reads)
            st, _ = port_oracle.hmm_align(rs.reads, rs.ev_mean, rs.ev_start_time, [model], ranks, jb)
            paths.append(st); off.append(off[-1] + st.shape[0])
        flat = np.concatenate(paths) if off[-1] else np.zeros(0, synth.ALIGN_STATE_DT)
        assert host.nphh_ea_consume(C.c_size_t(n), hm.p(np.array(off, np.uint64)), hm.p(flat)) == 0, host.nphh_last_error()
        rounds += 1


def scorereads(host, cases, mode):
    """ScoreReads over the cases' event alignments (nphh_scorereads, EPS events per segment; mode 0 builds the jobs only, 1 scores
    them on the device): (jobs, ranks, per-read (score, events, segments))"""
    model, rs, cs = cases
    n = len(cs)
    reads = np.array([read_slot(c, rs.n_reads) for c in cs], np.int32)      # g_reads handles == slots after load_batch
    refs = (C.c_char_p * n)(*[c["fetched"].encode() for c in cs])
    offs = np.array([c["ref_pos"] for c in cs], np.int32)
    jobs = np.zeros(256, synth.HMM_JOB_DT); ranks = np.zeros(1 << 18, np.uint32); nr = C.c_uint64(); sc = np.zeros((n, 3))
    p = hm.p
    k = host.nphh_scorereads(n, p(reads), refs, p(offs), EPS, mode, p(jobs), C.c_size_t(jobs.shape[0]), p(ranks), C.c_size_t(ranks.shape[0]),
                             C.byref(nr), p(sc))
    assert k >= 0, host.nphh_last_error()
    return jobs[:k].copy(), ranks[:nr.value].copy(), sc
