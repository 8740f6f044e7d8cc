"""SURVEY.md 8(f) row N2 — the variant-scoring callers as batch generators (nanopolish_b200/host/nph_variants.*):
Haplotype::apply_variant semantics, and score_variants_thresholded against an expectation composed from the
oracle's per-sequence scores + the reference's host arithmetic (score_set logsum, read-order early exit)."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import host_mirror as hm

host = hm.fixture()


def _apply(host, ref, pos0, variants):
    n = len(variants)
    pos = (C.c_size_t * n)(*[v[0] for v in variants])
    rs = (C.c_char_p * n)(*[v[1].encode() for v in variants])
    al = (C.c_char_p * n)(*[v[2].encode() for v in variants])
    out = C.create_string_buffer(len(ref) + sum(len(v[2]) for v in variants) + 8)
    rc = host.nphh_haplotype_apply(ref.encode(), C.c_size_t(pos0), n, pos, rs, al, out)
    return rc, out.value.decode()


def test_haplotype_apply_variant_semantics(host):
    ref = "ACGTACGTAC"      # reference positions 100..109
    assert _apply(host, ref, 100, [(103, "T", "G")]) == (10, "ACGGACGTAC")                 # substitution
    assert _apply(host, ref, 100, [(103, "TA", "T")]) == (9, "ACGTCGTAC")                  # deletion
    assert _apply(host, ref, 100, [(103, "T", "TGG")]) == (12, "ACGTGGACGTAC")             # insertion
    assert _apply(host, ref, 100, [(103, "A", "G")])[0] == -1                              # ref allele mismatch: refused
    assert _apply(host, ref, 100, [(99, "A", "G")])[0] == -1                               # outside the haplotype
    # a second variant at a reference base that was deleted by the first is refused, the first stays applied
    assert _apply(host, ref, 100, [(103, "TA", "T"), (104, "A", "C")]) == (-1, "ACGTCGTAC")
    # variants on either side of an insertion keep their reference coordinates
    assert _apply(host, ref, 100, [(103, "T", "TGG"), (105, "C", "T")]) == (12, "ACGTGGATGTAC")


def _expected_quality(port_oracle, rs, model_list, jobs_for, variants_seqs, base_seq, threshold, indel_bias, meth):
    """sum over reads in order of (score_set(variant) - score_set(base)) with the early exit, from oracle scores."""
    def score_set(seq, j):
        seqs = [(seq, "nucleotide", 0)]
        if meth:
            m = seq.replace("CG", "MG")
            if m != seq:
                seqs.append((m, "cpg", 1))
        sc = []
        for s, alpha, mid in seqs:
            ranks = synth.kmer_ranks_from_codes(synth.encode(s, alpha), 6, 4 if alpha == "nucleotide" else 5)
            jb = np.zeros(1, synth.HMM_JOB_DT)
            e0, e1 = jobs_for[j]
            jb[0] = (0, j, mid, e0, e1, ranks.shape[0], 1, 0, 0, 0)
            v, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model_list, ranks.astype(np.uint32), jb, indel_bias=indel_bias)
            sc.append(v[0])
        return float(np.float32(port_oracle.score_set_combine(np.array(sc, np.float32))))
    base = [score_set(base_seq, j) for j in range(rs.n_reads)]
    out = []
    for vs in variants_seqs:
        total = 0.0
        if vs is not None:
            for j in range(rs.n_reads):
                if abs(total) < threshold:
                    total += score_set(vs, j) - base[j]
        out.append(total)
    return out


def _variant_case():
    nuc, cpg = synth.load_model("nucleotide"), synth.load_model("cpg")
    rng = np.random.default_rng(11)
    codes = rng.integers(0, 4, 46, dtype=np.uint8)
    codes[20:22] = [1, 2]                                     # a CpG inside the window
    ref = synth._CODE2DNA[codes].tobytes().decode()
    rs = synth.gen_reads_from_sequence(codes, 14, nuc, seed=500)
    # candidates: substitutions, a deletion, an insertion, and one that does not apply
    cands = [(1000 + 10, ref[10], "ACGT".replace(ref[10], "")[0]), (1000 + 20, "C", "T"), (1000 + 30, ref[30:32], ref[30]),
             (1000 + 15, ref[15], ref[15] + "GA"), (1000 + 25, "ACGT".replace(ref[25], "")[1], "A")]
    return nuc, cpg, codes, ref, rs, cands


@pytest.mark.parametrize("meth,threshold", [(False, 100), (True, 30)])
def test_expectation_is_the_compiled_reference(host, port_oracle, ref_oracle, meth, threshold):
    """The expectation the GPU test below holds the C++ batcher to — composed from oracle scores, the score-set logsum and
    the read-order early exit — equals the COMPILED reference's score_variant_thresholded (src/common/nanopolish_variant.cpp:
    765-799, one OpenMP thread) for every candidate, including the one that does not apply."""
    nuc, cpg, codes, ref, rs, cands = _variant_case()
    windows = [(0, int(rs.reads[j]["n_events"]) - 1) for j in range(rs.n_reads)]
    vseqs = []
    for p_, r_, a_ in cands:
        rc, s_ = _apply(host, ref, 1000, [(p_, r_, a_)])
        vseqs.append(s_ if rc >= 0 else None)
    want = _expected_quality(port_oracle, rs, [nuc, cpg], windows, vseqs, ref, threshold, 0.8, meth)
    ref_oracle.clear_reads()
    rh = ref_oracle.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, ref_oracle.builtin_model("nucleotide"))
    got = ref_oracle.score_variants_thresholded(rh, windows, np.zeros(rs.n_reads, np.uint8), ref, 1000, cands, 0, threshold, meth, indel_bias=0.8)
    ref_oracle.clear_reads()
    assert list(got) == want, (list(got), want)
    assert got[-1] == 0.0 and (got[:-1] < 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("meth,threshold", [(False, 100), (True, 30)])
def test_score_variants_thresholded(host, port_oracle, meth, threshold):
    nuc, cpg, codes, ref, rs, cands = _variant_case()
    mh, ch = hm.register_model(host, nuc), hm.register_model(host, cpg)
    rh = hm.register_reads(host, rs, mh)
    for r in rh:
        host.nphh_read_add_model(r, b"cpg", ch)
    windows = [(0, int(rs.reads[j]["n_events"]) - 1) for j in range(rs.n_reads)]
    vseqs = []
    for p, r_, a_ in cands:
        rc, s = _apply(host, ref, 1000, [(p, r_, a_)])
        vseqs.append(s if rc >= 0 else None)
    assert vseqs[-1] is None and all(v is not None for v in vseqs[:-1])
    n = len(cands)
    q = np.zeros(n)
    p = hm.p
    reads = np.array(rh, np.int32)
    es = np.array([w[0] for w in windows], np.uint32); ee = np.array([w[1] for w in windows], np.uint32)
    rcs = np.zeros(rs.n_reads, np.uint8)
    mt = (C.c_char_p * 1)(b"cpg")
    rc = host.nphh_score_variants_thresholded(rs.n_reads, p(reads), p(es), p(ee), p(rcs), mh, ref.encode(), C.c_size_t(1000), n,
                                              (C.c_size_t * n)(*[c[0] for c in cands]), (C.c_char_p * n)(*[c[1].encode() for c in cands]),
                                              (C.c_char_p * n)(*[c[2].encode() for c in cands]), 0, threshold, 1 if meth else 0, mt,
                                              C.c_double(0.8), p(q))
    assert rc == 0, host.nphh_last_error()
    want = _expected_quality(port_oracle, rs, [nuc, cpg], windows, vseqs, ref, threshold, 0.8, meth)
    assert q[-1] == 0.0
    assert list(q) == want, (list(q), want)
    # the true sequence wins: every applicable candidate lowers the likelihood
    assert (q[:-1] < 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("meth,max_haplotypes", [(False, 1000), (True, 8)])
def test_score_variant_group_equals_compiled_reference(host, ref_oracle, meth, max_haplotypes):
    """nph::score_variant_group (haplotype enumeration + score_haplotypes: ONE launch for every (read, haplotype, alphabet
    alternative)) against the compiled reference's score_variant_group (src/common/nanopolish_variant.cpp:182-262): the same set
    of variant combinations survives (max_r from max_haplotypes, incompatible combinations dropped) and every
    (combination, read) score is the same double."""
    nuc, cpg, codes, ref, rs, cands = _variant_case()
    cands = cands[:4] + [(1000 + 20, "C", "A")]                 # the last one collides with candidate 1 (same reference base)
    mh, ch = hm.register_model(host, nuc), hm.register_model(host, cpg)
    rh = hm.register_reads(host, rs, mh)
    for r in rh:
        host.nphh_read_add_model(r, b"cpg", ch)
    windows = [(0, int(rs.reads[j]["n_events"]) - 1) for j in range(rs.n_reads)]
    ref_oracle.clear_reads()
    rrh = ref_oracle.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, ref_oracle.builtin_model("nucleotide"))
    want = ref_oracle.score_variant_group(rrh, windows, np.zeros(rs.n_reads, np.uint8), ref, 1000, cands, max_haplotypes, 3, meth, indel_bias=0.9)
    ref_oracle.clear_reads()
    n = len(cands)
    p = hm.p
    reads = np.array(rh, np.int32)
    es = np.array([w[0] for w in windows], np.uint32); ee = np.array([w[1] for w in windows], np.uint32)
    rcs = np.zeros(rs.n_reads, np.uint8)
    mt = (C.c_char_p * 1)(b"cpg")
    combos = np.zeros(4096, np.uint32); scores = np.zeros(4096 * rs.n_reads)
    k = host.nphh_score_variant_group(rs.n_reads, p(reads), p(es), p(ee), p(rcs), mh, ref.encode(), C.c_size_t(1000), n,
                                      (C.c_size_t * n)(*[c[0] for c in cands]), (C.c_char_p * n)(*[c[1].encode() for c in cands]),
                                      (C.c_char_p * n)(*[c[2].encode() for c in cands]), max_haplotypes, 3, 1 if meth else 0, mt,
                                      C.c_double(0.9), p(combos), p(scores), C.c_size_t(4096))
    assert k >= 0, host.nphh_last_error()
    got = {frozenset(i for i in range(n) if combos[c] >> i & 1): scores[c * rs.n_reads:(c + 1) * rs.n_reads] for c in range(k)}
    assert set(got) == set(want) and frozenset() in got
    assert frozenset({1, 4}) not in got                          # both rewrite reference base 1020: the combination does not apply
    if max_haplotypes == 8:
        assert max(len(c) for c in got) == 1                     # 1 + 5 < 8 but 1 + 5 + 10 is not: single variants only
    else:
        assert max(len(c) for c in got) >= 4
    for c in want:
        assert np.array_equal(got[c], want[c]), sorted(c)
