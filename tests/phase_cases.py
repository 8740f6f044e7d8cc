"""phase-reads test cases and the three ways to run them — test infrastructure.

A case is a read of tests/meth_cases.make_case (CIGAR with insertions, deletions and soft clips, IUPAC and lower-case contig
bases, both strands) plus a sorted variant list planted on its contig.  Its SAM line comes from
  ref_line     the compiled reference's own phase_single_read (oracle/_ref/libnpref_phase.so, oracle/phase_reads_harness.cpp)
  restated     tests/phase_restatement.py with oracle forward scores
  mirror_sam   the C++ host mirror nph::PhaseReads through the nphh_phase_reads shim (the device call)."""
import bisect
import ctypes as C
import os

import numpy as np

from nanopolish_b200 import synth
from tests import host_mirror as hm
from tests import meth_cases as mc
from tests import phase_restatement as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PHASE = os.path.join(ROOT, "oracle", "_ref", "libnpref_phase.so")
CONTIG = "chr1"
_NT16 = "=ACMGRSVTWYHKDBN"


def cases(rs, seed=7, mapq=60):
    """per read: the make_case dict with 'upper' (the fetched reference through toupper), 'pairs', 'rc', 'mapq' and a variant list"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(rs.n_reads):
        c = mc.make_case(i, rs, rng)
        end = c["ref_pos"] + c["ref_len"]
        c["upper"] = c["contig"][c["ref_pos"]:end + 1].upper()
        c["pairs"], c["rc"] = mc.event_alignment_record(c)
        c["mapq"] = mapq
        out.append(c)
    return out


def plant(case, rng, step=(30, 400)):
    """sorted variants (pos, ref, alt) on the case's span: SNPs on the reference base, REF mismatches, lower-case REFs, non-SNPs,
    two variants at one position, a tie (alt == ref), one variant past the record (so lower_bound is never the end)"""
    up, pos0 = case["upper"], case["ref_pos"]
    var = []
    p = int(rng.integers(0, step[1]))
    while p < len(up):
        b = up[p]
        alt = "ACGT"[(("ACGT".find(b) if b in "ACGT" else 0) + int(rng.integers(1, 4))) % 4]
        kind = rng.random()
        if kind < 0.07:
            var.append((pos0 + p, alt, b))                            # REF mismatch
        elif kind < 0.12:
            var.append((pos0 + p, b.lower(), alt))                    # lower-case REF
        elif kind < 0.17:
            var.append((pos0 + p, b + "A", alt))                      # not a SNP
        elif kind < 0.22:
            var += [(pos0 + p, b, alt), (pos0 + p, b, "ACGT"[("ACGT".find(alt) + 1) % 4])]   # the later one wins
        elif kind < 0.26:
            var.append((pos0 + p, b, b))                              # tie
        else:
            var.append((pos0 + p, b, alt))
        p += int(rng.integers(step[0], step[1] + 1))
    var.append((pos0 + len(up) + 5000, "A", "C"))
    return var


def restated(port_oracle, rs, model, i, case, var):
    """the SAM line phase_single_read writes for read i (None: no record), from the restatement and oracle scores"""
    pos = [v[0] for v in var]
    lo = bisect.bisect_left(pos, case["ref_pos"])
    if lo == len(var):
        return None
    hi = max(lo, bisect.bisect_right(pos, case["ref_pos"] + len(case["upper"]) - 1))
    up = case["upper"].encode()
    variants = np.array([(p, r[:1].encode(), a[:1].encode(), int(len(r) == 1 and len(a) == 1), 0) for p, r, a in var], synth.PHASE_VARIANT_DT)
    recs = np.zeros(1, synth.METH_RECORD_DT)
    pairs = np.array(case["pairs"], synth.PAIR_DT) if case["pairs"] else np.zeros(0, synth.PAIR_DT)
    recs[0] = (0, 0, i, 0, len(up), pairs.shape[0], case["ref_pos"], case["rc"], 0, (0, 0))
    sites, jobs, ranks, _ = pr.enumerate_batch(np.frombuffer(up, np.uint8), pairs, recs, variants, np.array([[lo, hi]], np.uint32), model.k)
    scores = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [model], ranks, jobs)[0] if jobs.shape[0] else []
    seq, qual = bytearray(up), bytearray([30] * len(up))
    for j, (_, v) in enumerate(sites):
        c, q = pr.quality(scores[2 * j], scores[2 * j + 1], variants[v]["ref_base"], variants[v]["alt_base"])
        o = int(variants[v]["ref_position"]) - case["ref_pos"]
        seq[o], qual[o] = c[0], q
    return sam_line(case["name"], case["flag"], CONTIG, case["ref_pos"], case["mapq"], bytes(seq), bytes(qual))


def nt16(c: int) -> str:
    ch = chr(c).upper()
    if "0" <= ch <= "3":
        return "ACGT"[ord(ch) - 48]
    return ch if ch in _NT16 else "N"


def sam_line(name, flag, contig, pos, mapq, seq: bytes, qual: bytes) -> str:
    return (f"{name}\t{flag}\t{contig}\t{pos + 1}\t{mapq}\t{len(seq)}M\t*\t0\t0\t" + "".join(nt16(c) for c in seq) + "\t" +
            "".join(chr(q + 33) for q in qual) + "\n")


class RefPhase:
    """phase_single_read of the compiled reference, one record per call"""

    def __init__(self):
        self.lib = L = C.CDLL(REF_PHASE)
        L.npref_phase_read.restype = C.c_longlong
        L.npref_model_builtin.restype = C.c_int
        self.mh = L.npref_model_builtin(b"r9.4_450bps", b"nucleotide", b"template", 6)
        L.npref_reads_clear()

    def register(self, rs, case_list):
        hs = []
        for i, r in enumerate(rs.reads):
            o, n = int(r["event_off"]), int(r["n_events"])
            m = np.ascontiguousarray(rs.ev_mean[o:o + n]); t = np.ascontiguousarray(rs.ev_start_time[o:o + n])
            h = self.lib.npref_read_create(C.c_uint32(n), hm.p(m), hm.p(t), C.c_double(r["shift"]), C.c_double(r["scale"]), C.c_double(r["drift"]),
                                           C.c_double(r["var"]), C.c_double(r["events_per_base"]), self.mh)
            c = case_list[i]
            a, b = np.ascontiguousarray(c["b2e_start"], np.int32), np.ascontiguousarray(c["b2e_stop"], np.int32)
            one = np.ones(n, np.float32)
            self.lib.npref_read_set_eventalign(h, c["name"].encode(), c["read_sequence"].encode(), hm.p(a), hm.p(b), C.c_size_t(a.shape[0]), hm.p(one), hm.p(one))
            hs.append(h)
        return hs

    def line(self, h, case, var, indel_bias=1.0):
        cg = np.ascontiguousarray(case["cigar"], np.uint32)
        vp = np.array([v[0] for v in var], np.int32)
        vr = (C.c_char_p * len(var))(*[v[1].encode() for v in var]); va = (C.c_char_p * len(var))(*[v[2].encode() for v in var])
        buf = C.create_string_buffer(1 << 20)
        n = self.lib.npref_phase_read(h, case["name"].encode(), CONTIG.encode(), case["contig"].encode(), case["ref_pos"], case["flag"], case["mapq"],
                                      hm.p(cg), cg.shape[0], len(var), hm.p(vp), vr, va, C.c_double(indel_bias), buf, C.c_size_t(1 << 20))
        assert n >= 0
        return buf.value.decode() if n else None


def mirror_sam(host, host_reads, case_list, var, indel_bias=1.0):
    """nph::PhaseReads over the cases (one contig stretch each, one variant list) -> the SAM text"""
    n = len(case_list)
    names = (C.c_char_p * n)(*[c["name"].encode() for c in case_list])
    refs = (C.c_char_p * n)(*[c["upper"].encode() for c in case_list])
    flags = np.array([c["flag"] for c in case_list], np.uint16); mapq = np.array([c["mapq"] for c in case_list], np.uint8)
    starts = np.array([c["ref_pos"] for c in case_list], np.int32)
    pl = [np.array(c["pairs"], np.int32).reshape(-1, 2) for c in case_list]
    pairs = np.ascontiguousarray(np.concatenate(pl) if pl else np.zeros((0, 2), np.int32))
    off = np.zeros(n + 1, np.uint64); off[1:] = np.cumsum([p.shape[0] for p in pl])
    vp = np.array([v[0] for v in var], np.int32)
    vr = (C.c_char_p * len(var))(*[v[1].encode() for v in var]); va = (C.c_char_p * len(var))(*[v[2].encode() for v in var])
    rh = np.array(host_reads, np.int32)
    cap = 1 << 26
    buf = C.create_string_buffer(cap)
    got = host.nphh_phase_reads(n, hm.p(rh), names, hm.p(flags), hm.p(mapq), hm.p(starts), refs, hm.p(pairs), hm.p(off), CONTIG.encode(), len(var), hm.p(vp), vr, va,
                                C.c_double(indel_bias), buf, C.c_size_t(cap))
    assert got >= 0, host.nphh_last_error()
    return buf.value.decode()
