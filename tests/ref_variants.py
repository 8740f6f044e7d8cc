"""The compiled reference's variant calling (oracle/_ref/libnpref_variants.so, oracle/variants_harness.cpp) — test infrastructure.

RefVariants is the RefOracle over that library: its own reads, profile_hmm_score / _align, and one method per entry point of the
harness, each taking a case of tests/hp_cases.py, screen_cases.py, support_cases.py, call_cases.py or candidate_cases.py."""
import ctypes as C
import os

import numpy as np

from oracle.oracle_py import RefOracle
from tests import call_cases as cc
from tests import candidate_cases as cand
from tests import hp_cases as hc

LIB = os.path.join(hc.ROOT, "oracle", "_ref", "libnpref_variants.so")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _cstrs(xs):
    return (C.c_char_p * max(1, len(xs)))(*[x if isinstance(x, bytes) else x.encode() for x in xs])


def _alleles(vs):
    """the harness's (positions, REF strings, ALT strings) of [(position, ref, alt)]"""
    return _p(np.array([v[0] for v in vs] or [0], np.int32)), _cstrs([v[1] for v in vs]), _cstrs([v[2] for v in vs])


class RefVariants(RefOracle):
    """RefOracle over oracle/_ref/libnpref_variants.so"""

    def __init__(self, path: str = LIB):
        super().__init__(path)
        L = self.lib
        for entry in ("npref_fix_homopolymers", "npref_screen_variants", "npref_expand_variants", "npref_call_haplotype", "npref_combinations",
                      "npref_all_support", "npref_variants_in_region", "npref_call_region"):
            getattr(L, entry).restype = C.c_longlong
        L.npref_fisher_exact.restype = C.c_double
        L.npref_fisher_exact.argtypes = [C.c_int] * 4

    @staticmethod
    def available(path: str = LIB) -> bool:
        return RefOracle.available(path)

    def register(self, c):
        self.clear_reads()
        rs = c["rs"]
        mh = self.builtin_model()
        hs = self.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, mh)
        for i, r in enumerate(rs.reads):
            o, n = int(r["event_off"]), int(r["n_events"])
            self.read_set_eventalign(hs[i], f"r{i}", "", np.zeros(0, np.int32), np.zeros(0, np.int32), np.ones(n, np.float32), c["dur"][o:o + n])
        return hs, mh

    def records(self, c, hs):
        """the case's event records as every entry point takes them: (n_records, read handles, rc, stride, pair offsets, pair counts,
        the (ref_pos, read_pos) pairs)"""
        recs, pairs = c["recs"], c["pairs"]
        rc = np.ascontiguousarray(recs["rc"], np.uint8)
        return (int(recs.shape[0]), _p(np.ascontiguousarray(hs[recs["read"]], np.int32)), _p(rc), _p(np.where(rc == 1, -1, 1).astype(np.int8)),
                _p(np.ascontiguousarray(recs["pair_off"], np.uint64)), _p(np.ascontiguousarray(recs["n_pairs"], np.uint32)),
                _p(np.ascontiguousarray(np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32))))

    def _text(self, entry: str, *args, cap: int = 1 << 22) -> bytes:
        out = C.create_string_buffer(cap)
        n = getattr(self.lib, entry)(*args, out, C.c_size_t(cap))
        assert n >= 0, n
        return out.raw[:n]

    def fixed(self, c, hs) -> str:
        """fix_homopolymers of an hp_cases case: the fixed sequence, then one line per variant it adds to the case's haplotype"""
        vs = [(hc.REGION_START + o, r, a) for o, r, a in c["variants"]]
        text = self._text("npref_fix_homopolymers", hc.CONTIG.encode(), c["region_start"], c["region_end"], c["region_ref"].encode(),
                          *self.records(c, hs), hc.REGION_START, c["draft"].encode(), len(vs), *_alleles(vs), c["min_flank"], cap=1 << 20)
        seq, *lines = text.decode().split("\n")
        return seq + "\n" + "".join(l + "\n" for l in lines[len(vs):] if l)

    def screened(self, c, hs):
        """screen_variants_by_score of a screen_cases case: one line per kept variant"""
        vs = c["candidates"]
        return self._text("npref_screen_variants", hc.CONTIG.encode(), c["region_start"], c["region_end"], c["region_ref"].encode(),
                          *self.records(c, hs), len(vs), *_alleles(vs), c["flank"], int(c["threshold"]), ",".join(c["types"]).encode(),
                          C.c_uint32(c["flags"])).decode().split("\n")[:-1]

    def expanded(self, region_start, region_ref, cands, min_flank):
        """expand_variants over a region without records: one line per output variant"""
        return self._text("npref_expand_variants", hc.CONTIG.encode(), region_start, region_start + len(region_ref) - 1, region_ref.encode(),
                          len(cands), *_alleles(cands), min_flank).decode().split("\n")[:-1]

    def infos(self, c, hs):
        """annotate_variants_with_all_support of a support_cases case: the INFO of every variant after the call"""
        vs = c["variants"]
        return self._text("npref_all_support", hc.CONTIG.encode(), c["region_start"], c["region_end"], c["region_ref"].encode(),
                          *self.records(c, hs), len(vs), *_alleles(vs), c["flank"], C.c_uint32(c["flags"]), cap=1 << 20).decode().split("\n")[:-1]

    def called(self, c, hs):
        """call_haplotype_from_candidates of a call_cases case: the derived sequence, then one line per variant of the derived haplotype"""
        n, rh, *rest = self.records(c, hs)
        vs = c["candidates"]
        return self._text("npref_call_haplotype", hc.CONTIG.encode(), c["region_start"], c["region_end"], c["region_ref"].encode(), n, rh,
                          _cstrs(cc.record_names(c)), *rest, len(vs), *_alleles(vs), cc.FLANK, cc.MIN_DISTANCE, c["max_haplotypes"],
                          c["ploidy"], c["genotype_only"], ",".join(c["types"]).encode(), c["all_support"],
                          C.c_uint32(cc.FLAGS)).decode().split("\n")[:-1]

    def fisher(self, n11, n12, n21, n22):
        return self.lib.npref_fisher_exact(n11, n12, n21, n22)

    def combinations(self, n, k, with_replacement):
        cap = 1 << 20
        out = np.zeros(cap, np.uint32)
        m = self.lib.npref_combinations(n, k, int(with_replacement), _p(out), C.c_size_t(cap))
        assert m >= 0
        return out[:m * k].reshape(m, k).tolist() if k else [[]] * m

    def variants_in_region(self, c):
        """AlignmentDB::get_variants_in_region of a candidate_cases case: one (ref_position, ref_seq, alt_seq, info) per variant, in
        the reference's order"""
        pp, off = cand.flat_pairs(c)
        return cand.parse(self._text("npref_variants_in_region", cand.CONTIG.encode(), c["region_start"], c["region_start"] + len(c["region_ref"]) - 1,
                                     c["region_ref"].encode(), len(c["bases"]), _cstrs(c["bases"]), _p(np.array(c["rc"] or [0], np.uint8)),
                                     _p(pp), _p(off), c["start"], c["stop"], C.c_double(c["min_frequency"]), c["min_depth"], cap=1 << 26))

    def call_region(self, c) -> bytes:
        """the default-mode region call of a candidate_cases.build_call case (npref_call_region): the VCF bytes"""
        hs, _ = self.register(c)
        n, rh, *rest = self.records(c, hs)
        pp, off = cand.flat_pairs(c)
        return self._text("npref_call_region", b"ctg", c["contig_length"], c["start_base"], c["end_base"], c["region_start"], c["region_end"],
                          c["region_ref"].encode(), n, rh, _cstrs(cc.record_names(c)), *rest, len(c["bases"]), _cstrs(c["bases"]),
                          _p(np.array(c["rc"] or [0], np.uint8)), _p(pp), _p(off), cand.CALL_FLANK, cand.CALL_MIN_DISTANCE,
                          cand.CALL_MAX_HAPLOTYPES, c["ploidy"], 0, b"", c["all_support"], c["snps_only"], C.c_double(c["min_frequency"]),
                          c["min_depth"], None if c["candidates"] is None else c["candidates"].encode(), cap=1 << 24)
