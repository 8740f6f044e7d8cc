"""get_variants_in_region test cases — test infrastructure.

A case is a region (its start, its reference), base-space records (bases as stored in the BAM, strand, aligned_bases), the
bounds [start, stop] and the filter (min_frequency, min_depth).  Records are written as operation lists over the region's reference
(rec()), or drawn from a seeded truth with basecall errors (synth.basecall_of).  Each case states the edge it was built to reach
and `claims(case, distinct)` checks it on the restatement's answer.  Cases with `before_start` records (aligned entirely before
start, where the reference dereferences end()) are never sent to the compiled reference."""
import hashlib

import numpy as np

from nanopolish_b200 import synth
from tests import candidate_restatement as cr

CONTIG = "ctg1"
F02 = float(np.float32(0.2))            # the reference's default -m: the float literal 0.2f widened to double


def _other(b: str) -> str:
    return "ACGT"[("ACGT".index(b) + 1) % 4] if b in "ACGT" else "A"


def rec(ref: str, region_start: int, pos: int, ops, rc=0):
    """(bases, aligned, rc) of a record starting at reference position pos: ops ('M', n) copy n reference bases, ('X', n) n mismatches,
    ('B', s) bases s aligned to the next len(s) reference bases, ('I', s) an insertion, ('D', n) a deletion, ('S', s) a soft clip"""
    bases, aligned, p = [], [], pos
    for op, a in ops:
        if op in "MX":
            for _ in range(a):
                b = ref[p - region_start]
                aligned.append((p, len(bases)))
                bases.append(b if op == "M" else _other(b))
                p += 1
        elif op == "B":
            for ch in a:
                aligned.append((p, len(bases)))
                bases.append(ch)
                p += 1
        elif op in "IS":
            bases += list(a)
        elif op == "D":
            p += a
    return "".join(bases).encode(), np.array(aligned, np.int64).reshape(-1, 2), rc


def _reference(n, seed, alphabet="ACGT"):
    rng = np.random.default_rng(seed)
    return "".join(rng.choice(list(alphabet), n))


def _case(name, region_start, ref, records, start, stop, min_frequency=F02, min_depth=1, before_start=False, claim=None):
    return dict(name=name, region_start=region_start, region_ref=ref, bases=[r[0] for r in records], aligned=[r[1] for r in records],
                rc=[r[2] for r in records], start=start, stop=stop, min_frequency=min_frequency, min_depth=min_depth, before_start=before_start,
                claim=claim)


def _random_reads(ref, region_start, n_reads, read_len, seed, p_sub, p_ins, p_del, max_clip=0):
    rng = np.random.default_rng(seed)
    out = []
    for r in range(n_reads):
        t0 = int(rng.integers(0, len(ref) - read_len))
        clip = (int(rng.integers(0, max_clip + 1)), int(rng.integers(0, max_clip + 1))) if max_clip else (0, 0)
        b, a = synth.basecall_of(ref, t0, read_len, rng, p_sub, p_ins, p_del, clip)
        a[:, 0] += region_start
        out.append((b, a, r % 2))
    return out


def _with_truth(ref, n_var, seed):
    """ref with n_var substitutions: the truth the reads are drawn from"""
    rng = np.random.default_rng(seed)
    t = list(ref)
    for p in rng.choice(np.arange(20, len(ref) - 20), n_var, replace=False):
        t[int(p)] = _other(t[int(p)])
    return "".join(t)


def build(name):
    RS = 5000
    if name == "substitutions":
        ref = _reference(600, 1)
        recs = _random_reads(_with_truth(ref, 12, 2), RS, 40, 150, 3, 0.02, 0.0, 0.0)
        return _case(name, RS, ref, recs, RS + 20, RS + 580, claim=lambda d: all(len(r) == 1 and len(a) == 1 for _, r, a in d))
    if name == "indels":
        ref = _reference(500, 4)
        R = lambda pos, ops, rc=0: rec(ref, RS, pos, ops, rc)
        recs = [R(RS + 10, [("M", 50), ("I", "A"), ("M", 30), ("I", "GTC"), ("M", 40), ("D", 1), ("M", 30), ("D", 4), ("M", 50)]) for _ in range(3)]
        recs += _random_reads(ref, RS, 20, 200, 5, 0.0, 0.02, 0.02)
        return _case(name, RS, ref, recs, RS + 5, RS + 480,
                     claim=lambda d: {(len(r), len(a)) for _, r, a in d} >= {(1, 2), (1, 4), (2, 1), (5, 1)})
    if name == "mismatch_gap":
        ref = _reference(300, 6)
        R = lambda pos, ops: rec(ref, RS, pos, ops)
        recs = [R(RS + 10, [("M", 40), ("X", 1), ("I", "TT"), ("M", 40)]),                  # a mismatch followed by a gap
                R(RS + 10, [("M", 60), ("I", "G"), ("X", 3), ("M", 40)]),                   # a gap, then mismatching pairs next skips
                R(RS + 10, [("M", 80), ("D", 2), ("X", 2), ("M", 30)])]
        return _case(name, RS, ref, recs, RS, RS + 290,
                     claim=lambda d: any(p == RS + 50 and len(r) == 1 and len(a) == 3 for p, r, a in d)
                     and any(p == RS + 69 and len(r) == 4 and len(a) == 5 for p, r, a in d))
    if name == "clips_strands_symbols":
        ref = list(_reference(300, 7))
        ref[100] = "N"
        ref = "".join(ref)
        R = lambda pos, ops, rc=0: rec(ref, RS, pos, ops, rc)
        recs = [R(RS + 20, [("S", "ACGTACG"), ("M", 60), ("X", 1), ("M", 60), ("S", "TTTT")], 1),
                R(RS + 30, [("M", 40), ("B", "="), ("M", 60)], 0),                           # '=' compares unequal to every base
                R(RS + 50, [("M", 30), ("B", "N"), ("M", 40)], 1),                           # N in a read
                R(RS + 90, [("M", 10), ("B", "N"), ("M", 30)], 0),                           # N read over N reference: equal
                R(RS + 90, [("M", 10), ("B", "A"), ("M", 30)], 1)]
        return _case(name, RS, ref, recs, RS + 10, RS + 280,
                     claim=lambda d: any(a == "=" for _, _, a in d) and any(a == "N" for _, _, a in d) and any(r == "N" for _, r, _ in d)
                     and not any(p == RS + 100 and a == "N" for p, _, a in d))
    if name in ("key_order_10k", "key_order_100k"):
        edge = 10_000 if name == "key_order_10k" else 100_000
        rs_ = edge - 150
        ref = _reference(300, 8)
        recs = []
        for k in range(6):
            recs.append(rec(ref, rs_, rs_ + 10 + k, [("M", 130 - k), ("X", 1), ("M", 9 + k), ("X", 1), ("M", 8), ("I", "CA"), ("M", 100)]))
        return _case(name, rs_, ref, recs, rs_ + 5, rs_ + 290, 0.0, 1,
                     claim=lambda d: any(p < edge for p, _, _ in d) and any(p >= edge for p, _, _ in d))
    if name == "sort_ties":
        # more than 16 variants, 2-4 alleles at several positions: std::sort's tie order, not key order, reaches the output
        ref = _reference(400, 9)
        recs = []
        for g, p in enumerate(range(40, 360, 16)):
            alts = ["X", "I", "D", "XX"][: 2 + g % 3]
            for a in alts:
                ops = {"X": [("X", 1)], "I": [("M", 1), ("I", "GG")], "D": [("M", 1), ("D", 2)], "XX": [("X", 2)]}[a]
                for _ in range(2):
                    recs.append(rec(ref, RS, RS + p - 20, [("M", 20)] + ops + [("M", 30)]))
        return _case(name, RS, ref, recs, RS + 5, RS + 390, 0.0, 1, claim=lambda d: len(d) > 16)
    if name == "stop_edges":
        ref = _reference(200, 10)
        stop = RS + 150
        R = lambda pos, ops: rec(ref, RS, pos, ops)
        recs = [R(RS + 100, [("M", 47), ("X", 1), ("M", 40)]),      # mismatch at stop - 3: next at stop - 2, kept
                R(RS + 100, [("M", 48), ("X", 1), ("M", 40)]),      # mismatch at stop - 2: next at stop - 1, dropped
                R(RS + 100, [("M", 49), ("X", 1), ("M", 40)]),      # mismatch at stop - 1: next is stop_iter, dropped
                R(RS + 100, [("M", 44), ("I", "T"), ("M", 40)])]    # a gap at stop - 6
        return _case(name, RS, ref, recs, RS + 10, stop,
                     claim=lambda d: any(p == stop - 3 for p, _, _ in d) and not any(p in (stop - 2, stop - 1) for p, _, _ in d))
    if name in ("bounds", "before_start"):
        ref = _reference(400, 11)
        start, stop = RS + 100, RS + 300
        R = lambda pos, ops: rec(ref, RS, pos, ops)
        recs = [R(RS + 50, [("M", 70), ("X", 1), ("M", 300 - 71)]),               # from before start to after stop
                R(RS + 310, [("M", 5), ("X", 1), ("M", 20)]),                       # entirely after stop
                (b"", np.zeros((0, 2), np.int64), 0),                             # empty
                R(RS + 200, [("X", 1)]),                                            # a single pair
                R(RS + 150, [("M", 20), ("X", 1), ("M", 100), ("X", 2), ("M", 100)])]
        if name == "before_start":
            recs.append(R(RS + 10, [("M", 40), ("X", 1), ("M", 20)]))               # entirely before start
        return _case(name, RS, ref, recs, start, stop, before_start=name == "before_start", claim=lambda d: len(d) >= 2)
    if name in ("freq_float", "freq_double", "depth_edge"):
        ref = _reference(200, 12)
        recs = [rec(ref, RS, RS + 20, [("M", 40), ("X", 1), ("M", 60)])]           # 1 of 5 reads: exactly 1/5
        recs += [rec(ref, RS, RS + 20, [("M", 101)]) for _ in range(4)]
        recs += [rec(ref, RS, RS + 80, [("M", 5), ("X", 1), ("M", 60)]) for _ in range(2)]
        mf = {"freq_float": F02, "freq_double": 0.2, "depth_edge": 0.1}[name]
        md = {"freq_float": 1, "freq_double": 5, "depth_edge": 6}[name]   # depth_edge: 7 at RS + 85 (kept), 5 at RS + 60 (dropped)
        return _case(name, RS, ref, recs, RS + 10, RS + 190, mf, md, claim=lambda d: d.get((RS + 60, ref[60], _other(ref[60])), (0, 0)) == (1, 5))
    if name == "deep_pile":
        ref = _reference(60, 13)
        recs = [rec(ref, RS, RS + 20, [("X", 1), ("M", 2)])] + [rec(ref, RS, RS + 20, [("M", 3)]) for _ in range(19_999)]
        return _case(name, RS, ref, recs, RS + 10, RS + 50, 0.0, 0, claim=lambda d: d[(RS + 20, ref[20], _other(ref[20]))] == (1, 20_000))
    if name == "region_50k":
        ref = _reference(50_000, 14)
        recs = _random_reads(_with_truth(ref, 40, 15), RS, 50 * 50_000 // 2_000, 2_000, 16, 0.04, 0.03, 0.03, max_clip=20)
        return _case(name, RS, ref, recs, RS + 40, RS + 49_960, claim=lambda d: len(d) > 1000)
    raise KeyError(name)


CASES = ["substitutions", "indels", "mismatch_gap", "clips_strands_symbols", "key_order_10k", "key_order_100k", "sort_ties", "stop_edges",
         "bounds", "before_start", "freq_float", "freq_double", "depth_edge", "deep_pile", "region_50k"]
REF_CASES = [n for n in CASES if n != "before_start"]


def fingerprint(c) -> str:
    h = hashlib.sha256()
    for b, a in zip(c["bases"], c["aligned"]):
        h.update(b + b"|" + np.ascontiguousarray(a, np.int64).tobytes())
    h.update(repr((c["region_start"], c["region_ref"], c["rc"], c["start"], c["stop"], c["min_frequency"], c["min_depth"])).encode())
    return h.hexdigest()


def flat_pairs(c):
    """aligned_bases of every record as one (n, 2) int32 array and per-record offsets (u8, n_records + 1)"""
    off = np.concatenate([[0], np.cumsum([a.shape[0] for a in c["aligned"]])]).astype(np.uint64)
    pp = np.concatenate([np.asarray(a, np.int32).reshape(-1, 2) for a in c["aligned"]] or [np.zeros((0, 2), np.int32)]).astype(np.int32)
    return np.ascontiguousarray(pp if pp.shape[0] else np.zeros((1, 2), np.int32)), off


def restated(c):
    return cr.distinct(c["region_ref"], c["region_start"], c["bases"], c["aligned"], c["start"], c["stop"])


def lines_of(kept):
    """the restated kept list as the harness's lines, INFO included (order: key order)"""
    out = []
    for p, r, a, cnt, d in kept:
        out.append(f"{p}\t{r}\t{a}\tBaseCalledReadsWithVariant={cnt};BaseCalledFraction={fmt(cnt / d)}")
    return out


def fmt(f: float) -> str:
    """std::stringstream << double with its defaults (%g, precision 6)"""
    return "%g" % f


def claims(c, dist):
    assert c["claim"] is None or c["claim"](dist), f"{c['name']}: the case does not reach the edge it was built for"


def parse(raw: bytes):
    return [tuple(int(f) if i == 0 else f for i, f in enumerate(l.split("\t"))) for l in raw.decode("latin-1").splitlines()]


# ---- the default-mode region call: call_variants_for_region + call_variants_main's VCF ----------------------------------------
# (name, ref_len, depth, read_bases, seed, n_true, ploidy, all_support, snps_only, candidates file, contig_length, end past the contig)
CALL_CASES = [
    ("vcf_50k_p1", 50_000, 50, 2_000, 21, 30, 1, 0, 0, False, 60_000, False),
    ("vcf_50k_p2", 50_000, 50, 2_000, 21, 30, 2, 0, 0, False, 60_000, False),
    ("vcf_all_support_snps", 3_000, 30, 600, 22, 8, 2, 1, 1, False, 8_000, True),
    ("vcf_candidates_file", 3_000, 30, 600, 23, 8, 1, 0, 1, True, 9_000, False),
]
CALL_FLANK, CALL_MIN_DISTANCE, CALL_MAX_HAPLOTYPES = 30, 10, 1000


def build_call(spec):
    """a gen_basecall_pileup region (about 10 % basecall error) and the window `variants` is asked for: start_base = region_start + BUFFER,
    end_base = last loaded base - BUFFER (or beyond the contig's end, clamped by the call)"""
    name, ref_len, depth, read_bases, seed, n_true, ploidy, all_support, snps, cand_file, contig_length, past_end = spec
    RS = 5000
    g = synth.gen_basecall_pileup(ref_len, depth, read_bases, synth.load_model("nucleotide"), seed=seed, region_start=RS, n_true_variants=n_true,
                                  p_sub=0.04, p_ins=0.03, p_del=0.03, max_clip=15)
    buffer = CALL_FLANK + 10
    if past_end:
        contig_length = RS + ref_len                                         # the loaded region ends at the contig's last base
    end_base = contig_length + 500 if past_end else RS + ref_len - 1 - buffer
    c = dict(name=name, rs=g["rs"], recs=g["recs"], pairs=g["pairs"], dur=np.ones(g["rs"].total_events, np.float32), draft=g["draft"],
             region_start=RS, region_end=RS + ref_len - 1, region_ref=g["draft"], bases=g["bases"], aligned=g["aligned"], rc=g["rc"],
             names=[f"read{r}" for r in range(g["rs"].reads.shape[0])], start_base=RS + buffer, end_base=end_base, contig_length=contig_length,
             ploidy=ploidy, all_support=all_support, snps_only=snps, min_frequency=F02, min_depth=20, candidates=None)
    if cand_file:
        truth = [i for i in range(ref_len) if g["draft"][i] != g["truth"][i]]
        rows = [(i, f"ctg\t{RS + i + 1}\t.\t{g['draft'][i]}\t{g['truth'][i]}\t12.5\tPASS\tX=1\tGT\t1") for i in truth]
        i = truth[len(truth) // 2] + 50                                      # a two-base substitution: dropped from the output by --snps
        rows.append((i, f"ctg\t{RS + i + 1}\t.\t{g['draft'][i:i + 2]}\t{_other(g['draft'][i])}{_other(g['draft'][i + 1])}\t3\tPASS\t.\tGT\t1"))
        # sorted: an unsorted list can join a later candidate to an earlier one into a window whose end precedes its start, where
        # the reference's substr_by_reference throws
        lines = ["##fileformat=VCFv4.2", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tsample"] + [l for _, l in sorted(rows)]
        lines.append(f"other\t{RS + 100}\t.\tA\tC\t1\tPASS\t.\tGT\t1")      # another contig
        lines.append(f"ctg\t{RS + 10}\t.\tA\tC\t1\tPASS\t.\tGT\t1")          # before the region's start
        lines.append(f"ctg\t{RS + ref_len}\t.\tA\tC\t1\tPASS\t.\tGT\t1")     # after its end
        c["candidates"] = "\n".join(lines) + "\n"
    return c


def call_fingerprint(c) -> str:
    h = hashlib.sha256(fingerprint(dict(c, start=c["start_base"], stop=c["end_base"])).encode())
    for a in (c["rs"].ev_mean, c["rs"].ev_start_time, c["recs"], c["pairs"]):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["names"], c["contig_length"], c["ploidy"], c["all_support"], c["snps_only"], c["candidates"])).encode())
    return h.hexdigest()


def call_args(c):
    """the arrays the host mirror's region call takes: event records (read index per record, rc, flat pairs, offsets) and base-space
    records"""
    recs, pairs = c["recs"], c["pairs"]
    pp, off = flat_pairs(c)
    return dict(rc=np.ascontiguousarray(recs["rc"], np.uint8),
                po=np.ascontiguousarray(recs["pair_off"], np.uint64), npair=np.ascontiguousarray(recs["n_pairs"], np.uint32),
                ep=np.ascontiguousarray(np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32)),
                seq_bases=c["bases"], seq_rc=np.array(c["rc"] or [0], np.uint8), sp=pp, soff=off,
                names=[c["names"][int(r)] for r in recs["read"]])


def _cstrs(xs):
    import ctypes as C
    return (C.c_char_p * max(len(xs), 1))(*[x if isinstance(x, bytes) else x.encode() for x in xs])

