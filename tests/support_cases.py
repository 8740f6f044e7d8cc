"""--calculate-all-support test cases and the ways to run them — test infrastructure.

A case is a seeded pile-up — synth.gen_hp_pileup through tests/hp_cases.py (a truth with homopolymer-length indels) or
synth.gen_pileup (a truth with substitutions), reads on both strands — plus a region over it, min_flanking_sequence, alignment_flags
and a variant list.  Its answers come from
  reference     the compiled reference's own annotate_variants_with_all_support (tests/ref_variants.py:
                oracle/_ref/libnpref_variants.so)
  restated      tests/support_restatement.py over the compiled reference's profile_hmm_score and add_logs (the same library)
  device        nph_all_support_batch
  mirror        nph::annotate_variants_with_all_support through the nphh_all_support shim (the device call)."""
import ctypes as C
import hashlib

import numpy as np

from nanopolish_b200 import synth
from tests import hp_cases as hc
from tests import hp_restatement as hr
from tests import support_restatement as sr

REGION_START = hc.REGION_START
CONTIG = hc.CONTIG
FLAGS = 3                               # HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, what `variants` passes

# (name, pile-up, trim, flank, alignment_flags, variants).  pile-up: ("snp", ref_len, depth, read_bases, seed, substitutions) or
# ("hp", ref_len, depth, read_bases, seed, homopolymer edits, hp_cases extras); trim (a, b): the region is the draft without its
# first a and last b bases.  variants:
#   truth   the truth's own edits: substitutions, or the homopolymer insertions and deletions anchored on the base before the run
#   edges   windows touching both region ends, each base as the reference base, multi-base deletions, an insertion, ref_seq of
#           flank + 1 and flank + 2 bases, a mismatch and a case-only mismatch, a duplicate, in an unsorted list
#   sparse  windows with no read and with exactly one read
#   dense   windows inside a record whose events advance 21 per base (the ratio test drops it)
CASES = [
    ("snp_truth", ("snp", 600, 12, 200, 3, 12), (0, 0), 10, FLAGS, "truth"),
    ("hp_truth", ("hp", 700, 12, 260, 3, 5, {}), (0, 0), 30, FLAGS, "truth"),
    ("edges_f7", ("hp", 500, 10, 200, 5, 4, {}), (6, 6), 7, 0, "edges"),
    ("edges_f30", ("snp", 700, 10, 260, 7, 6), (6, 9), 30, FLAGS, "edges"),
    ("sparse_f10", ("snp", 900, 2, 150, 9, 0), (0, 0), 10, FLAGS, "sparse"),
    ("dense_f10", ("hp", 800, 10, 400, 8, 4, dict(dense_at=(236, 32, 21))), (0, 0), 10, 0, "dense"),
    # windows of 341 bases: 336 k-mers, past the 320 columns of the widest single-strip forward class
    ("wide_f170", ("snp", 1400, 6, 600, 13, 10), (0, 0), 170, FLAGS, "truth"),
]


def _other(b: str) -> str:
    return "ACGT"[("ACGT".index(b.upper()) + 1) % 4]


def _pileup(kind, model):
    if kind[0] == "hp":
        _, ref_len, depth, read_bases, seed, n_err, ex = kind
        h = hc.build(("pileup", (ref_len, depth, read_bases, seed, n_err, 0), [], 30, 1.0, ex))
        truth = [(REGION_START + s - 1, h["draft"][s - 1:s + 1], h["draft"][s - 1]) if d < 0 else
                 (REGION_START + s - 1, h["draft"][s - 1], h["draft"][s - 1] + h["draft"][s]) for s, _, d in h["edits"]]
        return h["draft"], h["rs"], h["recs"], h["pairs"], h["dur"], h["deltas"], h["first"], truth
    _, ref_len, depth, read_bases, seed, n_sub = kind
    seqs = {}

    def keep(draft, truth):
        seqs["draft"], seqs["truth"] = draft, truth
        return draft, truth
    ref, rs, recs, pairs = synth.gen_pileup(ref_len, depth, read_bases, model, seed=seed, region_start=REGION_START, n_true_variants=n_sub,
                                            sequences=keep)
    draft = bytes(b"ACGT"[c] for c in ref).decode()
    truth = [(REGION_START + int(i), draft[i], "ACGT"[int(seqs["truth"][i])]) for i in np.flatnonzero(seqs["draft"] != seqs["truth"])]
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    return draft, rs, recs, pairs, np.ones(rs.total_events, np.float32), deltas, first, truth


def _edges(draft, rs_, re_, F):
    d = lambda p: draft[p - REGION_START]
    mid = (rs_ + re_) // 2
    v = [(rs_ + F, d(rs_ + F), _other(d(rs_ + F))), (re_ - F, d(re_ - F), _other(d(re_ - F)))]
    for b in "ACGT":                                                     # each base as the reference base
        p = next(p for p in range(rs_ + F + 3, re_ - F) if d(p) == b)
        v.append((p, b, _other(b)))
    ref = lambda p, n: draft[p - REGION_START:p - REGION_START + n]
    for p, r, a in [(mid - 9, ref(mid - 9, 4), d(mid - 9)),               # deletions of 3 and 2 bases
                    (mid - 3, ref(mid - 3, 3), d(mid - 3)),
                    (mid + 2, d(mid + 2), d(mid + 2) + "GT"),              # an insertion: its alt_seq is ignored
                    (mid + 6, ref(mid + 6, F + 1), d(mid + 6)),            # flank + 1 bases: applies
                    (mid + 8, ref(mid + 8, F + 2), d(mid + 8)),            # flank + 2 bases: substr clamps, never applies
                    (mid + 11, _other(d(mid + 11)), d(mid + 11)),          # a mismatch
                    (mid + 13, d(mid + 13).lower(), _other(d(mid + 13)))]: # the right base in lower case: bytes differ
        v.append((p, r, a))
    v.append(v[3])                                                       # a duplicate
    return v[len(v) // 2:] + v[:len(v) // 2]                             # unsorted


def _count(recs, pairs, p, F, max_ratio=20):
    return len(hr.event_sequences(recs, pairs, p - F, p + F, max_ratio))


def build(spec):
    name, kind, trim, F, flags, which = spec
    model = synth.load_model("nucleotide")
    draft, rs, recs, pairs, dur, deltas, first, truth = _pileup(kind, model)
    region_start, region_end = REGION_START + trim[0], REGION_START + len(draft) - 1 - trim[1]
    inside = lambda p: region_start <= p - F and p + F <= region_end
    if which == "truth":
        variants = [x for x in truth if inside(x[0])]
    elif which == "edges":
        variants = _edges(draft, region_start, region_end, F)
    elif which == "sparse":
        ps = range(region_start + F, region_end - F + 1)
        zero = [p for p in ps if _count(recs, pairs, p, F) == 0]
        one = [p for p in ps if _count(recs, pairs, p, F) == 1]
        pick = [zero[0], zero[-1], one[0], one[len(one) // 2]] + list(ps)[::97]
        variants = [(p, draft[p - REGION_START], _other(draft[p - REGION_START])) for p in pick]
    else:
        at, n, _ = kind[6]["dense_at"]
        ps = [REGION_START + at + F + 1, REGION_START + at + n // 2, REGION_START + at - F - 3]
        variants = [(p, draft[p - REGION_START], _other(draft[p - REGION_START])) for p in ps]
    params = np.zeros(1, synth.SUPPORT_PARAMS_DT)
    params[0] = (region_start, F, flags, 6)
    ref_seqs, varr = variant_array(variants)
    return dict(name=name, model=model, draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first,
                region_start=region_start, region_end=region_end, region_ref=draft[trim[0]:len(draft) - trim[1]], flank=F, flags=flags,
                variants=variants, params=params, ref_seqs=ref_seqs, varr=varr)


def random_case(seed: int, n_variants: int = 200, flank: int = 30, flags: int = FLAGS):
    """a homopolymer pile-up of 3 kb at depth 20 and n_variants random variants over its region: reference alleles of 0..4 draft bases,
    one in eight of them changed so that it does not apply, in random order with repeats"""
    model = synth.load_model("nucleotide")
    draft, rs, recs, pairs, dur, deltas, first, _ = _pileup(("hp", 3000, 20, 500, seed, 20, {}), model)
    rng = np.random.default_rng(seed)
    region_start, region_end = REGION_START, REGION_START + len(draft) - 1
    variants = []
    for p in rng.integers(region_start + flank, region_end - flank + 1, n_variants):
        r = draft[p - REGION_START:p - REGION_START + int(rng.integers(0, 5))]
        if rng.random() < 0.125:
            r = r[:-1] + _other(r[-1]) if r else "A"
        variants.append((int(p), r, "ACGT"[int(rng.integers(4))]))
    params = np.zeros(1, synth.SUPPORT_PARAMS_DT)
    params[0] = (region_start, flank, flags, 6)
    ref_seqs, varr = variant_array(variants)
    return dict(name=f"random{seed}", model=model, draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first,
                region_start=region_start, region_end=region_end, region_ref=draft, flank=flank, flags=flags, variants=variants, params=params,
                ref_seqs=ref_seqs, varr=varr)


def variant_array(variants):
    """(ref_seqs u1, SUPPORT_VARIANT_DT) of [(ref_position, ref_seq, alt_seq)]"""
    v = np.zeros(len(variants), synth.SUPPORT_VARIANT_DT)
    off = 0
    for i, (p, r, _) in enumerate(variants):
        v[i] = (p, len(r), off)
        off += len(r)
    return np.frombuffer("".join(r for _, r, _ in variants).encode() or b"\0", np.uint8).copy(), v


def fingerprint(c) -> str:
    h = hashlib.sha256()
    for a in (c["rs"].ev_mean, c["rs"].ev_start_time, c["recs"], c["pairs"], c["varr"], c["ref_seqs"]):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["draft"], c["variants"], c["flank"], c["flags"], c["region_start"], c["region_end"])).encode())
    return h.hexdigest()


def plan(c):
    """per variant (haplotypes, applied, event sequences [(record, e1, e2)]) of the restatement; hr.RefAbort where the reference
    asserts"""
    region = hr.Haplotype(c["region_start"], c["region_ref"])
    out = []
    for p, r, _ in c["variants"]:
        cs, ce, win = sr.window(region, p, c["flank"])
        haps, applied = sr.haplotypes(win, p, r)
        out.append((haps, applied, hr.event_sequences(c["recs"], c["pairs"], cs, ce)))
    return out


def restated(c, score_jobs, add_logs):
    """per variant (support f8[4], n_reads, applied, INFO).  score_jobs(jobs HMM_JOB_DT, seqs [bytes]) -> float32 scores"""
    pl = plan(c)
    recs = c["recs"]
    jobs, seqs = [], []
    for haps, _, ev in pl:
        for r, e1, e2 in ev:
            for h in haps:
                jobs.append((0, int(recs[r]["read"]), 0, e1, e2, len(h) - 5, -1 if recs[r]["rc"] else 1, int(recs[r]["rc"]), c["flags"], 0))
                seqs.append(h.encode())
    s = score_jobs(np.array(jobs, synth.HMM_JOB_DT), seqs) if jobs else np.zeros(0, np.float32)
    out, j = [], 0
    for haps, applied, ev in pl:
        scores = [s[j + 4 * i:j + 4 * i + 4] for i in range(len(ev))]
        j += 4 * len(ev)
        sup = sr.support(scores, add_logs)
        out.append((sup, len(ev), applied, sr.info(sup)))
    return out


def ref_restated(ref, c, hs, mh):
    """restated over the profile_hmm_score and add_logs of `ref` (a tests/ref_variants.py RefVariants holding the case's reads as
    registered: hs, mh)"""
    return restated(c, lambda jobs, seqs: ref.score_batch(hs, jobs, seqs, [mh])[0], ref.lib.npref_add_logs)


def device(eng, c, variants=None, params=None):
    rs = c["rs"]
    ref_seqs, varr = (c["ref_seqs"], c["varr"]) if variants is None else variant_array(variants)
    return eng.all_support_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(), c["deltas"],
                                 c["first"], c["recs"], c["params"] if params is None else params, ref_seqs, varr)


def _cstrs(xs):
    return (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])


def mirror(host, c, var_contig=CONTIG, variants=None):
    """nph::annotate_variants_with_all_support through the nphh_all_support shim: (status, [INFO per variant])"""
    from tests.test_host_mirror import _register, _register_reads
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    host.nphh_clear()
    rs = c["rs"]
    mh = _register(host, c["model"])
    hs = _register_reads(host, rs, mh)
    recs, pairs = c["recs"], c["pairs"]
    read = np.array([hs[int(x)] for x in recs["read"]], np.int32)
    rc = np.ascontiguousarray(recs["rc"], np.uint8)
    pp = np.ascontiguousarray(np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32))
    po = np.zeros(recs.shape[0] + 1, np.uint64)
    po[:-1] = recs["pair_off"]; po[-1] = pairs.shape[0]
    vs = c["variants"] if variants is None else variants
    vp = np.array([x[0] for x in vs] or [0], np.int32)
    out = C.create_string_buffer(1 << 20)
    host.nphh_all_support.restype = C.c_longlong
    n = host.nphh_all_support(CONTIG.encode(), c["region_start"], c["region_ref"].encode(), int(recs.shape[0]), p(read), p(rc), p(pp), p(po),
                              var_contig.encode(), len(vs), p(vp), _cstrs([x[1] for x in vs]), _cstrs([x[2] for x in vs]), c["flank"],
                              C.c_uint32(c["flags"]), C.c_double(1.0), out, C.c_size_t(1 << 20))
    if n < 0:
        return int(n), None
    return int(n), out.raw[:n].decode().split("\n")[:-1]
