"""screen_variants_by_score / expand_variants test cases and the ways to run them — test infrastructure.

A case is a seeded pile-up — synth.gen_pileup (a truth with substitutions), synth.gen_hp_pileup through tests/hp_cases.py (a truth
with homopolymer-length indels) or synth.gen_pileup_methylated (planted recognition sites), reads on both strands — plus a region
over it, opt::screen_flanking_sequence, alignment_flags, opt::screen_score_threshold, opt::methylation_types and a candidate list.
Its answers come from
  reference     the compiled reference's own screen_variants_by_score (tests/ref_variants.py: oracle/_ref/libnpref_variants.so)
  restated      tests/screen_restatement.py over the compiled reference's profile_hmm_score (the same library)
  device        nph_screen_variants_batch
  mirror        nph::screen_variants_by_score through the nphh_screen_variants shim (the device call)."""
import ctypes as C
import hashlib

import numpy as np

from nanopolish_b200 import synth
from tests import hp_cases as hc
from tests import screen_restatement as scr
from tests import support_cases as suc
from tests import var_meth_restatement as vmr

REGION_START = hc.REGION_START
CONTIG = hc.CONTIG
FLAGS = 3                               # HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, what `variants` passes
ALL_TYPES = ("cpg", "dam", "dcm")       # the device suite's model ids 1, 2, 3

# (name, pile-up, trim, flank, alignment_flags, score_threshold, methylation types, candidates).  pile-up: as tests/support_cases.py,
# or ("meth", ref_len, depth, read_bases, seed); trim (a, b): the region is the draft without its first a and last b bases.  candidates:
#   truth   the truth's own edits (substitutions, or homopolymer insertions and deletions) and a wrong substitution beside each
#   edges   windows exactly at and one base past both region ends; an exact and a case-only ref_seq mismatch; multi-base deletions
#           and insertions; an empty ref_seq, an empty alt_seq and both; several candidates and ref lengths at one position;
#           duplicates, in an unsorted list
#   sparse  windows with no read and with exactly one read
#   dense   windows inside a record whose events advance 21 per base (the ratio test drops it)
#   meth    every substitution and insertion of every seventh position, and every one that makes or breaks a site
CASES = [
    ("snp_truth", ("snp", 600, 12, 200, 3, 12), (0, 0), 10, FLAGS, 100, (), "truth"),
    ("hp_truth", ("hp", 700, 12, 260, 3, 5, {}), (0, 0), 10, FLAGS, 100, (), "truth"),
    ("snp_truth_t0", ("snp", 600, 12, 200, 3, 12), (0, 0), 10, FLAGS, 0, (), "truth"),
    ("edges_f3", ("hp", 500, 10, 200, 5, 4, {}), (6, 6), 3, 0, 25, (), "edges"),
    ("edges_f30", ("snp", 700, 10, 260, 7, 6), (6, 9), 30, FLAGS, 10 ** 9, (), "edges"),
    ("sparse_t1", ("snp", 900, 2, 150, 9, 0), (0, 0), 10, FLAGS, 1, (), "sparse"),
    ("dense_f10", ("hp", 800, 10, 400, 8, 4, dict(dense_at=(236, 32, 21))), (0, 0), 10, 0, 100, (), "dense"),
    ("meth_cpg", ("meth", 130, 10, 100, 72), (0, 0), 10, FLAGS, 100, ("cpg",), "meth"),
    ("meth_dam_dcm", ("meth", 130, 10, 100, 73), (0, 0), 10, 0, 100, ("dam", "dcm"), "meth"),
]

# (name, the CASES entry whose pile-up it uses, min_flanking_sequence, candidates): expand_variants of the truth (round 1), and of
# indels whose extended deletion ends exactly min_flank + 1 and min_flank bases before the region's end (kept, refused)
EXPAND = [
    ("expand_hp", "hp_truth", 30),
    ("expand_edges", "edges_f30", 30),
]


def _other(b: str) -> str:
    return "ACGT"[("ACGT".index(b.upper()) + 1) % 4]


def _pileup(kind, types):
    if kind[0] != "meth":
        return suc._pileup(kind, synth.load_model("nucleotide"))
    from tests.test_variants_methylation_oracle import methylated_pileup
    _, ref_len, depth, read_bases, seed = kind
    _, _, _, ref_chars, rs, recs, pairs = methylated_pileup(list(types), ref_len, depth, read_bases, seed)
    draft = ref_chars.tobytes().decode()
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    return draft, rs, recs, pairs, np.ones(rs.total_events, np.float32), deltas, first, []


def _edges(draft, lo, hi, F):
    d = lambda p: draft[p - REGION_START]
    ref = lambda p, n: draft[p - REGION_START:p - REGION_START + n]
    mid = (lo + hi) // 2
    v = [(lo + F, d(lo + F), _other(d(lo + F))),                         # calling_start == region_start
         (lo + F - 1, d(lo + F - 1), _other(d(lo + F - 1))),             # one base past it
         (hi - F - 1, d(hi - F - 1), _other(d(hi - F - 1))),             # calling_end == region_end
         (hi - F, d(hi - F), _other(d(hi - F))),                         # one base past it
         (hi - F - 3, ref(hi - F - 3, 3), d(hi - F - 3)),                # a deletion whose window ends at region_end
         (mid - 9, ref(mid - 9, 4), d(mid - 9)),                         # deletions of 3 and 2 bases
         (mid - 5, ref(mid - 5, 3), d(mid - 5)),
         (mid + 2, d(mid + 2), d(mid + 2) + "GT"),                       # insertions of 2 and 3 bases
         (mid + 3, d(mid + 3), d(mid + 3) + "TTA"),
         (mid + 4, ref(mid + 4, 2), ""),                                 # an empty alt_seq
         (mid + 5, "", "A"),                                             # an empty ref_seq (an insertion at the position)
         (mid + 6, "", ""),                                              # both empty
         (mid + 11, _other(d(mid + 11)), d(mid + 11)),                   # a mismatch
         (mid + 13, d(mid + 13).lower(), _other(d(mid + 13)))]           # the right base in lower case: bytes differ
    b = d(mid)
    v += [(mid, b, x) for x in "ACGT" if x != b]                         # several candidates and ref lengths at one position
    v += [(mid, ref(mid, 2), b), (mid, ref(mid, 3), b), (mid, b, b + "A")]
    v += [v[0], v[6], v[15]]                                             # duplicates
    return v[len(v) // 2:] + v[:len(v) // 2]                             # unsorted


def _count(recs, pairs, cs, ce):
    return len(hc.hr.event_sequences(recs, pairs, cs, ce))


def build(spec):
    name, kind, trim, F, flags, threshold, types, which = spec
    draft, rs, recs, pairs, dur, deltas, first, truth = _pileup(kind, types)
    region_start, region_end = REGION_START + trim[0], REGION_START + len(draft) - 1 - trim[1]
    d = lambda p: draft[p - REGION_START]
    inside = lambda p, r: region_start <= p - F and p + len(r) + F <= region_end
    if which == "truth":
        cands = []
        for p, r, a in truth:
            if inside(p, r):
                cands.append((p, r, a))
            if inside(p + 2, "A"):
                cands.append((p + 2, d(p + 2), _other(d(p + 2))))
    elif which == "edges":
        cands = _edges(draft, region_start, region_end, F)
    elif which == "sparse":
        ps = range(region_start + F, region_end - F)
        zero = [p for p in ps if _count(recs, pairs, p - F, p + 1 + F) == 0]
        one = [p for p in ps if _count(recs, pairs, p - F, p + 1 + F) == 1]
        pick = [zero[0], zero[-1], one[0], one[len(one) // 2]] + list(ps)[::97]
        cands = [(p, d(p), _other(d(p))) for p in pick]
    elif which == "dense":
        at, n, _ = kind[6]["dense_at"]
        ps = [REGION_START + at + F + 1, REGION_START + at + n // 2, REGION_START + at - F - 3]
        cands = [(p, d(p), _other(d(p))) for p in ps]
    else:
        cands = []
        for p in range(region_start + F + 1, region_end - F - 1):
            edits = [(p, d(p), x) for x in "ACGT" if x != d(p)] + [(p, d(p), d(p) + x) for x in "ACGT"]
            if p % 7 == 0:
                cands += edits
                continue
            for e in edits:                                              # and every edit that makes or breaks a site
                x = scr.plan(region_start, draft[trim[0]:len(draft) - trim[1]], recs, pairs, [e], F, types)[0]
                if x and (len(x[1]) != len(x[2]) or max(len(x[1]), len(x[2])) == 3):
                    cands.append(e)
    c = dict(name=name, draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first, region_start=region_start,
             region_end=region_end, region_ref=draft[trim[0]:len(draft) - trim[1]], flank=F, flags=flags, threshold=threshold,
             types=tuple(types), candidates=cands, truth=truth)
    c["params"] = params(c)
    return c


def params(c, rpr=8):
    p = np.zeros(1, synth.SCREEN_LIST_PARAMS_DT)
    p[0] = (c["region_start"], c["flank"], c["threshold"], c["flags"], 6, rpr)
    return p


def candidate_array(cands):
    """(alleles u1, SCREEN_CANDIDATE_DT) of [(ref_position, ref_seq, alt_seq)]"""
    v = np.zeros(len(cands), synth.SCREEN_CANDIDATE_DT)
    buf, off = [], 0
    for i, (p, r, a) in enumerate(cands):
        v[i] = (p, len(r), len(a), off, off + len(r))
        buf += [r, a]
        off += len(r) + len(a)
    return np.frombuffer("".join(buf).encode() or b"\0", np.uint8).copy(), v


def fingerprint(c) -> str:
    h = hashlib.sha256()
    for a in (c["rs"].ev_mean, c["rs"].ev_start_time, c["recs"], c["pairs"]):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["draft"], c["candidates"], c["flank"], c["flags"], c["threshold"], c["types"], c["region_start"], c["region_end"])).encode())
    return h.hexdigest()


def plan(c, candidates=None):
    return scr.plan(c["region_start"], c["region_ref"], c["recs"], c["pairs"], c["candidates"] if candidates is None else candidates,
                    c["flank"], c["types"])


def ref_restated(ref, c, hs, mh):
    """scr.screened over the profile_hmm_score of `ref` (a tests/ref_variants.py RefVariants holding the case's reads as registered:
    hs, mh), the type models being its built-in ones"""
    models = [mh] + [ref.builtin_model(alphabet=t) for t in c["types"]]
    recs = c["recs"]

    def score(reqs):
        jobs = [(0, int(recs[r]["read"]), 1 + t, e1, e2, len(s) - 5, -1 if recs[r]["rc"] else 1, int(recs[r]["rc"]), c["flags"], 0)
                for r, e1, e2, t, s in reqs]
        return ref.score_batch(hs, np.array(jobs, synth.HMM_JOB_DT), [s.encode() for *_, s in reqs], models)[0]
    return scr.screened(plan(c), score, c["threshold"])


def meth_arg(c):
    """(nph_screen_methylation, alt model ids) of the case's types with the device suite's models, None without types"""
    if not c["types"]:
        return None
    n = c["recs"].shape[0]
    ids = np.array([[1 + ALL_TYPES.index(t) for t in c["types"]]] * n, np.uint32).reshape(n, len(c["types"]))
    return synth.screen_methylation(list(c["types"]), 6), ids


def device(eng, c, candidates=None, params_=None, methylation="case"):
    rs = c["rs"]
    alleles, cands = candidate_array(c["candidates"] if candidates is None else candidates)
    return eng.screen_variants_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(),
                                     c["deltas"], c["first"], c["recs"], c["params"] if params_ is None else params_, alleles, cands,
                                     methylation=meth_arg(c) if methylation == "case" else methylation)


def hmm_scores(eng, c):
    """score_set_jobs of scr.screened through nph_hmm_score_batch: each sequence's k-mer ranks in its alphabet on the job's strand"""
    recs, rs = c["recs"], c["rs"]

    def score(reqs):
        ranks, rows = [], []
        for r, e1, e2, t, s in reqs:
            rc = int(recs[r]["rc"])
            ranks.append(vmr.kmer_ranks(vmr.NUC if t < 0 else vmr.mr.ALPHABETS[c["types"][t]], s, 6, bool(rc)))
            rows.append((int(recs[r]["read"]), 0 if t < 0 else 1 + ALL_TYPES.index(c["types"][t]), e1, e2, rc, c["flags"]))
        jobs = np.zeros(len(rows), synth.HMM_JOB_DT)
        off = 0
        for j, ((read, m, e1, e2, rc, fl), rk) in enumerate(zip(rows, ranks)):
            jobs[j] = (off, read, m, e1, e2, rk.shape[0], -1 if rc else 1, rc, fl, 0)
            off += rk.shape[0]
        return eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.concatenate(ranks).astype(np.uint32), jobs)
    return score


def _cstrs(xs):
    return (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])


def mirror(host, c, candidates=None):
    """nph::screen_variants_by_score through the nphh_screen_variants shim: (status, [line per kept variant]).  With types, the reads
    get the device suite's type models (nphh_read_add_model)"""
    from tests.test_host_mirror import _register, _register_reads
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    host.nphh_clear()
    rs = c["rs"]
    mh = _register(host, synth.load_model("nucleotide"))
    hs = _register_reads(host, rs, mh)
    if c["types"]:
        from tests.test_variants_methylation_oracle import type_models
        tm = type_models(c["types"])
        for t in c["types"]:
            h = _register(host, tm[t])
            for r in hs:
                host.nphh_read_add_model(int(r), t.encode(), h)
    recs, pairs = c["recs"], c["pairs"]
    read = np.array([hs[int(x)] for x in recs["read"]], np.int32)
    rc = np.ascontiguousarray(recs["rc"], np.uint8)
    pp = np.ascontiguousarray(np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32))
    po = np.zeros(recs.shape[0] + 1, np.uint64)
    po[:-1] = recs["pair_off"]; po[-1] = pairs.shape[0]
    vs = c["candidates"] if candidates is None else candidates
    vp = np.array([x[0] for x in vs] or [0], np.int32)
    out = C.create_string_buffer(1 << 22)
    host.nphh_screen_variants.restype = C.c_longlong
    n = host.nphh_screen_variants(CONTIG.encode(), c["region_start"], c["region_ref"].encode(), int(recs.shape[0]), p(read), p(rc), p(pp), p(po),
                                  CONTIG.encode(), len(vs), p(vp), _cstrs([x[1] for x in vs]), _cstrs([x[2] for x in vs]), c["flank"],
                                  C.c_uint32(c["threshold"]), ",".join(c["types"]).encode(), C.c_uint32(c["flags"]), C.c_double(1.0), out,
                                  C.c_size_t(1 << 22))
    if n < 0:
        return int(n), None
    return int(n), out.raw[:n].decode().split("\n")[:-1]


def expand_candidates(c):
    """the round-1 list of an expand case: the truth's indels and substitutions inside the region, and two deletions whose extension
    ends min_flank + 1 and min_flank bases before region_end"""
    d = lambda p: c["draft"][p - REGION_START]
    hi = c["region_end"]
    out = [(p, r, a) for p, r, a in c["truth"] if c["region_start"] <= p and p + len(r) <= hi]
    for gap in (31, 30):
        p = hi - gap - 2
        out.append((p, c["draft"][p - REGION_START:p - REGION_START + 2], d(p)))
    out.append((c["region_start"] + 40, d(c["region_start"] + 40), d(c["region_start"] + 40) + "C"))
    return out


def host_expand(host, c, cands, min_flank, var_contig=CONTIG):
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    vp = np.array([x[0] for x in cands] or [0], np.int32)
    out = C.create_string_buffer(1 << 22)
    host.nphh_expand_variants.restype = C.c_longlong
    n = host.nphh_expand_variants(CONTIG.encode(), c["region_start"], c["region_ref"].encode(), var_contig.encode(), len(cands), p(vp),
                                  _cstrs([x[1] for x in cands]), _cstrs([x[2] for x in cands]), min_flank, out, C.c_size_t(1 << 22))
    if n < 0:
        return int(n), None
    return int(n), out.raw[:n].decode().split("\n")[:-1]


def expand_lines(xs):
    return [f"{p}\t{r}\t{a}" for p, r, a in xs]
