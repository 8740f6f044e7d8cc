"""call_haplotype_from_candidates test cases and the ways to run them — test infrastructure.

A case is a seeded pile-up (tests/support_cases.py's substitution pile-ups, or tests/screen_cases.py's planted recognition sites),
reads on both strands, a region over it, the read names, the options of the call (ploidy, genotype_only, max_haplotypes, -q types,
calculate_all_support) and a candidate list.  Its answers come from
  reference     the compiled reference's own call_haplotype_from_candidates (tests/ref_variants.py: oracle/_ref/libnpref_variants.so)
  restated      tests/call_restatement.py over the compiled reference's profile_hmm_score (the same library), or over
                nph_hmm_score_batch
  mirror        nph::call_haplotype_from_candidates through the nphh_call_haplotype shim (nph_call_variant_groups_batch).
Every answer is the derived sequence, then per variant of the derived haplotype "position, alleles, quality bits, INFO, genotype"."""
import ctypes as C
import hashlib

import numpy as np

from nanopolish_b200 import synth
from tests import call_restatement as cr
from tests import host_mirror as hm
from tests import hp_cases as hc
from tests import screen_cases as sc
from tests import support_cases as suc
from tests import var_meth_restatement as vmr

REGION_START = hc.REGION_START
CONTIG = hc.CONTIG
FLAGS = 3                               # HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, what `variants` passes
FLANK, MIN_DISTANCE = 30, 10            # opt::min_flanking_sequence, opt::min_distance_between_variants

# (name, pile-up, ploidy, genotype_only, max_haplotypes, -q types, calculate_all_support, candidates, names).  pile-up: as
# tests/screen_cases.py's.  candidates:
#   truth     the truth's substitutions, each with a wrong substitution 2 bases on (one group of two)
#   cluster   groups of 1 to 10 substitutions 3 bases apart, the truth's among them (max_r < n where max_haplotypes is small);
#             cluster2 from 2 on (Combinations(n, ploidy) asserts ploidy <= n: ploidy 3 needs 3 combinations), cluster10 one of 10
#   edges     two alleles at one position and a duplicate (combinations that fail apply_variants, equal haplotypes whose sets tie),
#             a group whose only candidate does not apply (one combination), windows of 200 and 201 bases, an unsorted pair
#   sparse    windows with no read and with one read
#   meth      two substitutions at every eleventh position, some making or breaking a CpG
# names: "plain" r<i>; "keys" names whose key order differs from name order ("a0:0" < "a:0"), and one record of a read repeated
# (a read aligned twice in its windows)
CASES = [
    ("truth_p1", ("snp", 900, 12, 240, 3, 10), 1, 0, 64, (), 0, "truth", "plain"),
    ("truth_p2_all", ("snp", 900, 12, 240, 3, 10), 2, 1, 8, (), 1, "truth", "plain"),
    ("cluster_p2_h64", ("snp", 1000, 10, 260, 5, 14), 2, 0, 64, (), 0, "cluster", "plain"),
    ("cluster_p3_h4", ("snp", 1000, 10, 260, 5, 14), 3, 1, 4, (), 0, "cluster2", "plain"),
    ("cluster_p1_h1000", ("snp", 1000, 10, 260, 5, 14), 1, 0, 1000, (), 0, "cluster", "plain"),
    ("cluster_p2_h1000", ("snp", 700, 8, 240, 6, 10), 2, 0, 1000, (), 0, "cluster10", "plain"),
    ("edges_p2", ("snp", 1200, 10, 300, 7, 12), 2, 1, 64, (), 0, "edges", "plain"),
    ("sparse_p2", ("snp", 900, 2, 150, 9, 0), 2, 1, 8, (), 0, "sparse", "plain"),
    ("keys_p2", ("snp", 900, 12, 240, 3, 10), 2, 1, 8, (), 1, "truth", "keys"),
    ("meth_cpg_p2", ("meth", 130, 10, 100, 72), 2, 1, 64, ("cpg",), 0, "meth", "plain"),
]


def _other(b: str) -> str:
    return "ACGT"[("ACGT".index(b.upper()) + 1) % 4]


def _names(n, kind):
    if kind == "plain":
        return [f"r{i}" for i in range(n)]
    # "a:0" sorts after "a0:0" and "a.:0" ... ':' (0x3a) is above '.' (0x2e) and '0'-'9' (0x30-0x39)
    stems = ["a", "a0", "a.", "a-", "b", "b9", "A", "a00"]
    return [stems[i % len(stems)] + ("" if i < len(stems) else str(i)) for i in range(n)]


def build(spec):
    name, kind, ploidy, gt_only, max_h, types, all_support, which, names = spec
    draft, rs, recs, pairs, dur, deltas, first, truth = sc._pileup(kind, types)
    region_start, region_end = REGION_START, REGION_START + len(draft) - 1
    d = lambda p: draft[p - REGION_START]
    lo, hi = region_start + FLANK + 2, region_end - FLANK - 2
    inside = lambda p: lo <= p and p + 12 <= hi
    if which == "truth":
        cands = []
        for p, r, a in truth:
            if inside(p):
                cands += [(p, r, a), (p + 2, d(p + 2), _other(d(p + 2)))]
    elif which.startswith("cluster"):
        tp = sorted(p for p, _, _ in truth)
        sizes = {"cluster": list(range(1, 11)), "cluster2": list(range(2, 11)), "cluster10": [10]}[which]
        tset = {p: a for p, _, a in truth}
        cands, at = [], lo
        for m in sizes:                                  # each group starts at the next truth position, or right after the last
            start = next((p for p in tp if p >= at and inside(p + 3 * (m - 1))), at)
            grp = [start + 3 * j for j in range(m)]
            assert inside(grp[-1]), "the region is too short for the clusters"
            cands += [(p, d(p), tset.get(p, _other(d(p)))) for p in grp]
            at = grp[-1] + MIN_DISTANCE + 1
    elif which == "edges":
        p0 = lo + 5
        cands = [(p0, d(p0), _other(d(p0))), (p0, d(p0), _other(_other(d(p0)))), (p0 + 4, d(p0 + 4), _other(d(p0 + 4))),
                 (p0 + 4, d(p0 + 4), _other(d(p0 + 4)))]                                      # two alleles at one position; a duplicate
        p1 = p0 + 60
        cands += [(p1, _other(d(p1)), d(p1))]                                                 # does not apply: one combination
        for width, p2 in ((200, p0 + 120), (201, p0 + 380)):                                  # windows of 200 and 201 bases
            span = width - 2 * FLANK - 1
            steps = list(range(0, span, 10)) + [span]
            cands += [(p2 + s, d(p2 + s), _other(d(p2 + s))) for s in sorted(set(steps))]
        p3 = p0 + 640
        cands += [(p3 + 6, d(p3 + 6), _other(d(p3 + 6))), (p3, d(p3), _other(d(p3)))]       # unsorted: a negative distance joins
        cands += [(p, r, a) for p, r, a in truth if p > p3 + 60 and inside(p)][:3]
    elif which == "sparse":
        ps = range(lo, hi - 12)
        zero = [p for p in ps if len(hc.hr.event_sequences(recs, pairs, p - FLANK, p + 1 + FLANK)) == 0]
        one = [p for p in ps if len(hc.hr.event_sequences(recs, pairs, p - FLANK, p + 1 + FLANK)) == 1]
        pick = sorted({zero[0], zero[-1], one[0], one[len(one) // 2]} | set(list(ps)[::83]))
        cands = [(p, d(p), _other(d(p))) for p in pick]
    else:
        cands = []
        for p in range(lo, hi - 12, 11):
            cands += [(p, d(p), x) for x in "ACGT" if x != d(p)][:2]
    if names == "keys":                                                                       # a read aligned twice
        recs = np.concatenate([recs, recs[[1]]])
    c = dict(name=name, draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, region_start=region_start, region_end=region_end,
             region_ref=draft, ploidy=ploidy, genotype_only=gt_only, max_haplotypes=max_h, types=tuple(types), all_support=all_support,
             candidates=cands, names=_names(rs.reads.shape[0], names), truth=truth)
    return c


def record_names(c):
    return [c["names"][int(r)] for r in c["recs"]["read"]]


def fingerprint(c) -> str:
    h = hashlib.sha256()
    for a in (c["rs"].ev_mean, c["rs"].ev_start_time, c["recs"], c["pairs"]):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["draft"], c["candidates"], c["ploidy"], c["genotype_only"], c["max_haplotypes"], c["types"], c["all_support"],
                   c["names"], c["region_start"], c["region_end"])).encode())
    return h.hexdigest()


def strip_all_support(lines):
    """the lines without ;SupportFractionByBase=... (not restated)"""
    out = [lines[0]]
    for l in lines[1:]:
        f = l.split("\t")
        f[4] = f[4].split(";SupportFractionByBase=")[0]
        out.append("\t".join(f))
    return out


def ref_restated(ref, c, hs, mh):
    """restated over the profile_hmm_score of `ref` (a tests/ref_variants.py RefVariants holding the case's reads as registered: hs,
    mh), the type models being its built-in ones"""
    models = [mh] + [ref.builtin_model(alphabet=t) for t in c["types"]]
    recs = c["recs"]

    def score(reqs):
        jobs = [(0, int(recs[r]["read"]), 1 + t, e1, e2, len(s) - 5, -1 if recs[r]["rc"] else 1, int(recs[r]["rc"]), FLAGS, 0)
                for r, e1, e2, t, s in reqs]
        return ref.score_batch(hs, np.array(jobs, synth.HMM_JOB_DT), [s.encode() for *_, s in reqs], models)[0]
    return restated(c, score)


def restated(c, score):
    return cr.restated(c["region_start"], c["region_ref"], c["recs"], c["pairs"], record_names(c), c["candidates"], score, FLANK, MIN_DISTANCE,
                       c["max_haplotypes"], c["ploidy"], bool(c["genotype_only"]), c["types"])


def hmm_scores(eng, c):
    """cr.restated's score() through nph_hmm_score_batch: each sequence's k-mer ranks in its alphabet on the job's strand (model ids as
    tests/screen_cases.py's device suite uploads them)"""
    recs, rs = c["recs"], c["rs"]

    def score(reqs):
        ranks, jobs = [], np.zeros(len(reqs), synth.HMM_JOB_DT)
        off = 0
        for j, (r, e1, e2, t, s) in enumerate(reqs):
            rc = int(recs[r]["rc"])
            rk = vmr.kmer_ranks(vmr.NUC if t < 0 else vmr.mr.ALPHABETS[c["types"][t]], s, 6, bool(rc))
            m = 0 if t < 0 else 1 + sc.ALL_TYPES.index(c["types"][t])
            jobs[j] = (off, int(recs[r]["read"]), m, e1, e2, rk.shape[0], -1 if rc else 1, rc, FLAGS, 0)
            ranks.append(rk)
            off += rk.shape[0]
        return eng.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.concatenate(ranks).astype(np.uint32), jobs)
    return score


def mirror(host, c, candidates=None, ploidy=None, all_support=None):
    """nph::call_haplotype_from_candidates through the nphh_call_haplotype shim: (status, lines).  With types, the reads get the device
    suite's type models (nphh_read_add_model)"""
    hs = hm.register_case(host, c, synth.load_model("nucleotide"), sc.type_models(c["types"]).values())
    vs = c["candidates"] if candidates is None else candidates
    n, raw = hm.text(host, "nphh_call_haplotype", CONTIG.encode(), c["region_start"], c["region_ref"].encode(), *hm.records(c, hs),
                     hm.cstrs(record_names(c)), CONTIG.encode(), len(vs), *hm.alleles(vs), FLANK, MIN_DISTANCE, c["max_haplotypes"],
                     c["ploidy"] if ploidy is None else ploidy, c["genotype_only"], ",".join(c["types"]).encode(),
                     c["all_support"] if all_support is None else all_support, C.c_uint32(FLAGS), C.c_double(1.0))
    return n, (None if raw is None else raw.decode().split("\n")[:-1])


def device_inputs(c, genotype_all=1):
    """nph_call_variant_groups_batch's arrays for c's called groups, built as the mirror builds them: (params, groups, haplotypes,
    bases, combination variants, n_variants, key ranks)"""
    groups, haps, bases, cvars, nv = [], [], [], [], 0
    for first, end, cs, ce in cr.groups(c["candidates"], FLANK, MIN_DISTANCE):
        if ce - cs > 200:
            continue
        vs = c["candidates"][first:end]
        combos = cr.combinations(vs, cr.Hap(c["region_ref"][cs - REGION_START:ce - REGION_START + 1], cs), c["max_haplotypes"])
        if len(combos) <= 1:
            continue
        groups.append((cs, ce, len(haps), len(combos), nv, len(vs)))
        nv += len(vs)
        for ids, seq in combos:
            haps.append((sum(len(b) for b in bases), len(seq), len(ids), len(cvars)))
            bases.append(seq)
            cvars += list(ids)
    g = np.array(groups, synth.CALL_GROUP_DT)
    h = np.array(haps, synth.CALL_HAPLOTYPE_DT)
    b = np.frombuffer("".join(bases).encode() or b"\0", np.uint8).copy()
    p = np.zeros(1, synth.CALL_PARAMS_DT)
    p[0] = (c["region_start"], c["ploidy"], genotype_all, FLAGS, 6)
    names = [n + ":0" for n in c["names"]]
    order = sorted(set(names))
    kr = np.array([order.index(n) for n in names], np.uint32)
    return p, g, h, b, np.array(cvars or [0], np.uint32), nv, kr


def device(eng, c, recs=None, **kw):
    """nph_call_variant_groups_batch on c (records, params, groups, haplotypes, cvars, methylation replaceable)"""
    p, g, h, b, cv, nv, kr = device_inputs(c)
    for k, v in kw.items():
        if k == "params":
            p = v
        elif k == "groups":
            g = v
        elif k == "haplotypes":
            h = v
        elif k == "cvars":
            cv = v
    rs = c["rs"]
    recs = c["recs"] if recs is None else recs
    deltas, first = synth.compact_event_alignment(recs, c["pairs"], int(recs["ref_len"].sum())) if recs.shape[0] else (np.zeros(1, np.int16), np.zeros(1, np.int32))
    return eng.call_variant_groups_batch(rs.reads, rs.ev_mean, rs.ev_start_time, np.frombuffer(c["region_ref"].encode(), np.uint8).copy(), deltas, first,
                                         recs, kr, p, g, h, b, cv, nv, methylation=kw.get("methylation"))
