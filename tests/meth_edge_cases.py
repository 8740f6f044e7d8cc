"""call-methylation records built to reach named edges of the device front end in nanopolish_b200/csrc/methylation.cu:
meth_scan_kernel (the site ballot 32 bases at a time, the grouping, the window tests, warp_lower_bound / warp_first_valid),
meth_expand_kernel (the compact event alignment), meth_emit_kernel (the window, its methylated copy, reverse placement) and
meth_tsv_kernel (rows in chunks of 32).

Every case is a read whose events are generated from a chosen sequence with recognition sites planted at exact offsets
(synth.gen_reads_from_sequence), aligned with a chosen CIGAR to a contig, and presented the way the BAM / FASTA /
SquiggleRead present it to calculate_methylation_for_read (tests/meth_cases.py): the fetched reference, the CIGAR and the
base-to-event map, from which the device record and its aligned_events pair list follow.  Each case states one edge claim,
which check_claims confirms on the restatement (tests/meth_restatement.py).

Cases with the reference's parameters (`params` empty: min_separation 10, min_flank 10, max_span 200, min_event_span 10,
region filter allowed) are asked of the compiled reference; the others are checked on the restatement scored by the port oracle.
A case with `cut` keeps its pair list but presents only the first `cut` reference bases, so windows run past the end of the
record's reference while still bounded by the event alignment: the reference never meets that, the device must cut them like
std::string::substr does, or refuse a window shorter than k."""
from __future__ import annotations

import bisect
import hashlib
from dataclasses import dataclass, field

import numpy as np

from nanopolish_b200 import synth
from oracle import eventalign_py as ea
from tests import meth_cases as mc
from tests import meth_restatement as mr

K = 6
CHUNK = 32            # bases per ballot in meth_scan_kernel / meth_expand_kernel, rows per chunk in meth_tsv_kernel
WARPS = 8             # kWarps: warps per block of every kernel
GRID_PER_SM = 8       # every kernel launches at most sm_count * GRID_PER_SM blocks
MAX_WINDOW = 1024     # NPH_METH_MAX_WINDOW, include/nph.h
PAD = 300             # contig bases before the alignment (and after it, unless right_pad is False)
MODEL_ID = {"cpg": 1, "dam": 2, "dcm": 3}        # models: nucleotide, cpg, dam, dcm in this order
ALPHABETS = ("cpg", "dam", "dcm")
DEFAULT = dict(min_separation=10, min_flank=10, max_span=200, min_event_span=10)


def models():
    return [synth.load_model(a) for a in ("nucleotide",) + ALPHABETS]


@dataclass
class Case:
    name: str
    claim: str
    ref: str                            # the fetched reference ref_seq: the alignment covers ref[:-1] (all of it without right_pad)
    check: object                       # check(View) -> bool: the claim, on the restatement
    rev: bool = False
    ops: tuple | None = None            # CIGAR ops [(n, op)] over the aligned reference; None: all M
    nev: np.ndarray | None = None       # events per k-mer of the aligned reference, in reference order (None: random)
    alphabet: str = "cpg"
    params: dict = field(default_factory=dict)       # window parameters other than the reference's
    region: tuple = (-1, -1)
    right_pad: bool = True              # False: the contig ends where the alignment ends
    cut: int | None = None
    seed: int = 0

    @property
    def reference_case(self) -> bool:
        return not self.params and self.cut is None

    @property
    def kw(self) -> dict:
        return dict(DEFAULT, **self.params, region_start=self.region[0], region_end=self.region[1])

    @property
    def group(self) -> tuple:
        """the cases that share one device call: one parameter block, and cut records apart (the compact form, one delta per
        reference base, cannot carry the pairs past a record's reference)"""
        return (self.alphabet, tuple(sorted(self.kw.items())), self.cut is not None)


# ---------------------------------------------------------------- sequences
def _motifs(s: str, alphabet: str) -> list:
    a = mr.ALPHABETS[alphabet]
    return [i for i in range(len(s) - 1) if mr.is_motif_match(a, s, i)]


def plant(n: int, sites, alphabet: str = "cpg", seed: int = 0, site_of=None) -> str:
    """n random bases without a recognition site except the ones planted at `sites` (dcm: CCAGG, or CCTGG where site_of says)"""
    rng = np.random.default_rng(seed)
    a = mr.ALPHABETS[alphabet]
    s = list("ACGT"[x] for x in rng.integers(0, 4, n))
    for _ in range(100):
        hits = _motifs("".join(s), alphabet)
        if not hits:
            break
        for h in hits:
            s[h + 1] = "T" if s[h + 1] != "T" else "A"
    for j, p in enumerate(sites):
        site = a["sites"][site_of[j] if site_of else 0]
        s[p:p + len(site)] = list(site)
    out = "".join(s)
    assert len(out) == n
    assert _motifs(out, alphabet) == sorted(sites), (sites, _motifs(out, alphabet))
    return out


# ---------------------------------------------------------------- a case as the reference and the device see it
@dataclass
class Built:
    case: Case
    inputs: dict                       # meth_cases.make_case's dict: read_sequence, b2e_start/stop, contig, ref_pos, flag, cigar, name, ref_len
    ref: str                           # what the record presents (ref_seq, or its first `cut` bases)
    pairs: np.ndarray                  # PAIR_DT
    rc: int
    read: int                          # index in the batch's ReadSet


def _query(case: Case, rng):
    """the BAM query the CIGAR walks, and the query position of every aligned reference base (-1: deleted)"""
    body = case.ref if not case.right_pad else case.ref[:-1]
    ops = case.ops or ((len(body), "M"),)
    q, qpos, r = [], [], 0
    for n, op in ops:
        if op == "M":
            qpos += list(range(len(q), len(q) + n)); q += list(body[r:r + n]); r += n
        elif op == "D":
            qpos += [-1] * n; r += n
        else:                               # I, S: bases the reference does not have
            q += ["ACGT"[x] for x in rng.integers(0, 4, n)]
    assert r == len(body), (case.name, r, len(body))
    return "".join(q), qpos, ops


def build(cases):
    """-> (ReadSet with one read per case, [Built])"""
    nuc = synth.load_model("nucleotide")
    sets, built = [], []
    for i, c in enumerate(cases):
        rng = np.random.default_rng(1000 + c.seed + i)
        query, qpos, ops = _query(c, rng)
        read_seq = mc.revcomp(query) if c.rev else query
        nev = None
        if c.nev is not None:
            # per k-mer of the read: the reference-ordered counts moved onto the query, then into read order
            nk = len(query) - K + 1
            nq = np.ones(nk, np.int64)
            for ro, qp in enumerate(qpos):
                if qp >= 0 and qp < nk and ro < c.nev.shape[0]:
                    nq[qp] = c.nev[ro]
            nev = nq[::-1].copy() if c.rev else nq
        rs = synth.gen_reads_from_sequence(synth.encode(read_seq, "nucleotide"), 1, nuc, seed=7919 * (i + 1) + c.seed, nev=nev)
        left = "".join("ACGT"[x] for x in rng.integers(0, 4, PAD))
        body = c.ref if not c.right_pad else c.ref[:-1]
        right = (c.ref[-1] + "".join("ACGT"[x] for x in rng.integers(0, 4, PAD - 1))) if c.right_pad else ""
        which = rs.ev_kmer[0]
        nk = len(read_seq) - K + 1
        first = np.searchsorted(which, np.arange(nk), side="left")
        last = np.searchsorted(which, np.arange(nk), side="right") - 1
        inputs = dict(read_sequence=read_seq, b2e_start=np.where(last >= first, first, -1).astype(np.int32),
                      b2e_stop=np.where(last >= first, last, -1).astype(np.int32), contig=left + body + right, ref_pos=PAD,
                      flag=16 if c.rev else 0, cigar=ea.pack_cigar(list(ops)), name=f"edge_{i}_{c.name}", ref_len=len(body))
        assert mc.fetched_reference(inputs) == c.ref, c.name
        pl, rc = mc.event_alignment_record(inputs)
        pr = np.zeros(len(pl), synth.PAIR_DT)
        if pl:
            pr["ref_pos"], pr["read_pos"] = [p[0] for p in pl], [p[1] for p in pl]
        sets.append(rs)
        built.append(Built(c, inputs, c.ref if c.cut is None else c.ref[:c.cut], pr, rc, i))
    return concat(sets), built


def concat(sets):
    reads = np.concatenate([s.reads for s in sets])
    off = np.cumsum([0] + [s.total_events for s in sets[:-1]])
    reads["event_off"] += np.repeat(off, [s.n_reads for s in sets]).astype(np.uint64)
    return synth.ReadSet(reads, np.concatenate([s.ev_mean for s in sets]), np.concatenate([s.ev_start_time for s in sets]),
                         sum((s.seq_codes for s in sets), []), sum((s.ev_kmer for s in sets), []),
                         sum((s.kmer_first_event for s in sets), []), K)


def fingerprint(rs, b: Built) -> str:
    """hash of everything the reference reads for this case"""
    h = hashlib.sha256()
    r = rs.reads[b.read]
    o, n = int(r["event_off"]), int(r["n_events"])
    x = b.inputs
    for part in (x["read_sequence"].encode(), x["b2e_start"].tobytes(), x["b2e_stop"].tobytes(), x["contig"].encode(),
                 x["cigar"].tobytes(), rs.ev_mean[o:o + n].tobytes(), rs.ev_start_time[o:o + n].tobytes(), r.tobytes(),
                 repr((x["ref_pos"], x["flag"], x["name"], b.case.alphabet, b.case.region)).encode()):
        h.update(part)
    return h.hexdigest()[:24]


def records(built, read_index=None):
    """-> (ref_bases u8, pairs PAIR_DT, records METH_RECORD_DT) of these cases in one device call"""
    refs, prs = [], []
    recs = np.zeros(len(built), synth.METH_RECORD_DT)
    ro = po = 0
    for j, b in enumerate(built):
        r = np.frombuffer(b.ref.encode(), np.uint8)
        recs[j] = (ro, po, b.read if read_index is None else read_index[j], MODEL_ID[b.case.alphabet], r.shape[0], b.pairs.shape[0],
                   PAD, b.rc, 0, (0, 0))
        refs.append(r); prs.append(b.pairs)
        ro += r.shape[0]; po += b.pairs.shape[0]
    return np.concatenate(refs), np.concatenate(prs), recs


def restated(b: Built, moved=None):
    """the restatement's groups of one case: [(start, end, n_motif, e1, e2, ranks_u, ranks_m, sequence)]"""
    return mr.enumerate_record(b.ref, PAD, b.pairs["ref_pos"].tolist(), b.pairs["read_pos"].tolist(), b.rc, b.case.alphabet, K,
                               moved=moved, **b.case.kw)


def score(port, rs, mods, b: Built, groups):
    """(ll_unmethylated, ll_methylated) float32 per group: the port oracle on the restatement's jobs"""
    if not groups:
        return np.zeros((0, 2), np.float32)
    flags = synth.HAF_ALLOW_PRE_CLIP | synth.HAF_ALLOW_POST_CLIP
    jobs = np.zeros(2 * len(groups), synth.HMM_JOB_DT)
    ranks, off = [], 0
    for j, g in enumerate(groups):
        for t, rk in enumerate((g[5], g[6])):
            jobs[2 * j + t] = (off, b.read, MODEL_ID[b.case.alphabet], g[3], g[4], rk.shape[0], 1 if g[3] <= g[4] else -1, b.rc, flags, 0)
            ranks.append(rk); off += rk.shape[0]
    s, _ = port.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, mods, np.concatenate(ranks).astype(np.uint32), jobs)
    return s.reshape(-1, 2)


def tsv(b: Built, groups, ll) -> str:
    rows = [(g[0], g[1], g[2], ll[j, 0], ll[j, 1], g[7]) for j, g in enumerate(groups)]
    return mc.tsv_rows("chr1", "-" if b.rc else "+", b.inputs["name"], rows)


def answer(b: Built, groups, ll):
    """a case's answer in the reference harness's form: (tsv, int32[n, 4] start/end/n_motif/strands, float64[n, 2])"""
    s = np.array([(g[0], g[1], g[2], 1) for g in groups], np.int32).reshape(-1, 4)
    return tsv(b, groups, ll), s, ll.astype(np.float64).reshape(-1, 2)


def ask_reference(live, handles, rs, b: Built):
    x = b.inputs
    one = np.ones(int(rs.reads[b.read]["n_events"]), np.float32)
    live.read_set_eventalign(int(handles[b.read]), x["name"], x["read_sequence"], x["b2e_start"], x["b2e_stop"], one, one)
    return tuple(live.call_methylation(int(handles[b.read]), x["name"], "chr1", x["contig"], x["ref_pos"], x["flag"], x["cigar"],
                                       b.case.alphabet, region=b.case.region))


# ---------------------------------------------------------------- the 32-ary lower bound, restated with its probes
def lower_bound_trace(vals, v, lanes=32):
    """warp_lower_bound(pairs, n, v) as methylation.cu runs it -> (index, [(round, lane) whose probe holds exactly v], rounds)"""
    n = len(vals)
    lo, hi, rnd, hits = 0, n, 0, []
    while hi - lo > lanes:
        rnd += 1
        step = (hi - lo + lanes - 1) // lanes
        idx = [lo + (l + 1) * step - 1 for l in range(lanes)]
        less = [i < hi and vals[i] < v for i in idx]
        hits += [(rnd, l) for l, i in enumerate(idx) if i < hi and vals[i] == v]
        c = sum(less)
        nlo, nhi = lo + c * step, min(hi, lo + (c + 1) * step - 1)
        lo = min(nlo, hi); hi = max(nhi, lo)
    got = lo + sum(1 for i in range(lo, lo + lanes) if i < hi and vals[i] < v)
    assert got == bisect.bisect_left(vals, v)
    return got, hits, rnd


# ---------------------------------------------------------------- what a claim may look at
@dataclass
class View:
    b: Built
    sites: list                       # motif offsets in the record's reference
    groups: list                      # [(first, last, n_motif)] before any window test
    kept: list                        # restated output groups as (first, last, n_motif) offsets
    out: list                         # restated output groups, whole

    @property
    def n(self):
        return len(self.b.ref)

    @property
    def pair_offsets(self):
        return (self.b.pairs["ref_pos"].astype(np.int64) - PAD).tolist()

    def win(self, first, last):
        f = self.b.case.kw["min_flank"]
        return first - f, last + f

    def win_len(self, first, last):
        s, e = self.win(first, last)
        return min(e, self.n - 1) - s + 1

    def bounds(self, first, last):
        s, e = self.win(first, last)
        pr = self.b.pairs
        return mr.find_by_ref_bounds(pr["ref_pos"].tolist(), pr["read_pos"].tolist(), s + PAD, e + PAD)

    def has(self, first):
        return any(g[0] == first for g in self.kept)

    def contacts(self):
        """{(first site of a called group, site p, how p meets that group's window)}: cut-left (p < start <= p + rl - 1),
        flush-left (p == start), inside, flush-right (p + rl - 1 == end), cut-right (p <= end < p + rl - 1)"""
        rl = len(mr.ALPHABETS[self.b.case.alphabet]["sites"][0])
        out = set()
        for f, l, _ in self.kept:
            s, e = self.win(f, l)
            e = min(e, self.n - 1)
            for p in self.sites:
                if p + rl - 1 < s or p > e:
                    continue
                rel = ("cut-left" if p < s else "cut-right" if p + rl - 1 > e else "flush-left" if p == s
                       else "flush-right" if p + rl - 1 == e else "inside")
                out.add((f, p, rel))
        return out

    def lb_hits(self, rnd):
        """(boundary offset, lane) of every window boundary whose lower bound meets a probe exactly in round rnd"""
        vals = self.b.pairs["ref_pos"].tolist()
        out = []
        for f, l, _ in self.groups:
            for v in self.win(f, l):
                out += [(v, lane) for r, lane in lower_bound_trace(vals, v + PAD)[1] if r == rnd]
        return out

    def compact_steps(self):
        ev = self.b.pairs["read_pos"].astype(np.int64)
        return np.diff(ev)


def view(b: Built) -> View:
    a = b.case
    sites = _motifs(b.ref, a.alphabet)
    groups, cur = [], 0
    sep = a.kw["min_separation"]
    while cur < len(sites):
        end = cur + 1
        while end < len(sites) and sites[end] - sites[end - 1] <= sep:
            end += 1
        groups.append((sites[cur], sites[end - 1], end - cur)); cur = end
    out = restated(b)
    return View(b, sites, groups, [(g[0] - PAD, g[1] - PAD, g[2]) for g in out], out)


def refused(v: View) -> bool:
    """the device refuses the record: a window that passes every test is shorter than k"""
    kw = v.b.case.kw
    for f, l, _ in v.groups:
        s, e = v.win(f, l)
        if s <= kw["min_separation"] or l - f > kw["max_span"]:
            continue
        bd = v.bounds(f, l)
        if bd is None or abs(bd[1] - bd[0]) <= kw["min_event_span"]:
            continue
        sp, ep = f + PAD, l + PAD
        if (kw["region_start"] != -1 and sp < kw["region_start"]) or (kw["region_end"] != -1 and ep >= kw["region_end"]):
            continue
        if v.win_len(f, l) < K:
            return True
    return False


# ---------------------------------------------------------------- the cases
def _span_gaps(span):
    """gaps of 9 and 10 that add up to span (cpg sites every 9 or 10 bases stay one group)"""
    for nine in range(0, 40):
        if (span - 9 * nine) % 10 == 0 and span - 9 * nine >= 0:
            return [9] * nine + [10] * ((span - 9 * nine) // 10)
    raise ValueError(span)


def _at(start, gaps):
    out = [start]
    for g in gaps:
        out.append(out[-1] + g)
    return out


def scan_cases():
    out = []
    s = plant(200, [31, 63, 95, 127])
    out.append(Case("cpg-chunk-split", "cpg sites at 31, 63, 95, 127 straddle the 32-base ballots and each is a group that is called", s,
                    lambda v: all(v.has(p) for p in (31, 63, 95, 127))))
    for alpha, rl in (("dam", 4), ("dcm", 5)):
        for p in range(CHUNK - rl + 1, CHUNK):
            for rev in (False, True):
                s = plant(160, [p, p + 50], alpha, seed=p, site_of=[1, 0] if alpha == "dcm" else None)
                out.append(Case(f"{alpha}-split-{p}{'-rc' if rev else ''}",
                                f"a {alpha} site at {p} has {CHUNK - p} of its {rl} bases in the first ballot and is called"
                                + (" on the reverse strand" if rev else ""), s, lambda v, p=p: v.has(p) and v.has(p + 50), rev=rev, alphabet=alpha))
    s = plant(160, [33, 45, 57, 90])
    out.append(Case("groups-closed-in-one-ballot", "the sites at 45 and 57 close the groups of 33 and 45 inside one ballot (32..63)", s,
                    lambda v: [g[0] for g in v.groups[:3]] == [33, 45, 57] and all(33 <= g[0] < 64 for g in v.groups[:3])
                    and all(v.has(p) for p in (33, 45, 57))))
    s = plant(220, list(range(40, 137, 8)))
    out.append(Case("group-over-four-ballots", "one group of 13 sites from 40 to 136 spans ballots 1 to 4 and is called", s,
                    lambda v: v.kept and v.kept[0] == (40, 136, 13)))
    # the last scan position n - 2: its site (the alignment's last base and the base after it) joins the group of n - 12,
    # whose window is then no longer bounded by the event alignment; without it the group of n - 12 would be called
    n = 150
    s = plant(n, [40, n - 12, n - 2])
    out.append(Case("site-at-last-scan-position", "the site at n - 2 is found and extends the group of n - 12 past the event alignment", s,
                    lambda v: v.groups[-1][:2] == (n - 12, n - 2) and not v.has(n - 12) and v.has(40)
                    and v.bounds(n - 12, n - 12) is not None, ops=((n - 1, "M"), (6, "S"))))
    return out


def window_cases():
    out = []
    s = plant(120, [20, 60])
    out.append(Case("sub_start=min_separation", "the group at 20 has sub_start == min_separation (10) and is refused; 60 is called", s,
                    lambda v: v.win(20, 20)[0] == 10 and not v.has(20) and v.has(60)))
    s = plant(120, [21, 60])
    out.append(Case("sub_start=min_separation+1", "the group at 21 has sub_start == 11 and is called", s,
                    lambda v: v.win(21, 21)[0] == 11 and v.has(21)))
    for span, ok in ((200, True), (201, False)):
        sites = _at(30, _span_gaps(span))
        s = plant(sites[-1] + 60, sites)
        out.append(Case(f"span={span}", f"one group spans {span} bases and is {'called' if ok else 'refused'}", s,
                        lambda v, span=span, ok=ok: v.groups[0][1] - v.groups[0][0] == span and v.has(30) == ok))
    s = plant(160, [40, 50, 80, 91, 130])
    out.append(Case("separation=10,11", "sites 10 apart (40, 50) form one group, sites 11 apart (80, 91) two", s,
                    lambda v: (40, 50, 2) in v.kept and v.has(80) and v.has(91)))
    # event span: e2 - e1 is the number of events over [sub_start, sub_end) when every k-mer there has 0 or 1 events
    for de in (10, 11):
        nev = np.full(200, 2, np.int64)
        nev[30:50] = 0
        nev[30:50:2] = 1
        if de == 11:
            nev[31] = 1
        nev[50] = 1
        s = plant(140, [40, 100])
        out.append(Case(f"event-span={de}", f"the window of 40 spans exactly {de} events and is {'refused' if de == 10 else 'called'}", s,
                        lambda v, de=de: v.bounds(40, 40) is not None and abs(v.bounds(40, 40)[1] - v.bounds(40, 40)[0]) == de
                        and v.has(40) == (de == 11) and v.has(100), nev=nev))
    s = plant(200, [40, 80, 120, 160])
    out.append(Case("region-start=,end=", "start == region_start is called, end == region_end is not", s,
                    lambda v: [g[0] for g in v.kept] == [80, 120], region=(PAD + 80, PAD + 160)))
    out.append(Case("region-start-1,end-1", "start == region_start - 1 is not called, end == region_end - 1 is", s,
                    lambda v: [g[0] for g in v.kept] == [120, 160], region=(PAD + 81, PAD + 161), seed=1))
    # a window that ends exactly on the last base of a contig that ends with the alignment (not cut)
    n = 140
    s = plant(n, [40, n - 11])
    out.append(Case("window-ends-at-reference-end", "the window of n - 11 ends on the last reference base and is called whole", s,
                    lambda v: v.win(n - 11, n - 11)[1] == v.n - 1 and v.has(n - 11) and v.win_len(n - 11, n - 11) == 21,
                    ops=((n, "M"), (6, "S")), right_pad=False))
    return out


def lower_bound_cases():
    out = []
    for n_pairs in (32, 33):
        L = n_pairs + 2 * K
        s = plant(L + 1, [23])
        out.append(Case(f"pairs={n_pairs}", f"{n_pairs} pairs: {'no search round' if n_pairs == 32 else 'one round'}; the window of 23 is called",
                        s, lambda v, n_pairs=n_pairs: v.b.pairs.shape[0] == n_pairs and v.has(23)
                        and lower_bound_trace(v.b.pairs["ref_pos"].tolist(), PAD + 13)[2] == (0 if n_pairs == 32 else 1)
                        and (n_pairs == 32 or v.lb_hits(1))))
    for n_pairs in (1056, 1057):
        L = n_pairs + 2 * K
        step = (n_pairs + 31) // 32
        firsts = []
        for lane in (0, 1, 5, 17, 29):
            firsts.append((lane + 1) * step - 1 + K + 10)              # sub_start on probe `lane` of round 1
        if n_pairs == 1057:
            for lane in (3, 20):                                       # sub_start on probe 2 of round 2 inside that interval
                firsts.append(lane * step + 5 + K + 10)
        firsts = sorted(set(firsts))
        s = plant(L + 1, firsts, seed=n_pairs)
        rounds = 1 if n_pairs == 1056 else 2
        out.append(Case(f"pairs={n_pairs}", f"{n_pairs} pairs: {rounds} search round(s); window starts on probes of every round are called", s,
                        lambda v, firsts=firsts, n_pairs=n_pairs, rounds=rounds: v.b.pairs.shape[0] == n_pairs and all(v.has(f) for f in firsts)
                        and v.lb_hits(1) and (rounds == 1 or v.lb_hits(2))
                        and max(lower_bound_trace(v.b.pairs["ref_pos"].tolist(), PAD + f - 10)[2] for f in firsts) == rounds))
    return out


def alignment_cases():
    """the event alignment as the compact form carries it: where it starts, runs without entries, large steps"""
    out = []
    s = plant(200, [40, 120])
    out.append(Case("first-aligned-base-0", "a 6-base soft clip puts the first pair on reference base 0", s,
                    lambda v: v.pair_offsets[0] == 0 and v.has(40), ops=((6, "S"), (199, "M"))))
    for d in (25, 26, 27):
        s = plant(200, [60, 120], seed=d)
        out.append(Case(f"first-aligned-base-{d + K}", f"a leading {d}-base deletion puts the first pair on base {d + K}", s,
                        lambda v, d=d: v.pair_offsets[0] == d + K and v.has(60), ops=((d, "D"), (199 - d, "M"))))
    s = plant(200, [25, 80, 150])
    out.append(Case("boundary-before-first-entry", "the window of 25 starts at 15, before the first pair (36): not left-bounded, not called", s,
                    lambda v: v.pair_offsets[0] == 36 and v.bounds(25, 25) is None and not v.has(25) and v.has(80),
                    ops=((30, "D"), (169, "M"))))
    s = plant(240, [88, 150])
    out.append(Case("boundary-inside-deletion", "the window of 88 starts inside a 40-base deletion (50..89, across base 64) "
                    "and is left-bounded only by the pairs before it", s,
                    lambda v: 49 in v.pair_offsets and 50 not in v.pair_offsets and 89 not in v.pair_offsets and 90 in v.pair_offsets
                    and v.win(88, 88)[0] == 78 and v.has(88),
                    ops=((50, "M"), (40, "D"), (149, "M")), nev=np.full(300, 3, np.int64)))
    nev = np.full(300, 0, np.int64)
    nev[0] = 500
    s = plant(200, [40, 120])
    out.append(Case("no-pairs", "every k-mer's closest event is event 0: the aligned_events list is cleared and nothing is called", s,
                    lambda v: v.b.pairs.shape[0] == 0 and not v.kept and v.groups, nev=nev))
    for rev in (False, True):
        nev = np.full(300, 2, np.int64)
        nev[100] = 32767 if not rev else 1
        nev[101] = 32767 if rev else 2
        s = plant(200, [40, 105], seed=3)
        want = -32767 if rev else 32767
        out.append(Case(f"step{want:+d}", f"one event-index step of {want:+d} between reference bases 100 and 101, inside the window of 105", s,
                        lambda v, want=want: want in v.compact_steps().tolist() and v.has(105) and v.has(40), nev=nev, rev=rev))
    return out


def emit_cases():
    out = []
    # the site of the neighbouring group only partly inside the window at its left end (default parameters)
    s = plant(160, [40, 51, 100], "dam", seed=5)
    for rev in (False, True):
        out.append(Case(f"dam-partial-left{'-rc' if rev else ''}", "dam: the window of 51 starts on the A of the site at 40", s,
                        lambda v: v.win(51, 51)[0] == 41 and (51, 40, "cut-left") in v.contacts() and v.has(40),
                        alphabet="dam", rev=rev))
    s = plant(170, [40, 52, 110], "dcm", seed=6, site_of=[0, 1, 1])
    for rev in (False, True):
        out.append(Case(f"dcm-partial-left{'-rc' if rev else ''}", "dcm: the window of 52 starts on the third base of the site at 40"
                        + (" (placed at L - q - rl on the reverse strand)" if rev else ""),
                        s, lambda v: v.win(52, 52)[0] == 42 and (52, 40, "cut-left") in v.contacts(), alphabet="dcm", rev=rev))
    # min_flank > min_separation: other groups' sites cut by either end of a window, flush with either end, or wholly inside
    p = dict(min_separation=5, min_flank=15)
    for alpha, sites, of, want in (
            ("cpg", [40, 55, 70, 84, 100], None,
             {(40, 55, "cut-right"), (55, 40, "flush-left"), (55, 70, "cut-right"), (70, 84, "flush-right"), (100, 84, "cut-left")}),
            ("dam", [40, 53, 70, 82, 88], None,
             {(40, 53, "cut-right"), (53, 40, "inside"), (70, 53, "cut-left"), (70, 82, "flush-right"), (88, 70, "cut-left")}),
            ("dcm", [40, 52, 70, 81, 88], [1, 0, 1, 0, 1],
             {(40, 52, "cut-right"), (52, 40, "inside"), (70, 52, "cut-left"), (70, 81, "flush-right"), (88, 81, "inside")})):
        s = plant(170, sites, alpha, seed=8, site_of=of)
        text = ", ".join(f"{r} {q} in the window of {f}" for f, q, r in sorted(want))
        for rev in (False, True):
            out.append(Case(f"{alpha}-flank>separation{'-rc' if rev else ''}",
                            f"{alpha}, flank 15, separation 5: site {text}" + (" (placed at L - q - rl on the reverse strand)" if rev else ""),
                            s, lambda v, want=want, sites=sites: want <= v.contacts() and all(v.has(x) for x in sites),
                            alphabet=alpha, params=p, rev=rev))
    # the largest window: max_span + 2 * min_flank + 1 == NPH_METH_MAX_WINDOW
    span = MAX_WINDOW - 21
    sites = _at(30, _span_gaps(span))
    s = plant(sites[-1] + 80, sites, seed=9)
    for rev in (False, True):
        out.append(Case(f"window=1024{'-rc' if rev else ''}", "one group spans 1003 bases: its window is exactly 1024 bases", s,
                        lambda v: len(v.out) == 1 and v.win_len(30, sites[-1]) == MAX_WINDOW and v.has(30),
                        params=dict(max_span=span), rev=rev))
    # windows cut by the end of the record's reference (pairs continue past it): to k bases, and the site at n - 2
    s = plant(200, [40, 90, 137], seed=10)
    out.append(Case("cut-window", "the record ends 3 bases after the site at 137: its window is cut to 13 bases and called", s,
                    lambda v: v.n == 140 and v.win_len(137, 137) == 13 and v.has(137), cut=140))
    return out


def row_cases():
    out = []
    for n_rows in (31, 32, 33, 64, 65):
        sites = [30 + 12 * j for j in range(n_rows)]
        s = plant(sites[-1] + 40, sites, seed=n_rows)
        out.append(Case(f"rows={n_rows}", f"{n_rows} groups, each called: {n_rows} rows for meth_tsv_kernel's 32-row chunks", s,
                        lambda v, n_rows=n_rows: len(v.kept) == n_rows, rev=n_rows % 2 == 1))
    return out


def refusal_cases():
    """cut records whose last window, after every test, has k - 1 bases (refused) or k bases (called)"""
    out = []
    s = plant(200, [40, 90, 134], seed=11)
    for extra, ok in ((3, True), (2, False)):
        cut = 134 + extra
        # flank 3: the window of 134 is [131, 137] cut at cut - 1
        out.append(Case(f"cut-to-{'k' if ok else 'k-1'}", f"flank 3: the record ends {extra} bases after the site at 134; its window is cut to "
                        f"{K if ok else K - 1} bases and {'called' if ok else 'refused'}", s,
                        lambda v, ok=ok: v.win_len(134, 134) == (K if ok else K - 1) and refused(v) == (not ok) and v.bounds(134, 134) is not None,
                        params=dict(min_flank=3), cut=cut, nev=np.full(300, 3, np.int64)))
    return out


def all_cases():
    """every case a device call can take together with the others (the k - 1 refusal refuses its whole call)"""
    return scan_cases() + window_cases() + lower_bound_cases() + alignment_cases() + emit_cases() + row_cases() + refusal_cases()[:1]


def check_claims(built):
    """-> [(name, claim, holds)] for every case"""
    return [(b.case.name, b.case.claim, bool(b.case.check(view(b)))) for b in built]
