"""--fix-homopolymers test cases and the three ways to run them — test infrastructure.

A case is a seeded pile-up of synth.gen_hp_pileup (reads from a truth that differs from the draft by homopolymer-length indels,
event durations from the reference's gamma model) plus a haplotype over the draft (the draft with some variants applied) and
min_flanking_sequence.  Its answers come from
  ref_fixed     the compiled reference's own fix_homopolymers (tests/ref_variants.py: oracle/_ref/libnpref_variants.so)
  restated      tests/hp_restatement.py over the compiled reference's profile_hmm_score / profile_hmm_align (the same library)
  device        nph_homopolymer_likelihoods_batch for the restatement's windows."""
import ctypes as C
import hashlib
import os

import numpy as np

from nanopolish_b200 import synth
from tests import hp_restatement as hr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONTIG = "ctg"
REGION_START = 5000

# (name, pile-up (ref_len, depth, read_bases, seed, hp errors, planted long runs), haplotype variants (draft offset, ref, alt), or
# "inserts" / "moved" for the lists _inserts / _moved build, min_flanking_sequence, duration scale, extras).  extras:
#   plant          (draft index, length) runs written into the draft (synth.gen_hp_pileup)
#   region_trim    (a, b): the AlignmentDB region is the draft without its first a and last b bases (the haplotype keeps them all)
#   sparse_steps   per step s one more record, of the read with the most events, whose aligned events advance one event every s
#                  bases over the whole draft: windows of 9, 10 and 11 events
#   dense_at       (draft index, bases, events per base): one more record whose events advance that fast over that stretch, so
#                  windows inside it fail the event/bp ratio test
#   equal_times    a read whose events all start at one time: local_avg 0, rate inf, a NaN duration term, every score NaN,
#                  call npos and a NaN quality
F_EDGE, N_EDGE, TRIM = 10, 800, 6
EDGE_RUNS = ((100, 10), (150, 9), (200, 2), (250, 3))
CASES = [
    ("plain", (700, 12, 260, 3, 5, 0), [], 30, 1.0, {}),
    ("flank7", (500, 10, 200, 5, 4, 0), [], 7, 1.0, {}),
    ("short_durations", (500, 10, 200, 8, 4, 0), [], 12, 1e-4, {}),
    ("inserted_flanks", (700, 12, 260, 11, 5, 0), "inserts", 20, 1.0, {}),
    ("long_runs", (600, 20, 240, 21, 6, 6), [], 20, 1.0, {}),
    # inserted and substituted bases exactly at the calling-range ends of the runs the truth changes, and a same-letter substitution
    # on the first base of some of them (no reference position: the insertion / deletion is tried further along)
    ("moved", (900, 14, 300, 31, 8, 0), "moved", 15, 1.0, {}),
    # every test of the scan on both sides of its limit: runs of 10, 9, 2 and 3; a run one base short of the lower flank and one
    # base short of the upper flank; a calling range one base outside the trimmed region at either end
    ("edges_out", (N_EDGE, 10, 400, 41, 4, 0), [], F_EDGE, 1.0,
     dict(plant=((F_EDGE - 1, 3), (F_EDGE + TRIM - 1, 3)) + EDGE_RUNS + ((N_EDGE - F_EDGE - 3, 3), (N_EDGE - 1 - TRIM - F_EDGE - 3, 3)),
          region_trim=(TRIM, TRIM), sparse_steps=(3, 2.4, 2))),
    # ... and exactly at each limit; plus sparse, dense and equal-time reads
    ("edges_in", (N_EDGE, 10, 400, 42, 4, 0), [], F_EDGE, 1.0,
     dict(plant=((F_EDGE, 3), (F_EDGE + TRIM, 3)) + EDGE_RUNS + ((N_EDGE - 1 - F_EDGE - 3, 3), (N_EDGE - 2 - TRIM - F_EDGE - 3, 3)),
          region_trim=(TRIM, TRIM), sparse_steps=(3, 2.4, 2), dense_at=(236, 32, 21), equal_times=1)),
]


def _inserts(draft: str):
    """variants whose inserted bases sit at the calling-range ends of some homopolymers (the enclosing range moves over them)
    and one that deletes a run's neighbour"""
    out, i = [], 60
    while i < len(draft) - 60 and len(out) < 8:
        out.append((i, draft[i], draft[i] + "AC"[len(out) % 2]))      # insertion after base i
        out.append((i + 17, draft[i + 17], "ACGT"[("ACGT".index(draft[i + 17]) + 1) % 4]))   # substitution: no reference position
        i += 83
    return out


def _moved(draft: str, edits, flank: int):
    """for the runs the truth changes: bases without a reference position at both calling-range ends — alternately a substitution
    at hap_hp_start - flank and hap_hp_end + flank, and an insertion behind hap_hp_start - flank - 1 (its two bases have none) with
    a substitution at hap_hp_end + flank — and a same-letter substitution on the first base of every other run; positions in
    draft coordinates, no two variants within two bases of each other"""
    other = lambda c: "ACGT"[("ACGT".index(c) + 2) % 4]
    out, used = [], set()
    for q, (s, n, _) in enumerate(edits):
        e = s + n
        if q % 2 == 0:
            vs = [(s - flank, draft[s - flank], other(draft[s - flank])), (e + flank, draft[e + flank], other(draft[e + flank]))]
        else:
            vs = [(s - flank, draft[s - flank], draft[s - flank] + other(draft[s - flank])),
                  (e + flank, draft[e + flank], other(draft[e + flank]))]
        if q % 4 < 2:
            vs.append((s, draft[s], draft[s]))
        if any(abs(o - u) <= 2 for o, _, _ in vs for u in used):
            continue
        used.update(o for o, _, _ in vs)
        out += vs
    return sorted(out)


def _extra_records(recs, pairs, rs, n_draft, ex):
    """the records of sparse_steps and dense_at, appended (record order: after the pile-up's)"""
    r = int(np.argmax(rs.reads["n_events"]))
    add = []
    for step in ex.get("sparse_steps", ()):
        p = np.arange(20, n_draft - 20)
        add.append((((p - 20) / step).astype(np.int64), p))
    if "dense_at" in ex:
        at, n, rate = ex["dense_at"]
        p = np.arange(at, at + n)
        add.append(((p - at) * rate, p))
    for ev, p in add:
        assert ev.max() < int(rs.reads[r]["n_events"])
        pr = np.zeros(p.shape[0], synth.PAIR_DT)
        pr["ref_pos"], pr["read_pos"] = REGION_START + p, ev
        rec = np.zeros(1, synth.METH_RECORD_DT)
        rec[0] = (int(recs["ref_off"][-1]) + int(recs["ref_len"][-1]), pairs.shape[0], r, 0, int(p[-1] - p[0]) + 1, p.shape[0],
                  REGION_START + int(p[0]), 0, 0, (0, 0))
        recs, pairs = np.concatenate([recs, rec]), np.concatenate([pairs, pr])
    return recs, pairs


def build(spec):
    name, (ref_len, depth, read_bases, seed, n_err, long_runs), hv, min_flank, dscale, ex = spec
    model = synth.load_model("nucleotide")
    ref, rs, recs, pairs, dur, edits = synth.gen_hp_pileup(ref_len, depth, read_bases, model, seed=seed, region_start=REGION_START, n_hp_errors=n_err,
                                                           long_runs=long_runs, plant=ex.get("plant", ()))
    dur = (dur * np.float32(dscale)).astype(np.float32)
    draft = bytes(b"ACGT"[c] for c in ref).decode()
    variants = _inserts(draft) if hv == "inserts" else _moved(draft, edits, min_flank) if hv == "moved" else list(hv)
    recs, pairs = _extra_records(recs, pairs, rs, len(draft), ex)
    if "equal_times" in ex:
        R = rs.reads[ex["equal_times"]]
        o, n = int(R["event_off"]), int(R["n_events"])
        rs.ev_start_time[o:o + n] = rs.ev_start_time[o]
    deltas, first = synth.compact_event_alignment(recs, pairs, int(recs["ref_len"].sum()))
    hap = hr.Haplotype(REGION_START, draft)
    for off, r, a in variants:
        assert hap.apply_variant(REGION_START + off, r, a)
    trim = ex.get("region_trim", (0, 0))
    region_start, region_end = REGION_START + trim[0], REGION_START + len(draft) - 1 - trim[1]
    trace = []
    wins = hr.windows(hap, region_start, region_end, min_flank, trace)
    seqs, warr = hr.window_array(wins)
    params = np.zeros(1, synth.HP_PARAMS_DT)
    params[0] = (region_start, min_flank, 0, 0)
    return dict(name=name, model=model, draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, edits=edits, deltas=deltas, first=first,
                variants=variants, hap=hap, region_start=region_start, region_end=region_end, region_ref=draft[trim[0]:len(draft) - trim[1]],
                min_flank=min_flank, wins=wins, scan_trace=trace, seqs=seqs, warr=warr, params=params)


def fingerprint(c) -> str:
    h = hashlib.sha256()
    for a in (c["rs"].ev_mean, c["rs"].ev_start_time, c["dur"], c["recs"], c["pairs"], c["seqs"], c["warr"]):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["draft"], c["variants"], c["min_flank"], c["region_start"], c["region_end"])).encode())
    return h.hexdigest()


def ref_restated(ref, c, hs, mh):
    """per window (total_reads, e_lik, d_lik) over the HMMs of `ref` (a tests/ref_variants.py RefVariants holding the case's reads
    as registered: hs, mh), and the fixed text"""
    recs, rs = c["recs"], c["rs"]
    rec_reads = rs.reads[recs["read"]]

    def job(seq, r, e1, e2):
        jb = np.zeros(1, synth.HMM_JOB_DT)
        jb[0]["read"], jb[0]["event_start"], jb[0]["event_stop"], jb[0]["rc"] = int(recs[r]["read"]), e1, e2, int(recs[r]["rc"])
        return jb

    score = lambda seq, r, e1, e2: ref.score_batch(hs, job(seq, r, e1, e2), [seq.encode()], [mh])[0][0]

    def align(seq, r, e1, e2):
        ek, _, st = ref.align(hs[int(recs[r]["read"])], mh, seq.encode(), e1, e2, int(recs[r]["rc"]), 0)
        return [(int(e), int(k), chr(s)) for (e, k), s in zip(ek, st)]

    vectors = []
    for w in c["wins"]:
        seqs = hr.event_sequences(recs, c["pairs"], w["rcs"], w["rce"])
        e, d = hr.likelihoods(w, seqs, rec_reads, rs.ev_start_time, c["dur"], score, align)
        vectors.append((len(seqs), e, d))
    fixed = hr.fix_homopolymers(c["hap"], c["wins"], vectors)
    return vectors, hr.fixed_text(fixed, len(c["variants"]))


def event_edges(c):
    """per window the event sequences (record, e1, e2) and the ones the ratio test drops, over the case's records"""
    seqs, dropped = [], []
    for w in c["wins"]:
        seqs.append(hr.event_sequences(c["recs"], c["pairs"], w["rcs"], w["rce"]))
        dropped.append(hr.event_sequences(c["recs"], c["pairs"], w["rcs"], w["rce"], max_ratio=float("inf")))
    return seqs, [len(b) - len(a) for a, b in zip(seqs, dropped)]


def device(eng, c, max_chunk_pairs: int = 0):
    rs = c["rs"]
    params = c["params"].copy()
    params[0]["max_chunk_pairs"] = max_chunk_pairs
    ref_bases = np.frombuffer(c["region_ref"].encode(), np.uint8).copy()
    return eng.homopolymer_likelihoods_batch(rs.reads, rs.ev_mean, rs.ev_start_time, c["dur"], ref_bases, c["deltas"], c["first"], c["recs"],
                                             params, c["seqs"], c["warr"])


def vectors_of(liks):
    return [(int(x["total_reads"]), [float(v) for v in x["event_lik"]], [float(v) for v in x["duration_lik"]]) for x in liks]


def _cstrs(xs):
    return (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])


def mirror(host, c, indel_bias=1.0) -> str:
    """nph::fix_homopolymers through the nphh_fix_homopolymers shim (the device call): the fixed text"""
    from tests.test_host_mirror import _register, _register_reads
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    host.nphh_clear()
    rs = c["rs"]
    mh = _register(host, c["model"])
    hs = _register_reads(host, rs, mh)
    for i, r in enumerate(rs.reads):
        o, n = int(r["event_off"]), int(r["n_events"])
        host.nphh_read_set_durations(hs[i], p(np.ascontiguousarray(c["dur"][o:o + n])))
    recs, pairs = c["recs"], c["pairs"]
    read = np.array([hs[int(x)] for x in recs["read"]], np.int32)
    rc = np.ascontiguousarray(recs["rc"], np.uint8)
    pp = np.ascontiguousarray(np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32))
    po = np.zeros(recs.shape[0] + 1, np.uint64)
    po[:-1] = recs["pair_off"]; po[-1] = pairs.shape[0]
    assert (po[1:-1] == po[:-2] + recs["n_pairs"][:-1]).all()
    vp = np.array([REGION_START + o for o, _, _ in c["variants"]] or [0], np.int32)
    out = C.create_string_buffer(1 << 20)
    host.nphh_fix_homopolymers.restype = C.c_longlong
    n = host.nphh_fix_homopolymers(CONTIG.encode(), c["region_start"], c["region_ref"].encode(), int(recs.shape[0]), p(read), p(rc), p(pp), p(po),
                                   REGION_START, c["draft"].encode(), len(c["variants"]), p(vp), _cstrs([r for _, r, _ in c["variants"]]),
                                   _cstrs([a for _, _, a in c["variants"]]), c["min_flank"], C.c_double(indel_bias), out, C.c_size_t(1 << 20))
    assert n >= 0, (n, host.nphh_last_error())
    return out.raw[:n].decode()


def ranges(lib, entry: str, hap_ref: str, variants, start, end, lo, hi):
    """(position, sequence, (hap_lower, hap_upper, ref_lower, ref_upper)) of substr_by_reference / the enclosing range, through
    npref_haplotype_ranges (the compiled reference) or nphh_haplotype_ranges (the mirror)"""
    fn = getattr(lib, entry)
    fn.restype = C.c_longlong
    vp = np.array([REGION_START + o for o, _, _ in variants] or [0], np.int32)
    rng = np.zeros(4, np.int64)
    out = C.create_string_buffer(1 << 16)
    n = fn(REGION_START, hap_ref.encode(), len(variants), vp.ctypes.data_as(C.c_void_p), _cstrs([r for _, r, _ in variants]),
           _cstrs([a for _, _, a in variants]), C.c_longlong(start), C.c_longlong(end), C.c_longlong(lo), C.c_longlong(hi),
           rng.ctypes.data_as(C.c_void_p), out, C.c_size_t(1 << 16))
    return int(n), out.value.decode(), tuple(int(x) for x in rng)
