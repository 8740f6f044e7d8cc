"""Plain-Python restatement of methylation-aware candidate screening (`nanopolish variants -q ...`) — test infrastructure, the
checker of nph_screen_load_methylation (csrc/variants.cu).

Follows score_variant_thresholded (src/common/nanopolish_variant.cpp:765-799) with opt::methylation_types non-empty:
  generate_methylated_alternatives   nanopolish_variant.cpp:158-178 (a methylated copy per type where methylate changes the string)
  profile_hmm_score_set              src/hmm/nanopolish_profile_hmm.cpp:32-56 (log(n) penalties, the table log-sum of logsum.h:55-66)
on top of tests/var_restatement.py (candidates, event sequences) and tests/meth_restatement.py (methylate, match_to_site).
Windows may hold N: it ranks 0 in every alphabet, complements like the alphabet's first symbol, and never completes a site.
Pinned: tests/test_variants_methylation_oracle.py runs its qualities against the compiled reference."""
import math

import numpy as np

from nanopolish_b200 import synth
from tests import meth_restatement as mr
from tests import var_restatement as vr

NUC = dict(bases="ACGT", comp="TGCA", sites=[], sites_m=[], sites_mc=[])


def _reverse_complement(a, s):
    """Alphabet::reverse_complement; an unknown symbol complements like bases[0]"""
    rl = len(a["sites"][0]) if a["sites"] else 0
    comp = {b: c for b, c in zip(a["bases"], a["comp"])}
    out = [None] * len(s)
    i, j = 0, len(s) - 1
    while i < len(s):
        hit = None
        for si, site_m in enumerate(a["sites_m"]):
            off, ln, cov = mr.match_to_site(s, i, site_m, rl)
            if ln > 0 and cov:
                hit = (si, off, ln)
                break
        if hit:
            si, off, ln = hit
            for t in range(off, off + ln):
                out[j] = a["sites_mc"][si][t]
                j -= 1
                i += 1
        else:
            out[j] = comp.get(s[i], a["comp"][0])
            j -= 1
            i += 1
    return "".join(out)


def kmer_ranks(a, seq, k, rc):
    """HMMInputSequence(seq, alphabet).get_kmer_rank(i, k, rc) for i = 0..len-k; unknown symbols rank 0"""
    rank = {b: i for i, b in enumerate(a["bases"])}
    rc_seq = _reverse_complement(a, seq)
    A = len(a["bases"])
    out = np.zeros(len(seq) - k + 1, np.uint32)
    for i in range(out.shape[0]):
        km = seq[i:i + k] if not rc else rc_seq[len(seq) - i - k:len(seq) - i]
        r = 0
        for ch in km:
            r = r * A + rank.get(ch, 0)
        out[i] = r
    return out


def alternatives(seq: str, types):
    """generate_methylated_alternatives: [(type index or -1, string)] — the sequence, then its methylated copies in type order"""
    out = [(-1, seq)]
    for t, name in enumerate(types):
        m = mr.methylate(mr.ALPHABETS[name], seq)
        if m != seq:
            out.append((t, m))
    return out


def logsum_table():
    """p7_FLogsumInit's table (src/common/logsum.cpp): log(1 + exp(-i / 1000)) in double, stored as float"""
    return np.array([math.log(1.0 + math.exp(-i / 1000.0)) for i in range(16000)], np.float32)


_TBL = None


def score_set(scores):
    """profile_hmm_score_set's fold of one set's scores (float32: the sequence's first), restated in numpy float32 / float64"""
    global _TBL
    if _TBL is None:
        _TBL = logsum_table()
    pen = math.log(len(scores))
    score = float(np.float32(scores[0])) - pen
    for s in scores[1:]:
        alt = float(np.float32(s)) - pen
        a, b = np.float32(score), np.float32(alt)
        mx = a if a > b else b
        mn = a if a < b else b
        d = np.float32(mx - mn)
        if mn == -np.inf or not (d < np.float32(15.7)):
            score = float(mx)
        else:
            score = float(np.float32(mx + _TBL[int(np.float32(d * np.float32(1000.0)))]))
    return np.float32(score)


def position_scores(port_oracle, rs, models, types, ref: str, region_start: int, positions, records, pairs, flank=10, flags=0, indel_bias=1.0, k=6):
    """For each position i: None where the window leaves the region, else (candidates, event sequences, sets, scores) with
    sets[h] = [(type index or -1, string)] for the base haplotype (h = 0) and each candidate, and scores[read][h] the float32 scores of
    set h in set order.  models = [nucleotide model, model of types[0], ...] as uploaded (model id = index); all positions go to the
    port oracle as one batch."""
    lists = vr.pair_lists(records, pairs)
    n_ref = len(ref)
    out, rows, ranks_list = [], [], []
    for i in positions:
        cs, ce = i - flank, i + 1 + flank
        if cs < region_start or ce > region_start + n_ref - 1:
            out.append(None)
            continue
        window = ref[cs - region_start:ce - region_start + 1]
        seqs = vr.event_sequences(records, pairs, cs, ce, lists)
        cands = vr.candidates(ref, i - region_start)
        haps = [window] + [vr.apply(window, off - (cs - region_start), rseq, aseq) for (_, off, rseq, aseq) in cands]
        sets = [alternatives(h, types) for h in haps]
        flat = [(t, s) for st in sets for (t, s) in st]
        fw = [kmer_ranks(NUC if t < 0 else mr.ALPHABETS[types[t]], s, k, False) for t, s in flat]
        rv = [kmer_ranks(NUC if t < 0 else mr.ALPHABETS[types[t]], s, k, True) for t, s in flat]
        for (r, e1, e2) in seqs:
            rc = int(records[r]["rc"])
            ranks_list += rv if rc else fw
            rows += [(int(records[r]["read"]), 1 + t, e1, e2, rc, flags) for t, _ in flat]
        out.append((cands, seqs, sets, len(flat)))
    sc = np.zeros(0, np.float32)
    if rows:
        jobs = synth._finish_jobs(rows, ranks_list)
        jobs.jobs["stride"] = np.where(jobs.jobs["rc"] == 1, -1, 1)          # EventAlignmentRecord::stride
        sc, _ = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, models, jobs.kmer_ranks, jobs.jobs, indel_bias=indel_bias)
    at = 0
    for n, o in enumerate(out):
        if o is None:
            continue
        cands, seqs, sets, nf = o
        per_read = []
        for _ in seqs:
            row, h0 = [], at
            for st in sets:
                row.append(sc[h0:h0 + len(st)])
                h0 += len(st)
            per_read.append(row)
            at += nf
        out[n] = (cands, seqs, sets, per_read)
    return out


def accumulate(cands, seqs, sets, scores, threshold):
    """score_variant_thresholded's loop over the event sequences in order ->
    (qualities[9] with NaN for candidates the reference does not generate,
     DP rows the loop scores: (n(base) + n(variant)) E for each (candidate, sequence) pair it adds, n = the set's size)"""
    q = [math.nan] * 9
    totals = [0.0] * len(cands)
    rows = 0
    nb = len(sets[0])
    for ri, (r, e1, e2) in enumerate(seqs):
        if all(abs(t) >= threshold for t in totals):
            break
        base = float(score_set(scores[ri][0]))
        for c in range(len(cands)):
            if abs(totals[c]) < threshold:
                totals[c] += float(score_set(scores[ri][1 + c])) - base
                rows += (nb + len(sets[1 + c])) * (abs(e1 - e2) + 1)
    for (slot, _, _, _), t in zip(cands, totals):
        q[slot] = t
    return q, rows


def device_accounting(cands, seqs, sets, scores, threshold, reads_per_round):
    """What the device runs for one position: (jobs, DP rows, rounds, jobs without early exit).  Reads go reads_per_round at a time;
    every read of a round scores the base set and the set of each candidate live at the round's start."""
    totals = [0.0] * len(cands)
    alive = set(range(len(cands))) if seqs else set()
    jobs = rows = rounds = 0
    done = 0
    nb = len(sets[0])
    while alive and done < len(seqs):
        chunk = seqs[done:done + reads_per_round]
        rounds += 1
        for ri, (r, e1, e2) in enumerate(chunk, start=done):
            n = nb + sum(len(sets[1 + c]) for c in alive)
            jobs += n
            rows += n * (abs(e1 - e2) + 1)
            base = float(score_set(scores[ri][0]))
            for c in sorted(alive):
                if abs(totals[c]) < threshold:
                    totals[c] += float(score_set(scores[ri][1 + c])) - base
        done += len(chunk)
        alive = {c for c in alive if abs(totals[c]) < threshold}
    no_exit = len(seqs) * (nb + sum(len(s) for s in sets[1:])) if cands else 0
    return jobs, rows, rounds, no_exit
