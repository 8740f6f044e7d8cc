"""Cases of scorereads --train-transitions: one synthetic read each, its event alignment as model_score receives it, and the
compiled reference's model_score with training (oracle/_ref/libnpref_scorereads.so) next to the restatement
(tests/transition_restatement.py) over the reference's own profile_hmm_align and profile_hmm_score."""
import ctypes as C
import hashlib
import os

import numpy as np

from nanopolish_b200 import synth
from oracle.oracle_py import RefOracle
from tests import transition_restatement as tr

REF_SR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libnpref_scorereads.so")
CONTIG = "ctg"
K = 6
DNA = np.frombuffer(b"ACGT", np.uint8)

# name, n_events, eps, seed, rc, drift, scale, prior, alignment shape
CASES = [
    ("plain", 1600, 200, 1, 0, False, None, False, "truth"),
    ("rc", 1600, 200, 2, 1, False, None, False, "truth"),
    ("drift", 1600, 200, 3, 0, True, None, False, "truth"),
    ("prior", 1600, 200, 4, 0, False, None, True, "truth"),
    ("short_paths", 400, 3, 5, 0, False, None, False, "sparse"),
    ("short_paths4", 400, 4, 9, 0, False, None, False, "sparse"),
    ("wide_scale", 1200, 150, 6, 0, False, 4.0, False, "truth"),
    ("stalled", 1600, 100, 7, 0, False, None, False, "stalled"),
    ("no_segment", 300, 200, 8, 0, False, None, False, "truth"),
]


def build(spec):
    name, n_events, eps, seed, rc, drift, scale, prior, shape = spec
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(1, n_events, model, seed=seed, drift=drift)
    if scale is not None:
        rs.reads[0]["scale"] = scale
    which = rs.ev_kmer[0]
    E = int(rs.reads[0]["n_events"])
    contig = DNA[rs.seq_codes[0]].tobytes().decode()
    ref_pos = [int(w) for w in which]
    if shape == "stalled":
        # a stretch of events on one reference position: the segments inside it fetch <= k bases and are skipped
        ref_pos = [min(p, ref_pos[300]) if 300 <= e < 700 else p for e, p in enumerate(ref_pos)]
    if shape == "sparse":
        # two reference bases per event over the contig taken four times: segments of eps + 1 events fetch 2 * eps + 1 bases, so
        # their paths are a handful of states long
        contig = contig * 4
        ref_pos = [2 * e for e in range(E)]
    align = list(zip(ref_pos, range(E)))
    if rc:
        # a reverse-strand read: the contig is the reverse complement of the bases the events came from, k-mer q of the read sits
        # at contig position nk - 1 - q, and the alignment walks the events backwards (stride -1)
        nk = len(contig) - K + 1
        contig = revcomp(contig)
        align = [(nk - 1 - p, e) for p, e in align][::-1]
    return dict(name=name, rs=rs, model=model, eps=eps, rc=rc, prior=prior, contig=contig, align=align)


def fingerprint(c) -> str:
    h = hashlib.sha256()
    r = c["rs"]
    for a in (r.reads, r.ev_mean, r.ev_start_time, np.array(c["align"], np.int64)):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(repr((c["eps"], c["rc"], c["prior"], c["contig"])).encode())
    return h.hexdigest()[:32]


def revcomp(s: str) -> str:
    return s.translate(str.maketrans("ACGT", "TGCA"))[::-1]


def jobs_of(c, read=0):
    """the device jobs of model_score's segments: (HMM_JOB_DT jobs, base codes, the segments)"""
    segs, _ = tr.segments(c["align"], c["contig"], 0, c["eps"], K)
    rows, codes = [], []
    off = 0
    for e0, e1, seg in segs:
        s = revcomp(seg) if c["rc"] else seg                   # HMMInputSequence's m_rc_seq for rc
        cd = synth.encode(s, "nucleotide")
        rows.append((off, read, 0, e0, e1, len(seg) - K + 1, 1 if e0 <= e1 else -1, c["rc"], 0, 0))
        codes.append(cd)
        off += cd.shape[0]
    jobs = np.array(rows, synth.HMM_JOB_DT) if rows else np.zeros(0, synth.HMM_JOB_DT)
    return jobs, (np.concatenate(codes) if codes else np.zeros(1, np.uint8)), segs


class RefTT(RefOracle):
    """RefOracle over oracle/_ref/libnpref_scorereads.so: its reads, profile_hmm_score / _align, and model_score with training"""

    def __init__(self):
        super().__init__(REF_SR)
        self.lib.npref_model_score_train.restype = C.c_longlong

    @staticmethod
    def available() -> bool:
        return RefOracle.available(REF_SR)

    def model_score(self, c):
        """(score, counts[81], probs[30], print() text) of the reference"""
        self.clear_reads()
        mh = self.builtin_model()
        hs = self.register_reads(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, mh)
        rp = np.array([a for a, _ in c["align"]], np.int32); ei = np.array([b for _, b in c["align"]], np.int32)
        score = C.c_double(); counts = np.zeros(tr.WORDS, np.uint64); probs = np.zeros(tr.BINS); cap = 1 << 16
        text = C.create_string_buffer(cap)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        n = self.lib.npref_model_score_train(int(hs[0]), CONTIG.encode(), c["contig"].encode(), len(c["align"]), p(rp), p(ei), c["rc"], c["eps"],
                                             int(c["prior"]), C.byref(score), p(counts), p(probs), text, C.c_size_t(cap))
        assert n >= 0
        return score.value, counts, probs, text.raw[:n].decode()

    def prior_r9(self):
        out = np.zeros(tr.BINS)
        self.lib.npref_transition_prior_r9(out.ctypes.data_as(C.c_void_p))
        return out

    def restated(self, c, trace=None):
        """(score, counts, paths) by the restatement over the reference's profile_hmm_score and profile_hmm_align"""
        self.clear_reads()
        mh = self.builtin_model()
        hs = self.register_reads(c["rs"].reads, c["rs"].ev_mean, c["rs"].ev_start_time, mh)
        _, _, mean, _, _ = self.model_dump(mh)
        r = c["rs"].reads[0]
        scale, shift = float(r["scale"]), float(r["shift"])
        segs, _ = tr.segments(c["align"], c["contig"], 0, c["eps"], K)
        counts = np.zeros(tr.WORDS, np.uint64)
        total, nev, paths = 0.0, 0, []
        for e0, e1, seg in segs:
            jb = np.zeros(1, synth.HMM_JOB_DT)
            jb[0]["event_start"], jb[0]["event_stop"], jb[0]["rc"] = e0, e1, c["rc"]
            total += float(self.score_batch(hs, jb, [seg.encode()], [mh])[0][0])
            nev += abs(e0 - e1) + 1
            ek, _, st = self.align(hs[0], mh, seg.encode(), e0, e1, c["rc"], 0)
            path = [(int(e), int(k), chr(s)) for (e, k), s in zip(ek, st)]
            paths.append(path)
            ranks = np.zeros(len(seg) - K + 1, np.uint32)
            self.lib.npref_kmer_ranks(mh, seg.encode(), c["rc"], ranks.ctypes.data_as(C.c_void_p))
            tr.add_training(counts, path, ranks, lambda rk: tr.scaled_mean(float(mean[rk]), scale, shift), trace=trace)
        return (total / nev if nev else 1.0), counts, paths
