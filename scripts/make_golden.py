#!/usr/bin/env python
"""Generate tests/golden/ from the COMPILED REFERENCE (oracle/_ref/libnpref.so).

Run in the build container (where /root/reference exists):  python scripts/make_golden.py
Outputs (small, committed):
  tests/golden/r9.4_450bps.{nucleotide,cpg}.6mer.template.npz  pore-model tables dumped from the
      reference's PoreModelSet (k, level_mean, level_stdv, level_log_stdv as float64)
  tests/golden/r9.4_450bps.{dam,dcm}.6mer.template.npz  the same for `variants -q dam,dcm`
      [python scripts/make_golden.py models dam dcm: writes only the models named]
  tests/golden/hmm_golden.npz   inputs (seeds + job lists) and the reference's profile_hmm_score floats
  tests/golden/abea_golden.npz  inputs (seeds) and the reference's AlignedPair lists / verdicts
  tests/golden/eventalign_golden.npz  the reference's align_read_to_ref + emit_event_alignment_tsv output (TSV bytes,
      event CIGAR) for the seeded cases of tests/eventalign_cases.py        [python scripts/make_golden.py eventalign]
The GPU box has no /root/reference, so the -m gpu tests compare against these files and against the
plain-C oracle (which tests/test_oracle_vs_ref.py pins to the compiled reference bit-for-bit here).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle_py import RefOracle, build  # noqa: E402
from nanopolish_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def dump_models(ref, alphabets=("nucleotide", "cpg")):
    for alphabet in alphabets:
        h = ref.builtin_model(alphabet)
        k, a, mean, sd, lsd = ref.model_dump(h)
        np.savez_compressed(os.path.join(GOLD, f"r9.4_450bps.{alphabet}.6mer.template.npz"),
                            k=np.int32(k), alphabet_size=np.int32(a), level_mean=mean, level_stdv=sd,
                            level_log_stdv=lsd)
        print("model", alphabet, k, a, mean.shape)


def eventalign_golden(ref):
    from tests import eventalign_cases as EC
    model, rs, cases = EC.build_cases()
    ref.clear_reads()
    mh = ref.builtin_model("nucleotide")
    rh = ref.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, mh)
    out = {}
    for c in cases:
        slot, r = EC.read_slot(c, rs.n_reads), c["read"]
        ref.read_set_eventalign(rh[slot], r.name, r.read_sequence, r.b2e_start, c["b2e_stop"], r.stdv, r.duration)
        single_segment = not any((int(x) & 15) == 3 for x in c["cigar"])
        tsv, cigar, ea = ref.eventalign(rh[slot], c["contig_name"], c["contig"], c["ref_pos"], c["flag"], c["cigar"], c["read_idx"],
                                        c["region"], want_cigar=single_segment)
        out[f"tsv_{c['read_idx']}"] = np.frombuffer(tsv.encode(), np.uint8)
        out[f"cigar_{c['read_idx']}"] = np.frombuffer(cigar.encode(), np.uint8)
        print("eventalign", c["read_idx"], "flag", c["flag"], tsv.count("\n"), "rows", cigar[:40])
    np.savez_compressed(os.path.join(GOLD, "eventalign_golden.npz"), **out)


def main():
    os.makedirs(GOLD, exist_ok=True)
    build(ref=True)
    ref = RefOracle()
    if sys.argv[1:] == ["eventalign"]:
        eventalign_golden(ref)
        return
    if sys.argv[1:2] == ["models"]:
        dump_models(ref, sys.argv[2:])
        return
    dump_models(ref)
    from tests.golden_cases import make_hmm_cases, make_abea_cases   # shared with the tests
    # ---- HMM golden vectors
    out = {}
    for name, case in make_hmm_cases().items():
        ref.clear_reads()
        handles = [ref.builtin_model(a) for a in case["alphabets"]]
        rh = ref.register_reads(case["rs"].reads, case["rs"].ev_mean, case["rs"].ev_start_time, handles[0])
        scores, _ = ref.score_batch(rh, case["jobs"].jobs, case["jobs"].seqs, handles, indel_bias=case["indel_bias"])
        out[name] = scores
        print("hmm", name, scores.shape, scores[:3])
    np.savez_compressed(os.path.join(GOLD, "hmm_golden.npz"), **out)
    # ---- ABEA golden vectors
    out = {}
    for name, case in make_abea_cases().items():
        ref.clear_reads()
        h = ref.builtin_model("nucleotide")
        rs = case["rs"]
        rh = ref.register_reads(rs.reads, rs.ev_mean, rs.ev_start_time, h)
        seqs = [synth._CODE2DNA[c].tobytes() for c in rs.seq_codes]
        caps = [int(r["n_events"]) + len(s) for r, s in zip(rs.reads, seqs)]
        pairs, poff, npairs, _ = ref.abea_batch(rh, h, seqs, caps)
        flat = np.concatenate([pairs[int(poff[i]):int(poff[i]) + int(npairs[i])] for i in range(len(seqs))]) \
            if npairs.sum() else np.zeros((0, 2), np.int32)
        out[name + "_pairs"] = flat
        out[name + "_npairs"] = npairs
        print("abea", name, npairs)
    np.savez_compressed(os.path.join(GOLD, "abea_golden.npz"), **out)
    eventalign_golden(ref)


if __name__ == "__main__":
    main()
