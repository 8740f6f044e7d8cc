"""Timing of nph_screen_variants_batch on the two candidate lists of a `variants --consensus` region: the pile-up of
quick_all_support.py (a 50 kb draft region at depth 50, reads of 2 000 bases on both strands, a truth that differs from the draft by
400 homopolymer-length indels), flank 10, threshold 100, HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP.
  round0  the edits nph_screen_edits_batch passes (quality > 0) plus the truth's edits, as round 0 re-screens them
  round1  the truth expanded by expand_variants (min_flanking_sequence 30): each indel, its one-base-longer deletion, four insertions
Reports per list the candidates, windows, rounds, jobs with and without the early exit, the reference's DP rows and their rate, the
kernel time and the whole call, the card's name, power limit and SM clock read in the same run, and — where
oracle/_ref/libnpref_variants.so is built — the compiled reference's own screen_variants_by_score on one CPU thread over the first
candidates of the round-1 list, per candidate.  Prints one JSON line.

  python scripts/quick_screen_variants.py [reps]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from nanopolish_b200 import synth  # noqa: E402
from nanopolish_b200.engine import Engine  # noqa: E402
from tests import screen_cases as sc  # noqa: E402
from tests import screen_restatement as scr  # noqa: E402
from tests.ref_variants import RefVariants  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
model = synth.load_model("nucleotide")
eng = Engine(0)
eng.model_upload(model)

draft, rs, recs, pairs, dur, deltas, first, truth = sc.suc._pileup(("hp", 50_000, 50, 2000, 77, 400, {}), model)
c = dict(draft=draft, rs=rs, recs=recs, pairs=pairs, dur=dur, deltas=deltas, first=first, region_start=sc.REGION_START,
         region_end=sc.REGION_START + len(draft) - 1, region_ref=draft, flank=10, flags=sc.FLAGS, threshold=100, types=(), truth=truth)
c["params"] = sc.params(c)

# round 0: the edit screen's positive edits (slot 2j: substitution to j, 2j + 1: insertion of j, 8: deletion of the base) and the truth
ref = np.frombuffer(draft.encode(), np.uint8).copy()
t0 = time.perf_counter()
q, _, _ = eng.screen_edits_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs,
                                 synth.screen_params(sc.REGION_START, 6, 10, 100, sc.FLAGS, 8))
edit_ms = (time.perf_counter() - t0) * 1e3
round0 = []
for pi, s in zip(*np.nonzero(q > 0)):
    p, b = sc.REGION_START + int(pi), draft[pi]
    if s == 8:
        round0.append((p - 1, draft[pi - 1:pi + 1], draft[pi - 1]))
    else:
        x = "ACGT"[s // 2]
        round0.append((p, b, x) if s % 2 == 0 else (p, b, b + x))
n_edits = len(round0)
round0 += truth
round1 = scr.expand(sc.CONTIG, c["region_start"], c["region_ref"], truth, 30)

row = dict(region_bases=len(draft), depth=50, reads=int(recs.shape[0]), gpu=gpu, edit_screen_ms=edit_ms, edit_screen_positive=n_edits)
for name, cands in (("round0", round0), ("round1", round1)):
    res, cnt = sc.device(eng, c, candidates=cands)                      # warm-up: module load, buffers
    call_ms, kern_ms = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        res, cnt = sc.device(eng, c, candidates=cands)                  # synchronous: returns with the qualities on the host
        call_ms.append((time.perf_counter() - t0) * 1e3)
        kern_ms.append(float(cnt["kernel_ms"]))
    ms = float(np.median(call_ms))
    row[name] = dict(candidates=len(cands), kept=int(((res["quality"] > 0) & (res["status"] != scr.OUTSIDE)).sum()),
                     windows=int(cnt["n_windows"]), rounds=int(cnt["n_rounds"]), jobs=int(cnt["n_jobs"]),
                     jobs_without_exit=int(cnt["n_jobs_without_exit"]), reference_rows=int(cnt["n_reference_rows"]),
                     kernel_ms_median=float(np.median(kern_ms)), call_ms_median=ms, call_ms_min=float(np.min(call_ms)),
                     call_ms_max=float(np.max(call_ms)), reference_rows_per_s=int(cnt["n_reference_rows"]) / (ms / 1e3))
if RefVariants.available():
    refo = RefVariants()
    sub = dict(c, candidates=round1[:60])
    hs, _ = refo.register(sub)
    t0 = time.perf_counter()
    refo.screened(sub, hs)
    secs = time.perf_counter() - t0
    row.update(ref_candidates=60, ref_screen_s_1thread=secs, ref_ms_per_candidate_1thread=secs * 1e3 / 60)
print(json.dumps(row), flush=True)
eng.close()
