"""Python driver over the C ABI (include/nph.h) — used by tests/, bench.py and smoke().

The product is libnph.so; this wrapper only marshals numpy buffers (structured arrays with the
layouts in synth.py) into the C calls.  It never computes a score itself and has no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .synth import CALL_COUNTS_DT, CALL_GROUP_DT, CALL_GROUP_RESULT_DT, CALL_HAPLOTYPE_DT, CALL_VARIANT_RESULT_DT, ABEA_RES_DT, ALIGN_STATE_DT, CALIBRATION_DT, EVENT_DT, EVENT_RANGE_DT, METH_SITE_DT, METHFREQ_PARAMS_DT, HP_COUNTS_DT, HP_LIK_DT, HP_WINDOW_DT, PAIR_DT, PHASE_CALL_DT, PHASE_VARIANT_DT, POLYA_RES_DT, POLYI_RES_DT, RAW_RANGE_DT, SCREEN_CANDIDATE_DT, SCREEN_LIST_COUNTS_DT, SCREEN_RESULT_DT, SUPPORT_COUNTS_DT, SUPPORT_RESULT_DT, SUPPORT_VARIANT_DT


def _p(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    """One nph_ctx (one device, one stream)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = _lib.load()
        self.ctx = C.c_void_p()
        if stream is None:
            rc = self.lib.nph_create(C.byref(self.ctx), device)
        else:
            rc = self.lib.nph_create_on_stream(C.byref(self.ctx), device, C.c_void_p(stream))
        if rc != 0:
            raise _lib.NphError(rc, "nph_create", self.lib.nph_strerror(rc).decode())
        self.n_jobs = 0

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise _lib.NphError(rc, what, self.lib.nph_strerror(rc).decode() + " / " +
                                self.lib.nph_last_error(self.ctx).decode())

    def close(self):
        if self.ctx:
            self.lib.nph_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- call-methylation: enumeration + scoring on the device (include/nph.h, section N3) ----
    @staticmethod
    def meth_sites_cap(records, params) -> int:
        return int((records["ref_len"].astype(np.int64) // (int(params[0]["min_separation"]) + 1) + 2).sum())

    def methylation_batch(self, reads, ev_mean, ev_start_time, ref_bases, pairs, records, params, indel_bias: float = 1.0, out=None):
        """nph_methylation_batch: returns (site_off u8[n_records + 1], sites METH_SITE_DT[n_sites], scored_events)."""
        n = int(records.shape[0])
        cap = self.meth_sites_cap(records, params)
        site_off, sites = out if out is not None else (np.zeros(n + 1, np.uint64), np.zeros(max(cap, 1), METH_SITE_DT))
        scored = C.c_uint64()
        self._check(self.lib.nph_methylation_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                   _p(ref_bases), ref_bases.shape[0], _p(pairs), pairs.shape[0], _p(records), n, _p(params),
                                                   indel_bias, _p(site_off), _p(sites), sites.shape[0], C.byref(scored)), "nph_methylation_batch")
        return site_off, sites[:int(site_off[n])], int(scored.value)

    def methylation_batch_compact(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, params, indel_bias: float = 1.0, out=None):
        """nph_methylation_batch_compact (event alignments as int16 deltas per reference base)"""
        n = int(records.shape[0])
        cap = self.meth_sites_cap(records, params)
        site_off, sites = out if out is not None else (np.zeros(n + 1, np.uint64), np.zeros(max(cap, 1), METH_SITE_DT))
        scored = C.c_uint64()
        self._check(self.lib.nph_methylation_batch_compact(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                           _p(ref_bases), _p(deltas), ref_bases.shape[0], _p(first_event), _p(records), n, _p(params),
                                                           indel_bias, _p(site_off), _p(sites), sites.shape[0], C.byref(scored)), "nph_methylation_batch_compact")
        return site_off, sites[:int(site_off[n])], int(scored.value)

    # ---- phase-reads: SNP calls and qualities of a record batch (include/nph.h, nph_phase_reads_batch) ----
    def phase_reads_batch(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, variants, var_range,
                          indel_bias: float = 1.0, calls_cap: int | None = None):
        """nph_phase_reads_batch: records METH_RECORD_DT (compact event alignments), variants PHASE_VARIANT_DT, var_range u4[n_records, 2].
        Returns (call_off u8[n_records + 1], calls PHASE_CALL_DT[n_calls], scored_events).  calls_cap defaults to the sum of the ranges."""
        assert variants.dtype == PHASE_VARIANT_DT
        n = int(records.shape[0])
        var_range = np.ascontiguousarray(var_range, np.uint32)
        if calls_cap is None:
            calls_cap = int((var_range.reshape(-1, 2)[:, 1].astype(np.int64) - var_range.reshape(-1, 2)[:, 0]).clip(0).sum()) if n else 0
        call_off = np.zeros(n + 1, np.uint64)
        calls = np.zeros(max(calls_cap, 1), PHASE_CALL_DT)
        scored = C.c_uint64()
        self._check(self.lib.nph_phase_reads_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                   _p(ref_bases), _p(deltas), ref_bases.shape[0], _p(first_event), _p(records), n,
                                                   _p(variants), variants.shape[0], _p(var_range), indel_bias, _p(call_off), _p(calls), calls_cap,
                                                   C.byref(scored)), "nph_phase_reads_batch")
        return call_off, calls[:int(call_off[n])], int(scored.value)

    def methylation_load_compact(self, ref_bases, deltas, first_event, records, params, indel_bias: float = 1.0):
        self._check(self.lib.nph_methylation_load_compact(self.ctx, _p(ref_bases), _p(deltas), ref_bases.shape[0], _p(first_event), _p(records),
                                                          records.shape[0], _p(params), indel_bias), "nph_methylation_load_compact")
        self._meth_n = int(records.shape[0])

    def methylation_load(self, ref_bases, pairs, records, params, indel_bias: float = 1.0):
        self._check(self.lib.nph_methylation_load(self.ctx, _p(ref_bases), ref_bases.shape[0], _p(pairs), pairs.shape[0], _p(records),
                                                  records.shape[0], _p(params), indel_bias), "nph_methylation_load")
        self._meth_n = int(records.shape[0])

    def methylation_run(self):
        self._check(self.lib.nph_methylation_run(self.ctx), "nph_methylation_run")

    def methylation_counts(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self.lib.nph_methylation_counts(self.ctx, C.byref(a), C.byref(b), C.byref(c)), "nph_methylation_counts")
        return int(a.value), int(b.value), int(c.value)

    def methylation_sites_dev(self):
        """(device pointer, n_sites) of the last run's site records (nph_methylation_sites_dev)"""
        ptr, n = C.c_void_p(), C.c_uint64()
        self._check(self.lib.nph_methylation_sites_dev(self.ctx, C.byref(ptr), C.byref(n)), "nph_methylation_sites_dev")
        return int(ptr.value or 0), int(n.value)

    def methylation_tsv(self, contig: str, names: list, is_reverse: np.ndarray, cap: int | None = None) -> bytes:
        """nph_methylation_tsv: the methylation_calls.tsv rows of the last run, formatted on the device."""
        blob = "".join(names).encode()
        off = np.zeros(len(names) + 1, np.uint32)
        off[1:] = np.cumsum([len(n.encode()) for n in names])
        rev = np.ascontiguousarray(is_reverse, np.uint8)
        if cap is None:
            cap = 256 * max(1, self.methylation_counts()[0]) + 4096
        out = np.empty(cap, np.uint8)
        n = C.c_uint64()
        self._check(self.lib.nph_methylation_tsv(self.ctx, contig.encode(), blob, _p(off), _p(rev), _p(out), cap, C.byref(n)), "nph_methylation_tsv")
        return out[:int(n.value)].tobytes()

    def methylation_fetch(self, out=None):
        n_sites = self.methylation_counts()[0]
        site_off, sites = out if out is not None else (np.zeros(self._meth_n + 1, np.uint64), np.zeros(max(n_sites, 1), METH_SITE_DT))
        self._check(self.lib.nph_methylation_fetch(self.ctx, _p(site_off), _p(sites), sites.shape[0]), "nph_methylation_fetch")
        return site_off, sites[:n_sites]

    # ---- call-methylation: per-site methylation frequency on the device (calculate_methylation_frequency.py) ----
    def methylation_frequency_reset(self, call_threshold: float = 2.0, split_groups: bool = False):
        """nph_methfreq_reset: an empty accumulator with the script's -c / -s."""
        p = np.zeros(1, METHFREQ_PARAMS_DT)
        p[0]["call_threshold"], p[0]["split_groups"] = call_threshold, 1 if split_groups else 0
        self._check(self.lib.nph_methfreq_reset(self.ctx, _p(p)), "nph_methfreq_reset")

    def methylation_frequency_add(self, contig_id: int):
        """nph_methfreq_add: fold the rows of the last methylation run under contig_id."""
        self._check(self.lib.nph_methfreq_add(self.ctx, contig_id), "nph_methfreq_add")

    def methylation_frequency_counts(self):
        """(distinct keys, calls counted, rows skipped by the threshold)"""
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self.lib.nph_methfreq_counts(self.ctx, C.byref(a), C.byref(b), C.byref(c)), "nph_methfreq_counts")
        return int(a.value), int(b.value), int(c.value)

    def methylation_frequency_tsv(self, contigs: list, cap: int | None = None) -> bytes:
        """nph_methfreq_tsv: the frequency table so far; contigs[i] is the name of contig id i."""
        blob = np.frombuffer("".join(contigs).encode() or b"\0", np.uint8)
        off = np.zeros(len(contigs) + 1, np.uint32)
        off[1:] = np.cumsum([len(c.encode()) for c in contigs])
        n = C.c_uint64()
        if cap is None:              # a guess, then the size the call reports when the guess was short
            cap = 4096 + (256 + max((len(c.encode()) for c in contigs), default=0)) * self.methylation_frequency_counts()[0]
            out = np.empty(cap, np.uint8)
            if self.lib.nph_methfreq_tsv(self.ctx, _p(blob), _p(off), len(contigs), _p(out), cap, C.byref(n)) == 0:
                return out[:int(n.value)].tobytes()
            cap = max(cap, int(n.value))
        out = np.empty(max(cap, 1), np.uint8)
        self._check(self.lib.nph_methfreq_tsv(self.ctx, _p(blob), _p(off), len(contigs), _p(out), cap, C.byref(n)), "nph_methfreq_tsv")
        return out[:int(n.value)].tobytes()

    # ---- variants: candidate screening on the device (include/nph.h, section N2) ----
    def screen_edits_batch(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, params, indel_bias: float = 1.0,
                           methylation=None):
        """nph_screen_edits_batch: returns (qualities f8[n_pos, 9], n_reads u4[n_pos], scored_events).  methylation = (SCREEN_METH_DT[1],
        alt_model_ids u4[n_records, n_types]): nph_screen_edits_batch_methylation (`variants -q ...`)."""
        n_pos = int(ref_bases.shape[0]) - 1
        q = np.zeros((n_pos, 9), np.float64); nr = np.zeros(n_pos, np.uint32)
        scored = C.c_uint64()
        head = (self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0], _p(ref_bases), ref_bases.shape[0],
                _p(deltas), deltas.shape[0], _p(first_event), _p(records), records.shape[0], _p(params), indel_bias)
        if methylation is None:
            self._check(self.lib.nph_screen_edits_batch(*head, _p(q), _p(nr), C.byref(scored)), "nph_screen_edits_batch")
        else:
            meth, ids = methylation[0], np.ascontiguousarray(methylation[1], np.uint32)
            self._check(self.lib.nph_screen_edits_batch_methylation(*head, _p(meth), _p(ids), _p(q), _p(nr), C.byref(scored)),
                        "nph_screen_edits_batch_methylation")
        return q, nr, int(scored.value)

    # ---- variants --fix-homopolymers: length likelihoods of every calling window (include/nph.h, nph_homopolymer_likelihoods_batch) ----
    def homopolymer_likelihoods_batch(self, reads, ev_mean, ev_start_time, ev_duration, ref_bases, deltas, first_event, records, params,
                                      calling_seqs, windows, indel_bias: float = 1.0):
        """records METH_RECORD_DT (compact event alignments, as screening's), params HP_PARAMS_DT[1], calling_seqs u1, windows
        HP_WINDOW_DT.  Returns (HP_LIK_DT[n_windows], HP_COUNTS_DT scalar)."""
        assert windows.dtype == HP_WINDOW_DT
        out = np.zeros(max(windows.shape[0], 1), HP_LIK_DT)
        cnt = np.zeros(1, HP_COUNTS_DT)
        self._check(self.lib.nph_homopolymer_likelihoods_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), _p(ev_duration),
                                                               ev_mean.shape[0], _p(ref_bases), ref_bases.shape[0], _p(deltas), deltas.shape[0],
                                                               _p(first_event), _p(records), records.shape[0], _p(params), _p(calling_seqs),
                                                               calling_seqs.shape[0], _p(windows), windows.shape[0], indel_bias, _p(out), _p(cnt)),
                    "nph_homopolymer_likelihoods_batch")
        return out[:windows.shape[0]], cnt[0]

    # ---- variants --calculate-all-support: A/C/G/T read support of every variant (include/nph.h, nph_all_support_batch) ----
    def all_support_batch(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, params, ref_seqs, variants,
                          indel_bias: float = 1.0):
        """records METH_RECORD_DT (compact event alignments, as screening's), params SUPPORT_PARAMS_DT[1], ref_seqs u1, variants
        SUPPORT_VARIANT_DT.  Returns (SUPPORT_RESULT_DT[n_variants], SUPPORT_COUNTS_DT scalar)."""
        assert variants.dtype == SUPPORT_VARIANT_DT
        out = np.zeros(max(variants.shape[0], 1), SUPPORT_RESULT_DT)
        cnt = np.zeros(1, SUPPORT_COUNTS_DT)
        self._check(self.lib.nph_all_support_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                   _p(ref_bases), ref_bases.shape[0], _p(deltas), deltas.shape[0], _p(first_event), _p(records),
                                                   records.shape[0], _p(params), _p(ref_seqs), ref_seqs.shape[0], _p(variants), variants.shape[0],
                                                   indel_bias, _p(out), _p(cnt)),
                    "nph_all_support_batch")
        return out[:variants.shape[0]], cnt[0]

    # ---- screen_variants_by_score on a candidate list (include/nph.h, nph_screen_variants_batch) ----
    def screen_variants_batch(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, params, alleles, candidates,
                              indel_bias: float = 1.0, methylation=None):
        """records METH_RECORD_DT (compact event alignments, as screening's), params SCREEN_LIST_PARAMS_DT[1], alleles u1, candidates
        SCREEN_CANDIDATE_DT, methylation None or (SCREEN_METH_DT[1], alt model ids n_records x n_types).  Returns
        (SCREEN_RESULT_DT[n_candidates], SCREEN_LIST_COUNTS_DT scalar)."""
        assert candidates.dtype == SCREEN_CANDIDATE_DT
        out = np.zeros(max(candidates.shape[0], 1), SCREEN_RESULT_DT)
        cnt = np.zeros(1, SCREEN_LIST_COUNTS_DT)
        meth, ids = (None, None) if methylation is None else (methylation[0], np.ascontiguousarray(methylation[1], np.uint32))
        self._check(self.lib.nph_screen_variants_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                       _p(ref_bases), ref_bases.shape[0], _p(deltas), deltas.shape[0], _p(first_event), _p(records),
                                                       records.shape[0], _p(params), _p(alleles), alleles.shape[0], _p(candidates),
                                                       candidates.shape[0], indel_bias, _p(meth), _p(ids), _p(out), _p(cnt)),
                    "nph_screen_variants_batch")
        return out[:candidates.shape[0]], cnt[0]

    def call_variant_groups_batch(self, reads, ev_mean, ev_start_time, ref_bases, deltas, first_event, records, key_rank, params, groups,
                                  haplotypes, bases, combination_variants, n_variants: int, indel_bias: float = 1.0, methylation=None):
        """records METH_RECORD_DT (compact event alignments, as screening's), key_rank u4 per read (the rank of its "name:strand"), params
        CALL_PARAMS_DT[1], groups CALL_GROUP_DT, haplotypes CALL_HAPLOTYPE_DT, bases u1, combination_variants u4, methylation None or
        (SCREEN_METH_DT[1], alt model ids n_records x n_types).  Returns (CALL_GROUP_RESULT_DT[n_groups], CALL_VARIANT_RESULT_DT[n_variants],
        CALL_COUNTS_DT scalar)."""
        assert groups.dtype == CALL_GROUP_DT and haplotypes.dtype == CALL_HAPLOTYPE_DT
        gout = np.zeros(max(groups.shape[0], 1), CALL_GROUP_RESULT_DT)
        vout = np.zeros(max(n_variants, 1), CALL_VARIANT_RESULT_DT)
        cnt = np.zeros(1, CALL_COUNTS_DT)
        kr = np.ascontiguousarray(key_rank, np.uint32)
        cv = np.ascontiguousarray(combination_variants, np.uint32)
        meth, ids = (None, None) if methylation is None else (methylation[0], np.ascontiguousarray(methylation[1], np.uint32))
        self._check(self.lib.nph_call_variant_groups_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                           _p(ref_bases), ref_bases.shape[0], _p(deltas), deltas.shape[0], _p(first_event),
                                                           _p(records), records.shape[0], _p(kr), _p(params), _p(groups), groups.shape[0],
                                                           _p(haplotypes), haplotypes.shape[0], _p(bases), bases.shape[0], _p(cv), cv.shape[0],
                                                           n_variants, indel_bias, _p(meth), _p(ids), _p(gout), _p(vout), _p(cnt)),
                    "nph_call_variant_groups_batch")
        return gout[:groups.shape[0]], vout[:n_variants], cnt[0]

    def screen_load(self, ref_bases, deltas, first_event, records, params, indel_bias: float = 1.0, methylation=None):
        head = (self.ctx, _p(ref_bases), ref_bases.shape[0], _p(deltas), deltas.shape[0], _p(first_event), _p(records), records.shape[0], _p(params),
                indel_bias)
        if methylation is None:
            self._check(self.lib.nph_screen_load(*head), "nph_screen_load")
        else:
            meth, ids = methylation[0], np.ascontiguousarray(methylation[1], np.uint32)
            self._check(self.lib.nph_screen_load_methylation(*head, _p(meth), _p(ids)), "nph_screen_load_methylation")
        self._screen_n = int(ref_bases.shape[0]) - 1

    def screen_run(self):
        self._check(self.lib.nph_screen_run(self.ctx), "nph_screen_run")

    def screen_counts(self):
        a, b, c, d, e = C.c_uint32(), C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self.lib.nph_screen_counts(self.ctx, C.byref(a), C.byref(b), C.byref(c), C.byref(d), C.byref(e)), "nph_screen_counts")
        return dict(rounds=int(a.value), jobs=int(b.value), scored_events=int(c.value), jobs_without_exit=int(d.value), reference_events=int(e.value))

    def screen_fetch(self, with_reference_rows: bool = False):
        q = np.zeros((self._screen_n, 9), np.float64); nr = np.zeros(self._screen_n, np.uint32)
        rows = np.zeros(self._screen_n, np.uint64) if with_reference_rows else None
        self._check(self.lib.nph_screen_fetch(self.ctx, _p(q), _p(nr), _p(rows)), "nph_screen_fetch")
        return (q, nr, rows) if with_reference_rows else (q, nr)

    # ---- models / reads / jobs ----------------------------------------------------------
    def model_upload(self, model) -> int:
        mid = C.c_uint32()
        mean = np.ascontiguousarray(model.level_mean, np.float64)
        sd = np.ascontiguousarray(model.level_stdv, np.float64)
        lsd = np.ascontiguousarray(model.level_log_stdv, np.float64)
        self._check(self.lib.nph_model_upload(self.ctx, _p(mean), _p(sd), _p(lsd), mean.shape[0], model.k,
                                              model.alphabet_size, C.byref(mid)), "nph_model_upload")
        return mid.value

    def reads_load(self, reads, ev_mean, ev_start_time):
        self._check(self.lib.nph_reads_load(self.ctx, _p(reads), reads.shape[0], _p(ev_mean),
                                            _p(ev_start_time), ev_mean.shape[0]), "nph_reads_load")

    def hmm_jobs_load(self, kmer_ranks, jobs, indel_bias: float = 1.0):
        self._check(self.lib.nph_hmm_jobs_load(self.ctx, _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs),
                                               jobs.shape[0], indel_bias), "nph_hmm_jobs_load")
        self.n_jobs = int(jobs.shape[0])

    def hmm_score(self, scores_dev_ptr: int | None = None):
        self._check(self.lib.nph_hmm_score(self.ctx, C.c_void_p(scores_dev_ptr) if scores_dev_ptr else None),
                    "nph_hmm_score")

    def hmm_scores_fetch(self, out: np.ndarray | None = None) -> np.ndarray:
        if out is None:
            out = np.empty(self.n_jobs, np.float32)
        self._check(self.lib.nph_hmm_scores_fetch(self.ctx, _p(out), out.shape[0]), "nph_hmm_scores_fetch")
        return out

    def hmm_score_batch(self, reads, ev_mean, ev_start_time, kmer_ranks, jobs, indel_bias: float = 1.0,
                        out: np.ndarray | None = None) -> np.ndarray:
        """== [profile_hmm_score(seq_j, data_j, flags_j) for j]  through the one-shot C call."""
        if out is None:
            out = np.empty(jobs.shape[0], np.float32)
        self._check(self.lib.nph_hmm_score_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean),
                                                 _p(ev_start_time), ev_mean.shape[0], _p(kmer_ranks),
                                                 kmer_ranks.shape[0], _p(jobs), jobs.shape[0], indel_bias,
                                                 _p(out)), "nph_hmm_score_batch")
        self.n_jobs = int(jobs.shape[0])
        return out

    def hmm_score_batch_seq(self, reads, ev_mean, ev_start_time, seq_codes, jobs, indel_bias: float = 1.0,
                            out: np.ndarray | None = None) -> np.ndarray:
        """the same with base codes instead of k-mer ranks (nph_hmm_score_batch_seq; jobs' rank_off = code offsets)"""
        if out is None:
            out = np.empty(jobs.shape[0], np.float32)
        self._check(self.lib.nph_hmm_score_batch_seq(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                     _p(seq_codes), seq_codes.shape[0], _p(jobs), jobs.shape[0], indel_bias, _p(out)),
                    "nph_hmm_score_batch_seq")
        self.n_jobs = int(jobs.shape[0])
        return out

    def train_transitions_batch(self, reads, ev_mean, ev_start_time, seq_codes, jobs, groups=None, n_groups: int = 2,
                                ignore_edge_length: int = 5, max_chunk_jobs: int = 0, indel_bias: float = 1.0):
        """scorereads --train-transitions (nph_train_transitions_batch): the forward scores of the jobs, TT_COUNTS_DT[n_groups] counts
        of their Viterbi paths, and the number of chunks of Viterbi states; last_tt_ms then holds the device ms of K3 (with its
        state-offset kernel) and of the observation kernel"""
        from .synth import TT_COUNTS_DT, TT_PARAMS_DT
        scores = np.empty(jobs.shape[0], np.float32)
        counts = np.zeros(n_groups, TT_COUNTS_DT)
        params = np.zeros(1, TT_PARAMS_DT)
        params[0] = (n_groups, ignore_edge_length, max_chunk_jobs, 0, 0.0, 0.0)
        g = None if groups is None else np.ascontiguousarray(groups, np.uint8)
        self._check(self.lib.nph_train_transitions_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time), ev_mean.shape[0],
                                                         _p(seq_codes), seq_codes.shape[0], _p(jobs), jobs.shape[0], _p(g), _p(params),
                                                         indel_bias, _p(scores), _p(counts)), "nph_train_transitions_batch")
        self.last_tt_ms = (float(params[0]["viterbi_ms_out"]), float(params[0]["observe_ms_out"]))     # K3 + offsets, observation
        return scores, counts, int(params[0]["n_chunks_out"])

    def hmm_jobs_load_seq(self, seq_codes, jobs, indel_bias: float = 1.0):
        self._check(self.lib.nph_hmm_jobs_load_seq(self.ctx, _p(seq_codes), seq_codes.shape[0], _p(jobs), jobs.shape[0], indel_bias),
                    "nph_hmm_jobs_load_seq")
        self.n_jobs = int(jobs.shape[0])

    def score_set_combine(self, scores: np.ndarray, n_alt: int) -> np.ndarray:
        s = np.ascontiguousarray(scores, np.float32)
        g = s.shape[0] // n_alt
        out = np.empty(g, np.float32)
        self._check(self.lib.nph_score_set_combine(_p(s), g, n_alt, _p(out)), "nph_score_set_combine")
        return out

    # ---- Viterbi alignment (profile_hmm_align) -------------------------------------------
    def hmm_align_batch(self, reads, ev_mean, ev_start_time, kmer_ranks, jobs, indel_bias: float = 1.0):
        """== [profile_hmm_align(seq_j, data_j, flags_j) for j]: list of ALIGN_STATE_DT arrays (empty where the
        reference would assert), plus l_fm of each alignment's final state."""
        n = jobs.shape[0]
        E = np.abs(jobs["event_stop"].astype(np.int64) - jobs["event_start"].astype(np.int64)) + 1
        caps = E + jobs["n_kmers"].astype(np.int64) + 2
        off = np.zeros(n + 1, np.uint64)
        off[1:] = np.cumsum(caps)
        states = np.zeros(int(off[-1]), ALIGN_STATE_DT)
        counts = np.zeros(n, np.uint32)
        scores = np.zeros(n, np.float32)
        self._check(self.lib.nph_hmm_align_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time),
                                                 ev_mean.shape[0], _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs), n,
                                                 indel_bias, _p(states), _p(off), _p(counts), _p(scores)),
                    "nph_hmm_align_batch")
        return [states[int(off[j]):int(off[j]) + int(counts[j])] for j in range(n)], scores

    def hmm_align(self, kmer_ranks, jobs, indel_bias: float = 1.0):
        """hmm_align_batch against the reads a preceding reads_load() left resident (eventalign's chained rounds)."""
        n = jobs.shape[0]
        E = np.abs(jobs["event_stop"].astype(np.int64) - jobs["event_start"].astype(np.int64)) + 1
        off = np.zeros(n + 1, np.uint64)
        off[1:] = np.cumsum(E + jobs["n_kmers"].astype(np.int64) + 2)
        states = np.zeros(int(off[-1]), ALIGN_STATE_DT)
        counts = np.zeros(n, np.uint32)
        scores = np.zeros(n, np.float32)
        self._check(self.lib.nph_hmm_align(self.ctx, _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs), n, indel_bias,
                                           _p(states), _p(off), _p(counts), _p(scores)), "nph_hmm_align")
        return [states[int(off[j]):int(off[j]) + int(counts[j])] for j in range(n)], scores

    def eventalign_chain(self, pairs, event_map_start, ref_ranks_fwd, ref_ranks_rc, chains, indel_bias: float = 1.0, out=None):
        """eventalign's segment chains (align_read_to_ref's per-segment loop) walked on the device against the resident
        reads: returns (records EA_RECORD_DT[sum out_cap], results EA_RESULT_DT[n_chains]); chain c's records are
        records[out_off : out_off + n_records]."""
        from .synth import EA_RECORD_DT, EA_RESULT_DT
        n = chains.shape[0]
        total = int((chains["out_off"] + chains["out_cap"]).max()) if n else 0
        if out is not None:                      # caller-owned (e.g. page-locked) output buffers
            records, results = out
            assert records.shape[0] >= total and results.shape[0] >= n
        else:
            records = np.zeros(total, EA_RECORD_DT)
            results = np.zeros(n, EA_RESULT_DT)
        self._check(self.lib.nph_eventalign_chain(self.ctx, _p(pairs), pairs.shape[0], _p(event_map_start), event_map_start.shape[0],
                                                  _p(ref_ranks_fwd), _p(ref_ranks_rc), ref_ranks_fwd.shape[0], _p(chains), n,
                                                  indel_bias, _p(records), total, _p(results)), "nph_eventalign_chain")
        return records, results

    def eventalign_chain_run(self, pairs, event_map_start, ref_ranks_fwd, ref_ranks_rc, chains, indel_bias: float = 1.0):
        """nph_eventalign_chain_run: the chains walked as eventalign_chain walks them, the records left on the device for
        eventalign_tsv / eventalign_records_fetch.  Returns results EA_RESULT_DT[n_chains]."""
        from .synth import EA_RESULT_DT
        n = chains.shape[0]
        total = int((chains["out_off"] + chains["out_cap"]).max()) if n else 0
        results = np.zeros(n, EA_RESULT_DT)
        self._check(self.lib.nph_eventalign_chain_run(self.ctx, _p(pairs), pairs.shape[0], _p(event_map_start), event_map_start.shape[0],
                                                      _p(ref_ranks_fwd), _p(ref_ranks_rc), ref_ranks_fwd.shape[0], _p(chains), n,
                                                      indel_bias, total, _p(results)), "nph_eventalign_chain_run")
        return results

    def eventalign_records_fetch(self, records_total: int):
        from .synth import EA_RECORD_DT
        records = np.zeros(records_total, EA_RECORD_DT)
        self._check(self.lib.nph_eventalign_records_fetch(self.ctx, _p(records), records_total), "nph_eventalign_records_fetch")
        return records

    def eventalign_tsv(self, inputs: dict, print_read_names=False, scale_events=False, signal_index=False, samples=False,
                       out: np.ndarray | None = None, want_row_off: int = 0):
        """nph_eventalign_tsv: the eventalign.tsv rows of the last eventalign_chain_run, written on the device.  inputs: what
        synth.eventalign_tsv_inputs builds (reads EA_TSV_READ_DT, chain_read, text, ref, rc_ref, ev_mean, ev_stdv, ev_duration,
        ev_start_time, samples).  out: a caller-owned (page-locked) uint8 buffer; without one the call is made twice, the
        first time for the size.  want_row_off: the number of rows, to get their offsets too.  Returns (bytes, read_off u8[n_reads
        + 1], refused u1[n_reads], row_off or None)."""
        class Batch(C.Structure):
            _fields_ = [("reads", C.c_void_p), ("n_reads", C.c_size_t), ("chain_read", C.c_void_p), ("text", C.c_void_p), ("n_text", C.c_size_t),
                        ("ref", C.c_void_p), ("rc_ref", C.c_void_p), ("n_ref", C.c_size_t), ("ev_mean", C.c_void_p), ("ev_stdv", C.c_void_p),
                        ("ev_duration", C.c_void_p), ("ev_start_time", C.c_void_p), ("n_events", C.c_size_t), ("samples", C.c_void_p),
                        ("n_samples", C.c_size_t)]
        i = inputs
        adr = lambda a: a.ctypes.data if a is not None and a.size else None
        b = Batch(adr(i["reads"]), i["reads"].shape[0], adr(i["chain_read"]), adr(i["text"]), i["text"].shape[0], adr(i["ref"]), adr(i["rc_ref"]),
                  i["ref"].shape[0], adr(i["ev_mean"]), adr(i["ev_stdv"]), adr(i["ev_duration"]), adr(i.get("ev_start_time")), i["ev_mean"].shape[0],
                  adr(i.get("samples")), i["samples"].shape[0] if i.get("samples") is not None else 0)
        opt = np.array([print_read_names, scale_events, signal_index, samples], np.uint8)
        nr = i["reads"].shape[0]
        read_off, refused = np.zeros(nr + 1, np.uint64), np.zeros(nr, np.uint8)
        row_off = np.zeros(want_row_off + 1, np.uint64) if want_row_off else None
        n = C.c_uint64(0)

        def call(buf):
            return self.lib.nph_eventalign_tsv(self.ctx, C.byref(b), _p(opt), _p(buf) if buf is not None else None, buf.shape[0] if buf is not None else 0,
                                               _p(row_off) if row_off is not None else None, _p(read_off), _p(refused), C.byref(n))
        if out is None:
            rc = call(None)
            if rc == 0 or n.value == 0:                      # no rows, or an error that is not about room
                self._check(rc, "nph_eventalign_tsv")
                return b"", read_off, refused, row_off
            out = np.empty(n.value, np.uint8)
        self._check(call(out), "nph_eventalign_tsv")
        return out[:n.value].tobytes(), read_off, refused, row_off

    # ---- ABEA ---------------------------------------------------------------------------
    def abea_batch(self, reads, ev_mean, ev_start_time, kmer_ranks, jobs, model_id: int, pairs_total: int):
        pairs = np.zeros(pairs_total, PAIR_DT)
        res = np.zeros(jobs.shape[0], ABEA_RES_DT)
        self._check(self.lib.nph_abea_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), _p(ev_start_time),
                                            ev_mean.shape[0], _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs),
                                            jobs.shape[0], model_id, _p(pairs), pairs_total, _p(res)),
                    "nph_abea_batch")
        return pairs, res

    def abea_jobs_load(self, kmer_ranks, jobs, model_id: int, pairs_total: int):
        self._check(self.lib.nph_abea_jobs_load(self.ctx, _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs),
                                                jobs.shape[0], model_id, pairs_total), "nph_abea_jobs_load")
        self._abea_n = int(jobs.shape[0])
        self._abea_pairs = int(pairs_total)

    def abea_run(self):
        self._check(self.lib.nph_abea_run(self.ctx), "nph_abea_run")

    def abea_fetch(self):
        pairs = np.zeros(self._abea_pairs, PAIR_DT)
        res = np.zeros(self._abea_n, ABEA_RES_DT)
        self._check(self.lib.nph_abea_fetch(self.ctx, _p(pairs), self._abea_pairs, _p(res), self._abea_n),
                    "nph_abea_fetch")
        return pairs, res

    def mom_batch(self, reads, ev_mean, kmer_ranks, jobs, model_id: int) -> np.ndarray:
        out = np.zeros((jobs.shape[0], 2), np.float64)
        self._check(self.lib.nph_mom_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), ev_mean.shape[0],
                                           _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs), jobs.shape[0],
                                           model_id, _p(out)), "nph_mom_batch")
        return out

    # ---- event detection (scrappie detect_events) ---------------------------------------------
    def detect_events_batch(self, raw, reads, params, out=None):
        """== [detect_events(read_i)]: list of EVENT_DT arrays, one per raw read.  out: (events EVENT_DT[room], counts u4[n_reads]) to
        reuse (page-locked) buffers across calls."""
        total = int((reads["event_off"] + reads["event_cap"]).max()) if reads.shape[0] else 0
        events, counts = out if out is not None else (np.zeros(total, EVENT_DT), np.zeros(reads.shape[0], np.uint32))
        assert events.shape[0] >= total and counts.shape[0] >= reads.shape[0]
        self._check(self.lib.nph_detect_events_batch(self.ctx, _p(raw), raw.shape[0], _p(reads), reads.shape[0], _p(params),
                                                     _p(events), total, _p(counts)), "nph_detect_events_batch")
        return [events[int(r["event_off"]):int(r["event_off"]) + int(c)] for r, c in zip(reads, counts)]

    # ---- raw trimming and post-ABEA calibration (the rest of load_from_raw) -----------------------
    def trim_raw_batch(self, raw, reads, trim_start=200, trim_end=10, varseg_chunk=100, varseg_thresh=0.0):
        """== trim_and_segment_raw per read: RAW_RANGE_DT[n_reads], {0,0} where nothing survives."""
        out = np.zeros(reads.shape[0], RAW_RANGE_DT)
        self._check(self.lib.nph_trim_raw_batch(self.ctx, _p(raw), raw.shape[0], _p(reads), reads.shape[0], trim_start, trim_end,
                                                varseg_chunk, varseg_thresh, _p(out)), "nph_trim_raw_batch")
        return out

    def recalibrate_batch(self, reads, ev_mean, kmer_ranks, jobs, model_id, pairs, results):
        """base_to_event_map + events_per_base + recalibrate_model per ABEA job: (EVENT_RANGE_DT[n_ranks], CALIBRATION_DT[n_jobs])."""
        b2e = np.zeros(kmer_ranks.shape[0], EVENT_RANGE_DT)
        cal = np.zeros(jobs.shape[0], CALIBRATION_DT)
        self._check(self.lib.nph_recalibrate_batch(self.ctx, _p(reads), reads.shape[0], _p(ev_mean), ev_mean.shape[0], _p(kmer_ranks),
                                                   kmer_ranks.shape[0], _p(jobs), jobs.shape[0], model_id, _p(pairs), pairs.shape[0],
                                                   _p(results), _p(b2e), _p(cal)), "nph_recalibrate_batch")
        return b2e, cal

    def load_from_raw_batch(self, raw, kmer_ranks, jobs, model_id, params, events_cap=None, pinned=None):
        """SquiggleRead::load_from_raw for a batch in one call.  Returns (event_off u64[n+1], mean, stdv, start_time,
        duration, base_to_event EVENT_RANGE_DT[n_ranks], CALIBRATION_DT[n_jobs]); event arrays are compact, job order."""
        n = jobs.shape[0]
        cap = int(events_cap if events_cap is not None else raw.shape[0] // 3 + 16 * n)
        off = np.zeros(n + 1, np.uint64)
        if pinned is not None:            # caller-staged output buffers (e.g. page-locked): mean, stdv, start_time, duration, b2e, cal
            mean, stdv, start, dur, b2e, cal = pinned
        else:
            mean = np.zeros(cap, np.float32); stdv = np.zeros(cap, np.float32); start = np.zeros(cap, np.float64); dur = np.zeros(cap, np.float32)
            b2e = np.zeros(kmer_ranks.shape[0], EVENT_RANGE_DT)
            cal = np.zeros(n, CALIBRATION_DT)
        self._check(self.lib.nph_load_from_raw_batch(self.ctx, _p(raw), raw.shape[0], _p(kmer_ranks), kmer_ranks.shape[0], _p(jobs), n, model_id,
                                                     _p(params), _p(off), _p(mean), _p(stdv), _p(start), _p(dur), cap, _p(b2e), _p(cal)),
                    "nph_load_from_raw_batch")
        tot = int(off[-1])
        return off, mean[:tot], stdv[:tot], start[:tot], dur[:tot], b2e, cal

    def polya_batch(self, raw, jobs, ev_duration, base_to_event):
        """nanopolish polya's per-read estimate (segmentation, read rate, tail length, QC) for a batch in one call.
        raw: float32 whole raw signals; jobs: POLYA_JOB_DT; ev_duration: float32 event durations; base_to_event:
        EVENT_RANGE_DT (the layout of load_from_raw_batch's outputs).  Returns POLYA_RES_DT[n_jobs];
        nanopolish_b200.polya.rows() turns it into the reference's TSV rows."""
        return self._tail_batch("nph_polya_batch", POLYA_RES_DT, raw, jobs, ev_duration, base_to_event)

    def detect_polyi_batch(self, raw, jobs, ev_duration, base_to_event):
        """nanopolish detect-polyi's per-read result (polya_batch's fields under the poly(I) segmentation model, then the
        poly(I) / poly(A) switch in the tail and its detection tag) for a batch in one call.  Takes polya_batch's inputs;
        returns POLYI_RES_DT[n_jobs], which nanopolish_b200.detect_polyi.rows() turns into the reference's TSV rows."""
        return self._tail_batch("nph_detect_polyi_batch", POLYI_RES_DT, raw, jobs, ev_duration, base_to_event)

    def _tail_batch(self, symbol, result_dt, raw, jobs, ev_duration, base_to_event):
        n = jobs.shape[0]
        out = np.zeros(n, result_dt)
        self._check(getattr(self.lib, symbol)(self.ctx, _p(raw), raw.shape[0], _p(jobs), n, _p(ev_duration), ev_duration.shape[0],
                                              _p(base_to_event), base_to_event.shape[0], _p(out)), symbol)
        return out

    # ---- measurement ----------------------------------------------------------------------
    def last_trim_ranges(self, n_jobs: int) -> np.ndarray:
        """[start, end) of the samples each job of the last load_from_raw_batch kept (what SRF_LOAD_RAW_SAMPLES stores)."""
        from .synth import RAW_RANGE_DT
        out = np.zeros(n_jobs, RAW_RANGE_DT)
        self._check(self.lib.nph_last_trim_ranges(self.ctx, _p(out), n_jobs), "nph_last_trim_ranges")
        return out

    def sync(self):
        self._check(self.lib.nph_sync(self.ctx), "nph_sync")

    def last_kernel_ms(self):
        ms, n = C.c_float(), C.c_int()
        self._check(self.lib.nph_last_kernel_ms(self.ctx, C.byref(ms), C.byref(n)), "nph_last_kernel_ms")
        return ms.value, n.value

    def stream(self) -> int:
        return int(self.lib.nph_stream(self.ctx) or 0)
