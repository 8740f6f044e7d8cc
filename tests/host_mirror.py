"""The C++ host mirror's C shim (nanopolish_b200/libnph_host.so: the nphh_* functions of nanopolish_b200/host/nph_host_capi.cpp) —
test infrastructure.

load() is the one CDLL over it, with every entry's return type declared once.  The rest are the steps the callers of the region
shims (nphh_screen_variants, nphh_all_support, nphh_fix_homopolymers, nphh_call_haplotype, nphh_call_region) share: register a
case's models and reads, build its event-record and allele arguments, and call into an output buffer."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_SO = os.path.join(ROOT, "nanopolish_b200", "libnph_host.so")

# every entry that does not return int, as nph_host_capi.cpp declares it (ctypes reads an undeclared return as a 32-bit int)
RESTYPES = dict.fromkeys(
    ("nphh_read_num_samples", "nphh_abea", "nphh_score_variant_group", "nphh_call_methylation_timed", "nphh_call_methylation",
     "nphh_phase_reads", "nphh_call_methylation_flat", "nphh_modbam_tags", "nphh_polya", "nphh_detect_polyi", "nphh_ea_run",
     "nphh_ea_run_rounds", "nphh_ea_next_round", "nphh_ea_text", "nphh_ea_tsv_all", "nphh_ea_tsv_all_samples", "nphh_ea_tsv_all_opt",
     "nphh_ea_run_tsv", "nphh_format_fixed_check", "nphh_rolling_ranks_check", "nphh_ea_num_segments", "nphh_scorereads",
     "nphh_scorereads_train", "nphh_transition_training", "nphh_aligned_segments", "nphh_fix_homopolymers", "nphh_all_support",
     "nphh_screen_variants", "nphh_call_haplotype", "nphh_expand_variants", "nphh_haplotype_ranges", "nphh_variants_in_region",
     "nphh_call_region"), C.c_longlong)
RESTYPES.update(nphh_last_error=C.c_char_p, nphh_kmer_rank=C.c_uint32, nphh_read_sample=C.c_float, nphh_fisher_exact=C.c_double)


@functools.cache
def load() -> C.CDLL:
    lib = C.CDLL(HOST_SO)
    for entry, restype in RESTYPES.items():
        getattr(lib, entry).restype = restype
    lib.nphh_fisher_exact.argtypes = [C.c_int] * 4
    return lib


def fixture():
    """a module-scoped fixture holding load(): a test module writes `host = host_mirror.fixture()`"""
    def host():
        return load()
    return pytest.fixture(scope="module")(host)


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def cstrs(xs):
    """a char*[] of str or bytes (one null entry when xs is empty)"""
    return (C.c_char_p * max(1, len(xs)))(*[x if isinstance(x, bytes) else x.encode() for x in xs])


def register_model(host, model):
    mean = np.ascontiguousarray(model.level_mean); sd = np.ascontiguousarray(model.level_stdv)
    lsd = np.ascontiguousarray(model.level_log_stdv)
    return host.nphh_model_create(model.alphabet.encode(), model.k, mean.shape[0], p(mean), p(sd), p(lsd))


def register_reads(host, rs, mh):
    hs = []
    for r in rs.reads:
        o, n = int(r["event_off"]), int(r["n_events"])
        m = np.ascontiguousarray(rs.ev_mean[o:o + n]); t = np.ascontiguousarray(rs.ev_start_time[o:o + n])
        hs.append(host.nphh_read_create(n, p(m), p(t), C.c_double(r["shift"]), C.c_double(r["scale"]), C.c_double(r["drift"]),
                                        C.c_double(r["var"]), C.c_double(r["events_per_base"]), mh))
    return hs


def register_case(host, c, model, types=(), durations=None):
    """clear the mirror's reads, register `model` and the case's reads (c["rs"]), give every read each type model of `types` under
    its alphabet (nphh_read_add_model) and, with `durations` (per event, flat as the reads' events), each read's event durations:
    the read handles"""
    host.nphh_clear()
    rs = c["rs"]
    hs = register_reads(host, rs, register_model(host, model))
    for m in types:
        h = register_model(host, m)
        for r in hs:
            host.nphh_read_add_model(int(r), m.alphabet.encode(), h)
    if durations is not None:
        for i, r in enumerate(rs.reads):
            o, n = int(r["event_off"]), int(r["n_events"])
            host.nphh_read_set_durations(hs[i], p(np.ascontiguousarray(durations[o:o + n])))
    return hs


def records(c, hs):
    """the case's event records as the region shims take them: (n_records, read handles, rc, (ref_pos, read_pos) pairs, pair offsets
    (n_records + 1)).  Each record's pairs are gathered by its pair_off / n_pairs, so a record listed twice gets its own copy"""
    recs, pairs = c["recs"], c["pairs"]
    read = np.array([hs[int(x)] for x in recs["read"]], np.int32)
    pp = np.stack([pairs["ref_pos"], pairs["read_pos"]], 1).astype(np.int32)
    order = np.concatenate([np.arange(int(r["pair_off"]), int(r["pair_off"]) + int(r["n_pairs"])) for r in recs] or [np.zeros(0, np.int64)])
    po = np.concatenate([[0], np.cumsum(recs["n_pairs"].astype(np.uint64))]).astype(np.uint64)
    return int(recs.shape[0]), p(read), p(np.ascontiguousarray(recs["rc"], np.uint8)), p(np.ascontiguousarray(pp[order])), p(po)


def alleles(vs):
    """(positions, REF strings, ALT strings) of [(position, ref, alt)]"""
    return p(np.array([v[0] for v in vs] or [0], np.int32)), cstrs([v[1] for v in vs]), cstrs([v[2] for v in vs])


def text(host, entry, *args, cap=1 << 22):
    """entry(*args, out, cap) into a buffer of cap bytes: (status, the bytes written, or None where the status is negative)"""
    out = C.create_string_buffer(cap)
    n = int(getattr(host, entry)(*args, out, C.c_size_t(cap)))
    return n, (out.raw[:n] if n >= 0 else None)
