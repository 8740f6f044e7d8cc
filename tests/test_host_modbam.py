"""call-methylation's modBAM output (--modbam-output): the Mm / Ml tags of create_modbam_record and
create_reference_modbam_record (src/basemods/nanopolish_basemods.cpp:35-238) from the C++ host
(nanopolish_b200/host/nph_methylation.*) against the COMPILED reference's create_modbam_record (oracle/_ref: the TU is
linked with --gc-sections, htslib's tag writers replaced by stubs that keep what they are handed)."""
import ctypes as C

import numpy as np
import pytest

from oracle import eventalign_py as EP
from tests import host_mirror as hm

K = 6
host = hm.fixture()


def _host_tags(host, seq, ref_pos, flag, cigar, calls, reference_mode=0):
    n = len(calls)
    sp = np.array([c[0] for c in calls], np.int32)
    seqs = (C.c_char_p * max(n, 1))(*[c[1].encode() for c in calls])
    lm = np.array([c[2] for c in calls], np.float64); lu = np.array([c[3] for c in calls], np.float64)
    mm = C.create_string_buffer(1 << 16); ml = np.zeros(1 << 14, np.uint8)
    p = hm.p
    cg = np.ascontiguousarray(cigar, np.uint32)
    k = host.nphh_modbam_tags(seq.encode(), int(ref_pos), int(flag), p(cg), int(cg.shape[0]), n, p(sp), seqs, p(lm), p(lu), reference_mode,
                              mm, C.c_size_t(1 << 16), p(ml), C.c_size_t(ml.shape[0]))
    assert k >= 0, host.nphh_last_error()
    return mm.value.decode(), ml[:k].copy()


def _record(rng, n_ref=900, reverse=False):
    """a reference stretch rich in CG, a read derived from it with substitutions / insertions / deletions, its CIGAR, and
    ScoredSites for CG groups of the reference (sequence = ref[first-k+1 : last+k], like calculate_methylation_for_read)"""
    ref = list("".join("ACGT"[c] for c in rng.integers(0, 4, n_ref)))
    for p in rng.choice(np.arange(20, n_ref - 20), 60, replace=False):
        ref[p], ref[p + 1] = "C", "G"
    ref = "".join(ref)
    ops, read = [(6, "S")], list("ACGTAC")
    i = 0
    while i < n_ref:
        m = int(min(n_ref - i, rng.integers(40, 120)))
        seg = list(ref[i:i + m])
        for j in rng.choice(m, size=min(2, m), replace=False):
            seg[j] = "ACGT"[(("ACGT".index(seg[j])) + 1) % 4]              # substitutions: some calls land on a non-C base
        read += seg; ops.append((m, "M")); i += m
        if i >= n_ref:
            break
        if rng.random() < 0.5:
            ins = int(rng.integers(1, 4)); read += ["ACGT"[c] for c in rng.integers(0, 4, ins)]; ops.append((ins, "I"))
        else:
            d = int(min(n_ref - i, rng.integers(1, 5))); ops.append((d, "D")); i += d     # some CGs have no aligned read base
    seq = "".join(read)
    ref_pos = 5000
    sites = [p for p in range(K, n_ref - K - 1) if ref[p:p + 2] == "CG"]
    calls, cur = [], 0
    while cur < len(sites):
        end = cur + 1
        while end < len(sites) and sites[end] - sites[end - 1] <= 10:
            end += 1
        first, last = sites[cur], sites[end - 1]
        if rng.random() < 0.8:
            ll_u = float(rng.uniform(-300, -60)); ll_m = ll_u + float(rng.normal(0, 6))
            calls.append((ref_pos + first, ref[first - K + 1:last + K], ll_m, ll_u))
        cur = end
    return ref, seq, ref_pos, (EP.BAM_FREVERSE if reverse else 0), EP.pack_cigar(ops), calls


@pytest.mark.parametrize("reverse", [False, True])
def test_modbam_tags_match_compiled_reference(host, ref_oracle, reverse):
    rng = np.random.default_rng(31 + int(reverse))
    for rep in range(6):
        ref, seq, ref_pos, flag, cigar, calls = _record(rng, reverse=reverse)
        want_mm, want_ml = ref_oracle.modbam(seq, ref_pos, flag, cigar, calls)
        got_mm, got_ml = _host_tags(host, seq, ref_pos, flag, cigar, calls)
        assert got_mm == want_mm and np.array_equal(got_ml, want_ml)
        assert want_mm.startswith("C+m?,") and want_mm.endswith(";") and want_ml.shape[0] == want_mm.count(",") > 20
    # no calls at all: the bare tag
    assert _host_tags(host, seq, ref_pos, flag, cigar, [])[0] == ref_oracle.modbam(seq, ref_pos, flag, cigar, [])[0] == "C+m?;"


def test_reference_modbam_tags(host):
    """create_reference_modbam_record: every called CG of the reference span, deltas counted in reference Cs."""
    rng = np.random.default_rng(77)
    ref, seq, ref_pos, flag, cigar, calls = _record(rng)
    mm, ml = _host_tags(host, ref, ref_pos, 0, cigar, calls, reference_mode=1)
    positions = []
    for start, s, ll_m, ll_u in calls:
        positions += [start + j - s.find("CG") for j in range(len(s) - 1) if s[j:j + 2] == "CG"]
    deltas, prev = [], 0
    for pos in positions:
        i = pos - ref_pos
        deltas.append(ref[prev:i].count("C")); prev = i + 1
    assert mm == "C+m?," + ",".join(str(d) for d in deltas) + ";"
    codes = []
    for start, s, ll_m, ll_u in calls:
        pm = np.exp(ll_m) / (np.exp(ll_m) + np.exp(ll_u))
        codes += [min(255, int(pm * 255))] * s.count("CG")
    assert ml.tolist() == codes


def test_modbam_rejects_spliced_records(host):
    rng = np.random.default_rng(5)
    ref, seq, ref_pos, flag, cigar, calls = _record(rng)
    spliced = np.concatenate([cigar[:2], EP.pack_cigar([(30, "N")]), cigar[2:]])
    mm = C.create_string_buffer(64); ml = np.zeros(8, np.uint8)
    p = hm.p
    assert host.nphh_modbam_tags(seq.encode(), ref_pos, 0, p(spliced), int(spliced.shape[0]), 0, None, (C.c_char_p * 1)(), None, None, 0,
                                 mm, C.c_size_t(64), p(ml), C.c_size_t(8)) < 0           # the reference exits on spliced alignments
