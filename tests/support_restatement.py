"""Plain-Python restatement of `nanopolish variants --calculate-all-support` — test infrastructure (the checker of
csrc/all_support.cu and of the host mirror built on it), never imported by the product.

Follows annotate_variants_with_all_support, src/common/nanopolish_variant.cpp:801-859, with the pieces it calls:
  Haplotype::substr_by_reference, apply_variant                  src/nanopolish_haplotype.cpp:33-140 (tests/hp_restatement.py)
  AlignmentDB::get_event_subsequences                            src/alignment/nanopolish_alignment_db.cpp:172-221 (hp_restatement)
  add_logs (p7_FLogsum on floats: the double overload narrows)   src/common/nanopolish_common.h:100-116
  the stringstream of std::fixed << std::setprecision(3), and Variant::add_info
The forward scores (profile_hmm_score, floats) and add_logs come from the caller: the compiled reference's own, or the device's
scores with the plain-C port's log-sum."""
import math

import numpy as np

from tests import hp_restatement as hr

BASES = "ACGT"
KEY = "SupportFractionByBase"


def window(region: hr.Haplotype, ref_position: int, flank: int):
    """(calling_start, calling_end, the window haplotype): substr_by_reference of the unedited region, hr.RefAbort where the
    reference asserts (a window outside the region)"""
    cs, ce = ref_position - flank, ref_position + flank
    return cs, ce, region.substr_by_reference(cs, ce)


def haplotypes(win: hr.Haplotype, ref_position: int, ref_seq: str):
    """([the four haplotype sequences], whether apply_variant applied): ref_seq replaced by b on a fresh copy of the window"""
    out, applied = [], False
    for b in BASES:
        h = win.copy()
        applied = h.apply_variant(ref_position, ref_seq, b)
        out.append(h.seq)
    return out, applied


def support(scores, add_logs):
    """the four support fractions of one variant from its reads' four float32 scores each, in record order: sum = s[0], then
    sum = add_logs(s[hi], sum); support[hi] += exp(double(s[hi]) - double(sum)); then / len(scores) (0 / 0: a NaN with the sign bit
    set, as x86-64 divides)"""
    sup = [0.0] * 4
    for s in scores:
        s = [np.float32(x) for x in s]
        total = s[0]
        for hi in range(1, 4):
            total = np.float32(add_logs(s[hi], total))
        for hi in range(4):
            sup[hi] += math.exp(float(s[hi]) - float(total))
    n = len(scores)
    if n == 0:
        return np.full(4, -np.nan)
    return np.array([x / float(n) for x in sup], np.float64)


def fixed3(x: float) -> str:
    """operator<< of a double under std::fixed and setprecision(3)"""
    x = float(x)
    if math.isnan(x):
        return "-nan" if math.copysign(1.0, x) < 0 else "nan"
    if math.isinf(x):
        return "-inf" if x < 0 else "inf"
    return f"{x:.3f}"


def info(values) -> str:
    return KEY + "=" + ",".join(fixed3(v) for v in values)


def add_info(existing: str, kv: str) -> str:
    return kv if not existing else existing + ";" + kv
