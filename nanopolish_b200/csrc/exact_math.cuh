// exact_math.cuh — the two scalar primitives of the DP inner loops, written so that the result is
// bit-identical to the reference's IEEE-754 arithmetic while costing as few issue slots as possible.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define NPH_LOGSUM_CUT 15700        // (max - min) >= 15.7f returns max: table entries from here on hold 0.0f
// lsum_sat's index reaches 2^14: its table has 16385 entries, and entries NPH_LOGSUM_CUT .. 2^14 hold 0.0f
#define NPH_LOGSUM_TBL_LEN 16385

// ---- quantised log-sum ---------------------------------------------------------------------
// Reference (src/common/logsum.h:55-66):
//     max = a > b ? a : b;  min = a < b ? a : b;
//     (min == -inf || max - min >= 15.7f) ? max : max + tbl[(int)((max - min) * 1000.f)]
// Two forms, which return the same float for every pair of operands (both read entry floor(RN(|d| * 1000)) wherever the
// reference reads the table, and a 0.0f entry or -inf + log 2 = -inf everywhere else):
//   * lsum, 8 instructions: the index clamped to the zero entry NPH_LOGSUM_CUT; a table of NPH_LOGSUM_CUT + 1 entries or more.
//   * lsum_sat, 7 instructions: the clamp folded into the multiply; a table of NPH_LOGSUM_TBL_LEN entries.  The forward kernel
//     uses this one.  tests/cuda/check_lsum_saturated.cu compares it with the reference and with lsum on the device.
struct LogsumTable {
    uint32_t biased_base;   // shared-window byte address of entry 0, minus 4 * (bit pattern of the floor's offset) (mod 2^32)
    uint32_t scale;         // 4, as a RUNTIME value: bits * scale + base then stays one IMAD on the FMA pipe; with a literal 4 ptxas
                            // picks LEA, which issues on the half-rate ALU pipe that FMNMX already loads
};

// `bias` must be NPH_LOGSUM_ADDR_BIAS (lsum) or NPH_LOGSUM_SAT_ADDR_BIAS (lsum_sat) and must reach the kernel as a RUNTIME
// value (a kernel parameter): when ptxas can see the constant it re-associates (bits*4 + base) - const into two instructions.
#define NPH_LOGSUM_ADDR_BIAS (0u - 4u * 0x4B000000u)
#define NPH_LOGSUM_SAT_ADDR_BIAS (0u - 4u * 0x44000000u)
__device__ __forceinline__ LogsumTable make_logsum_table(const float* smem_tbl, uint32_t bias, uint32_t scale = 4u)
{
    LogsumTable t;
    t.biased_base = (uint32_t)__cvta_generic_to_shared(smem_tbl) + bias;
    t.scale = scale;
    return t;
}

__device__ __forceinline__ float lsum_lookup(float mx, float u, const LogsumTable tb)
{
    const uint32_t adr = (uint32_t)__float_as_int(u) * tb.scale + tb.biased_base;
    float v;
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(adr));
    return __fadd_rn(mx, v);
}

// lsum, in 8 SASS instructions (2 ALU-pipe, 5 FMA-pipe, 1 LDS):
//     mx  = fmaxf(a, b)                                   FMNMX
//     d   = a - b                 (|d| == max - min exactly: RN is sign-symmetric)   FADD
//     t   = fminf(|d| * 1000, 15700)                      FMUL (|.| is a free source modifier), FMNMX
//     u   = t +(round-down) 2^23  -> bits = 0x4B000000 + floor(t)                     FADD.RM
//     adr = bits * 4 + (table_base - 4 * 0x4B000000)      IMAD   (mod 2^32)
//     r   = mx + shared[adr]                              LDS, FADD
// The clamp lands on table entry 15700, which holds 0.0f: that reproduces "return max" for
// max - min >= 15.7f (15.7f * 1000.f rounds to exactly 15700.0f, and every smaller float maps to an
// index <= 15699), for min == -inf (difference +inf), and for both -inf (difference NaN: fminf
// returns the non-NaN operand, and -inf + 0 = -inf).
__device__ __forceinline__ float lsum(float a, float b, const LogsumTable tb)
{
    const float mx = fmaxf(a, b);
    const float d = __fsub_rn(a, b);
    const float t = fminf(__fmul_rn(fabsf(d), 1000.0f), (float)NPH_LOGSUM_CUT);
    return lsum_lookup(mx, __fadd_rd(t, 8388608.0f), tb);
}

// lsum_sat, in 7 SASS instructions (1 ALU-pipe, 5 FMA-pipe, 1 LDS):
//     mx  = fmaxf(a, b)                                   FMNMX
//     d   = a - b                                         FADD
//     t   = sat(|d| * (1000 * 2^-14))                     FMUL.SAT (|.| is a free source modifier)
//     u   = t +(round-down) 2^9   -> bits = 0x44000000 + floor(t * 2^14)              FADD.RM
//     adr = bits * 4 + (table_base - 4 * 0x44000000)      IMAD   (mod 2^32)
//     r   = mx + shared[adr]                              LDS, FADD
// Why the index is the reference's, entries >= 15700 being 0.0f:
//   * 1000 * 2^-14 = 0.06103515625 is exact, and scaling by a power of two commutes with round-to-nearest
//     while the result is normal: RN(|d| * 1000 * 2^-14) = RN(|d| * 1000) * 2^-14.  Saturation clamps to [0, 1],
//     so t * 2^14 = min(RN(|d| * 1000), 16384).  If the scaled product is subnormal (|d| * 1000 < 2^-112) both
//     forms give index 0.
//   * t lies in [0, 1] and the spacing of floats in [512, 1024) is 2^-14, so t + 512 rounded down is
//     512 + floor(t * 2^14) * 2^-14, whose bit pattern is 0x44000000 + floor(t * 2^14) (at most 0x44004000 = 513.0f).
//   * max - min >= 15.7f: 15.7f * 1000.f rounds to exactly 15700.0f and every smaller float maps to an index
//     <= 15699, so exactly these differences read an entry in 15700 .. 16384, which holds 0.0f: "return max".
//   * min == -inf, max finite: |d| = +inf, saturates to 1, entry 16384 (0.0f).  Both -inf: d is NaN, which
//     saturation turns into 0, entry 0 (log 2); -inf + log 2 = -inf.
// Without lsum's clamp onto one zero word, a difference in [15.7, 16.384) reads its own zero word: slightly more bank
// conflicts for one instruction less (DESIGN §3.4).
__device__ __forceinline__ float lsum_sat(float a, float b, const LogsumTable tb)
{
    const float mx = fmaxf(a, b);
    const float d = __fsub_rn(a, b);
    const float t = __saturatef(__fmul_rn(fabsf(d), 0.06103515625f));
    return lsum_lookup(mx, __fadd_rd(t, 512.0f), tb);
}

// ---- add_logs(a, b) = p7_FLogsum on floats (ref: src/common/logsum.h:55-66) with the reference's table below NPH_LOGSUM_CUT
__host__ __device__ inline float nph_flogsum(float a, float b, const float* tbl)
{
    const float mx = a > b ? a : b, mn = a < b ? a : b;
    const float d = mx - mn;
    return (mn == -INFINITY || !(d < 15.7f)) ? mx : mx + tbl[(int)(d * 1000.f)];
}

// ---- profile_hmm_score_set's fold of one group of scores (ref: src/hmm/nanopolish_profile_hmm.cpp:32-56) --------------------
// s[0] is the nucleotide sequence's score, s[1 .. n-1] those of its methylated alternatives; pen = log(n) from host libm.
//     score = s[0] - pen;  per alternative: add_logs((float)score, (float)(s[i] - pen)) -> score (double)
// with add_logs the table log-sum of src/common/logsum.h:55-66.  tbl needs the reference's entries below NPH_LOGSUM_CUT (the host's
// own table or the context's device copy).  Every operation is a single IEEE operation (no multiply feeds an add), so host and
// device round alike.  !(d < 15.7f) also catches NaN / inf differences (a NaN or +inf score): no out-of-range table index.
__host__ __device__ inline float nph_score_set_fold(const float* s, uint32_t n, double pen, const float* tbl)
{
    double score = (double)s[0] - pen;
    for (uint32_t i = 1; i < n; ++i) {
        const double alt = (double)s[i] - pen;
        score = nph_flogsum((float)score, (float)alt, tbl);
    }
    return (float)score;
}

// ---- phase-reads' call and quality of one SNP from its two scores (ref: src/nanopolish_phase_reads.cpp:293-317) ---------------
//     log_sum = add_logs(alt, ref)   (p7_FLogsum on the float scores, as nph_score_set_fold's step)
//     log_p_wrong = (alt > ref ? ref : alt) - log_sum;   q = std::min(30.0, -10 * log_p_wrong / log(10));   q_char = (int)q + 33
// The call is alt_base when alt > ref, else ref_base.  std::min(30, q) returns 30 for a NaN q.  Every step is one IEEE operation
// and log(10) is the constant the compiler folds, so host and device round alike.
struct NphPhaseCall { char call; uint8_t q_char; };
__host__ __device__ inline NphPhaseCall nph_phase_quality(float ref, float alt, char ref_base, char alt_base, const float* tbl)
{
    const double log_sum = nph_flogsum(alt, ref, tbl);
    const bool is_alt = alt > ref;
    const double log_p_wrong = (double)(is_alt ? ref : alt) - log_sum;
    const double q = -10.0 * log_p_wrong / 2.302585092994045684;       // log(10), correctly rounded
    const double qc = q < 30.0 ? q : 30.0;
    return NphPhaseCall{is_alt ? alt_base : ref_base, (uint8_t)((int)qc + 33)};
}

// ---- correctly rounded float division with a precomputed reciprocal --------------------------
// The Gaussian z-score (x - mu) / sigma is an IEEE division in the reference (emissions.h:53).
// sigma is fixed per k-mer column, so y = RN(1/sigma) is computed once (__frcp_rn) and each cell
// pays 5 FMA-pipe instructions and no branch instead of the ~10 + slow-path branch of __fdiv_rn:
//     q0 = RN(a*y); r0 = RN(a - q0*b) [fma]; q1 = RN(q0 + r0*y) [fma]; r1 = RN(a - q1*b); q = RN(q1 + r1*y)
// This is Markstein's division: with y the correctly rounded reciprocal and q1 within one ulp of
// a/b, the final fused step rounds a/b correctly.  The proof needs no over/underflow in the
// intermediates; our operands (|a| < 2^12, 2^-8 < b < 2^8) are far from both, and a == 0, which
// makes every term zero, is exact.  tests/cuda/check_exact_math.cu compares it with __fdiv_rn on
// ~10^10 operand pairs including all-ones-mantissa divisors (the classical hard case).
__device__ __forceinline__ float div_by_cached_rcp(float a, float b, float y)
{
    const float q0 = __fmul_rn(a, y);
    const float r0 = __fmaf_rn(-q0, b, a);
    const float q1 = __fmaf_rn(r0, y, q0);
    const float r1 = __fmaf_rn(-q1, b, a);
    return __fmaf_rn(r1, y, q1);
}

// ---- the Gaussian's last two operations in one FMUL + one FFMA ---------------------------------
// The reference forms cc + (-0.5f*a)*a (emissions.h:54): three roundings.  Scaling by 2^-1 commutes with
// round-to-nearest while the result stays normal, so RN(RN(-0.5a)*a) = -0.5*RN(a*a) whenever
// 0.5*a*a >= 2^-126; the FMA's product RN(a*a)*(-0.5) is then exact and only the final add rounds, as in
// the reference.  Below that (|a| < 2^-62.5, a != 0) both forms add less than half an ulp of cc and return cc,
// unless |cc| < 2^-100.  For a nonzero a = RN((x - mu)/sigma) the first case needs |x - mu| < 2^-54 * sigma, which
// two pA levels cannot give, and cc = log(1/sqrt(2pi)) - log(sigma) is 0 or at least 2^-25 in magnitude.  a == 0
// gives cc + (-0) in both forms; |a| stays far below the 2^63 where a*a would overflow (|x - mu| < 2^12, sigma > 2^-8).
// tests/cuda/check_emission_fold.cu compares it with the literal form on the device.
__device__ __forceinline__ float add_neg_half_square(float cc, float a)
{
    return __fmaf_rn(__fmul_rn(a, a), -0.5f, cc);
}

// Gaussian log-density of level x under a column's {mu, sd, cc = log(1/sqrt(2pi)) - log sd, ry = RN(1/sd)} (emissions.h:51-55).  The Viterbi
// replay calls the function its fill called, so it reproduces the fill's values bit for bit.
__device__ __forceinline__ float log_gauss(float x, float mu, float sd, float cc, float ry)
{
    return add_neg_half_square(cc, div_by_cached_rcp(__fsub_rn(x, mu), sd, ry));
}
