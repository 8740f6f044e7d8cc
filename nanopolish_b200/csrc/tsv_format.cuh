// tsv_format.cuh — printf("%.Nlf") and printf("%d") without the C library, and the methylation_calls.tsv row built from them,
// for host and device.  The one copy of these rules: libnph's kernels and the host library (nanopolish_b200/host) both use it.
//
// fixed_of<N>(double), N <= 3: v = m * 2^-sft exactly (m < 2^53), so v * 10^N = (m * 10^N) * 2^-sft fits 64-bit integer
// arithmetic with an exact remainder, and round-half-to-even on it is the decimal string glibc prints (it rounds the exact
// value, in the default rounding mode) and the one Python's "%.Nf" prints (also the exact value, ties to even).  Magnitudes of
// 2^52 and above and non-finite values are refused (ok = false).
// fixed_of<N>(float), N <= 5: v = m * 2^e exactly (m < 2^24), so m * 10^N < 2^41 and, below 2^39, a left shift stays < 2^56.
// Magnitudes of 2^39 and above and non-finite values are refused.
// Callers format refused values with the C library.  tests/cuda/check_tsv_format.cu checks this header against snprintf on
// host and device.  Plain C++14 without CUDA headers compiles it too (the host library).
#pragma once
#include <cstdint>
#include <cstring>
#include "../../include/nph.h"

#if defined(__CUDACC__)
#define NPH_HD __host__ __device__ __forceinline__
#else
#define NPH_HD inline
#endif

namespace nph_tsv {

struct Fixed {
    uint64_t q;      // round_half_even(|v| * 10^N)
    bool neg, ok;
};

template <int N> struct Pow10 { static constexpr uint64_t v = 10u * Pow10<N - 1>::v; };
template <> struct Pow10<0> { static constexpr uint64_t v = 1u; };

// round_half_even(x * 2^-sft) for sft >= 1 and x < 2^63
NPH_HD uint64_t shift_round(uint64_t x, int sft)
{
    if (sft > 63) return 0;                  // x < 2^63 is below half a unit of the last printed digit
    uint64_t q = x >> sft;
    const uint64_t rem = x & (((uint64_t)1 << sft) - 1), half = (uint64_t)1 << (sft - 1);
    if (rem > half || (rem == half && (q & 1))) q += 1;
    return q;
}

template <int N>
NPH_HD Fixed fixed_of(double v)
{
    static_assert(N >= 0 && N <= 3, "m * 10^N must fit 64 bits for every m < 2^53");
    uint64_t bits;
    memcpy(&bits, &v, 8);
    const uint32_t expo = (uint32_t)((bits >> 52) & 0x7ff);
    uint64_t m = bits & 0xfffffffffffffull;
    int sft;                                 // |v| = m * 2^-sft, sft >= 1
    if (expo == 0) sft = 1074; else { m |= (uint64_t)1 << 52; sft = 1075 - (int)expo; }
    Fixed f;
    f.neg = (bits >> 63) != 0;
    f.ok = !(expo == 0x7ff || expo >= 1075);
    f.q = f.ok ? shift_round(m * Pow10<N>::v, sft) : 0;
    return f;
}

template <int N>
NPH_HD Fixed fixed_of(float v)
{
    static_assert(N >= 0 && N <= 5, "m * 10^N << 15 must fit 64 bits for every m < 2^24");
    uint32_t bits;
    memcpy(&bits, &v, 4);
    const uint32_t expo = (bits >> 23) & 0xff;
    uint64_t m = bits & 0x7fffff;
    int e;                                   // |v| = m * 2^e
    if (expo == 0) e = -149; else { m |= 0x800000; e = (int)expo - 150; }
    Fixed f;
    f.neg = (bits >> 31) != 0;
    f.ok = expo < 127 + 39;                  // also refuses 0xff: inf, nan
    const uint64_t x = m * Pow10<N>::v;
    f.q = !f.ok ? 0 : e >= 0 ? x << e : shift_round(x, -e);
    return f;
}

NPH_HD int ndigits(uint64_t x)
{
    int n = 1;
    while (x >= 10u) { x /= 10u; ++n; }
    return n;
}

template <int N>
NPH_HD int fixed_len(const Fixed& f) { return (f.neg ? 1 : 0) + ndigits(f.q / Pow10<N>::v) + (N > 0 ? 1 + N : 0); }

NPH_HD char* put_u64(char* o, uint64_t v)
{
    const int n = ndigits(v);
#ifdef __CUDA_ARCH__
    for (int i = n - 1; i >= 0; --i) { o[i] = (char)('0' + (int)(v % 10u)); v /= 10u; }
#else
    // host: two digits per division (the host row formatters are bound by these divisions)
    static const char kPairs[201] =
        "0001020304050607080910111213141516171819202122232425262728293031323334353637383940414243444546474849"
        "5051525354555657585960616263646566676869707172737475767778798081828384858687888990919293949596979899";
    int i = n;
    while (v >= 100u) { const uint32_t r = (uint32_t)(v % 100u); v /= 100u; i -= 2; o[i] = kPairs[2 * r]; o[i + 1] = kPairs[2 * r + 1]; }
    if (v >= 10u) { o[0] = kPairs[2 * v]; o[1] = kPairs[2 * v + 1]; } else o[0] = (char)('0' + v);
#endif
    return o + n;
}

template <int N>
NPH_HD char* put_fixed(char* o, const Fixed& f)
{
    if (f.neg) *o++ = '-';
    o = put_u64(o, f.q / Pow10<N>::v);
    if (N == 0) return o;
    *o++ = '.';
    uint64_t fp = f.q % Pow10<N>::v;
    for (int i = N - 1; i >= 0; --i) { o[i] = (char)('0' + (int)(fp % 10u)); fp /= 10u; }
    return o + N;
}

NPH_HD int int_len(int v) { return v < 0 ? 1 + ndigits((uint64_t)(-(int64_t)v)) : ndigits((uint64_t)v); }

NPH_HD char* put_i64(char* o, int64_t v)
{
    if (v < 0) { *o++ = '-'; return put_u64(o, 0ull - (uint64_t)v); }
    return put_u64(o, (uint64_t)v);
}

NPH_HD char* put_int(char* o, int v) { return put_i64(o, v); }

NPH_HD char* put_bytes(char* o, const char* s, uint32_t n)
{
#ifdef __CUDA_ARCH__
    for (uint32_t i = 0; i < n; ++i) o[i] = s[i];
#else
    memcpy(o, s, n);
#endif
    return o + n;
}

// ---- methylation_calls.tsv ----------------------------------------------------------------------------------------
// One row of the reference's write_methylation_results_as_tsv, "%s\t%c\t%d\t%d\t%s\t%.2lf\t%.2lf\t%.2lf\t%d\t%d\t%s\n":
// chromosome, strand, start, end, read_name, log_lik_ratio, log_lik_methylated, log_lik_unmethylated, num_calling_strands,
// num_motifs, sequence.  The three numbers must be ok; a row with a refused one is the C library's to print.
struct MethRow {
    const char* contig; uint32_t contig_len;
    char strand;                               // '+' or '-'
    int start, end;
    const char* name; uint32_t name_len;
    Fixed diff, m, u;                          // fixed_of<2> of sum_m - sum_u, sum_m, sum_u
    int strands_scored, n_motif;
    const char* seq; uint32_t seq_len;
};

NPH_HD uint32_t meth_row_len(const MethRow& r)
{
    return r.contig_len + 3u + (uint32_t)int_len(r.start) + 1u + (uint32_t)int_len(r.end) + 1u + r.name_len + 1u +
           (uint32_t)fixed_len<2>(r.diff) + 1u + (uint32_t)fixed_len<2>(r.m) + 1u + (uint32_t)fixed_len<2>(r.u) + 1u +
           (uint32_t)int_len(r.strands_scored) + 1u + (uint32_t)int_len(r.n_motif) + 1u + r.seq_len + 1u;
}

NPH_HD char* put_meth_row(char* o, const MethRow& r)
{
    o = put_bytes(o, r.contig, r.contig_len);
    *o++ = '\t'; *o++ = r.strand; *o++ = '\t';
    o = put_int(o, r.start); *o++ = '\t';
    o = put_int(o, r.end); *o++ = '\t';
    o = put_bytes(o, r.name, r.name_len); *o++ = '\t';
    o = put_fixed<2>(o, r.diff); *o++ = '\t';
    o = put_fixed<2>(o, r.m); *o++ = '\t';
    o = put_fixed<2>(o, r.u); *o++ = '\t';
    o = put_int(o, r.strands_scored); *o++ = '\t';
    o = put_int(o, r.n_motif); *o++ = '\t';
    o = put_bytes(o, r.seq, r.seq_len);
    *o++ = '\n';
    return o;
}

// The printed numbers and the sequence column of the row of site record ms of a record that is its read's only scored strand
// (the other strand's entries are 0.0): the three "%.2lf" likelihoods, and the sequence as [seq_b, seq_b + seq_len) of the
// record's reference.  Shared by both row writers and by the per-site frequency accumulator that reads the rows.
struct RowNums { Fixed diff, m, u; uint32_t seq_b, seq_len; bool seq_ok; };

// seq_ok = false: the sequence column would start before the record's reference (the reference's substr throws)
static constexpr char kSeqRefused[] =
    "a group starts fewer than k - 1 bases into its record's reference: the sequence column of its row is undefined (min_flank too small for k)";

NPH_HD RowNums row_numbers(const nph_meth_site& ms, const nph_meth_record& R, uint32_t k)
{
    RowNums r;
    // ScoredSite: ll_*[strand] = the float score, the other strand 0.0; the writer sums the two strands in double
#ifdef __CUDA_ARCH__
    const double sum_m = __dadd_rn((double)ms.ll_methylated, 0.0), sum_u = __dadd_rn((double)ms.ll_unmethylated, 0.0);
    const double diff = __dsub_rn(sum_m, sum_u);
#else
    const double sum_m = (double)ms.ll_methylated + 0.0, sum_u = (double)ms.ll_unmethylated + 0.0;
    const double diff = sum_m - sum_u;
#endif
    r.diff = fixed_of<2>(diff);
    r.m = fixed_of<2>(sum_m);
    r.u = fixed_of<2>(sum_u);
    // the sequence column starts k - 1 bases before the first site and ends k bases after the last, cut at the end of the
    // record's reference
    const int bs = (ms.start_position - R.ref_start_pos) - (int)k + 1;
    const uint32_t e0 = (uint32_t)(ms.end_position - R.ref_start_pos) + k, e = e0 < R.ref_len ? e0 : R.ref_len;
    r.seq_ok = bs >= 0 && (uint32_t)bs <= e;
    r.seq_b = r.seq_ok ? (uint32_t)bs : 0u; r.seq_len = r.seq_ok ? e - (uint32_t)bs : 0u;
    return r;
}

} // namespace nph_tsv
