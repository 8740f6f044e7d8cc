// tsv_format.cuh — the number formatting of methylation_calls.tsv rows and of the per-site frequency table without the C
// library, for host and device.
//
// printf("%.Nf", v) for N <= 3 decimals: v = m * 2^-sft exactly (m < 2^53), so v * 10^N = (m * 10^N) * 2^-sft fits 64-bit
// integer arithmetic with an exact remainder, and round-half-to-even on it is the decimal string glibc prints (it rounds the
// exact value, in the default rounding mode) and the one Python's "%.Nf" prints (also the exact value, ties to even).
// Magnitudes of 2^52 and above and non-finite values are refused (ok = false): the caller formats those rows with the C
// library.  The same arithmetic as nanopolish_b200/host/nph_host.cpp format_fixed, which is checked against snprintf;
// tests/cuda/check_tsv_format.cu (N = 2) and tests/cuda/check_freq_format.cu (N = 3) check this header against snprintf on
// host and device.
#pragma once
#include <cstdint>
#include <cstring>

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
using Fixed2 = Fixed;

template <int N> struct Pow10 { static constexpr uint64_t v = 10u * Pow10<N - 1>::v; };
template <> struct Pow10<0> { static constexpr uint64_t v = 1u; };

template <int N>
NPH_HD Fixed fixed_of(double v)
{
    static_assert(N >= 1 && N <= 3, "m * 10^N must fit 64 bits for every m < 2^53");
    uint64_t bits;
    memcpy(&bits, &v, 8);
    Fixed f;
    f.neg = (bits >> 63) != 0;
    const uint32_t expo = (uint32_t)((bits >> 52) & 0x7ff);
    f.ok = !(expo == 0x7ff || expo >= 1075);
    uint64_t m = bits & 0xfffffffffffffull;
    int sft;                                 // |v| = m * 2^-sft, sft >= 1
    if (expo == 0) sft = 1074; else { m |= (uint64_t)1 << 52; sft = 1075 - (int)expo; }
    const uint64_t x = m * Pow10<N>::v;      // < 2^53 * 1000 < 2^63
    uint64_t q = 0;
    if (f.ok && sft <= 63) {
        q = x >> sft;
        const uint64_t rem = x & (((uint64_t)1 << sft) - 1), half = (uint64_t)1 << (sft - 1);
        if (rem > half || (rem == half && (q & 1))) q += 1;
    }                                        // sft >= 64: x < 2^63 is below half a unit of the last printed digit
    f.q = q;
    return f;
}

NPH_HD Fixed fixed2_of(double v) { return fixed_of<2>(v); }

NPH_HD int ndigits(uint64_t x)
{
    int n = 1;
    while (x >= 10u) { x /= 10u; ++n; }
    return n;
}

template <int N>
NPH_HD int fixed_len(const Fixed& f) { return (f.neg ? 1 : 0) + ndigits(f.q / Pow10<N>::v) + 1 + N; }
NPH_HD int fixed2_len(const Fixed& f) { return fixed_len<2>(f); }

NPH_HD char* put_u64(char* o, uint64_t v)
{
    const int n = ndigits(v);
    for (int i = n - 1; i >= 0; --i) { o[i] = (char)('0' + (int)(v % 10u)); v /= 10u; }
    return o + n;
}

template <int N>
NPH_HD char* put_fixed(char* o, const Fixed& f)
{
    if (f.neg) *o++ = '-';
    o = put_u64(o, f.q / Pow10<N>::v);
    *o++ = '.';
    uint64_t fp = f.q % Pow10<N>::v;
    for (int i = N - 1; i >= 0; --i) { o[i] = (char)('0' + (int)(fp % 10u)); fp /= 10u; }
    return o + N;
}
NPH_HD char* put_fixed2(char* o, const Fixed& f) { return put_fixed<2>(o, f); }

NPH_HD int int_len(int v) { return v < 0 ? 1 + ndigits((uint64_t)(-(int64_t)v)) : ndigits((uint64_t)v); }

NPH_HD char* put_int(char* o, int v)
{
    if (v < 0) { *o++ = '-'; return put_u64(o, (uint64_t)(-(int64_t)v)); }
    return put_u64(o, (uint64_t)v);
}

} // namespace nph_tsv
