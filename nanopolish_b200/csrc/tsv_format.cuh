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
// Further down: printf("%g") of a float (put_g6) and the eventalign.tsv row (ea_row_numbers, ea_kmers_at, put_ea_row), checked
// by tests/cuda/check_g_format.cu.
#pragma once
#include <cmath>
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

// ---- printf("%g") of a float ---------------------------------------------------------------------------------------
// What an ostream prints for a float (six significant digits, trailing zeros dropped, d.ddddde+XX outside 1e-4 <= |v| < 1e6).
// |v| = m * 2^e exactly (m < 2^24).  With X the decimal exponent, |v| * 10^(5 - X) = N / D in 64-bit integers (m * 10^11 <
// 2^61, 2^39 <= 2^63, D <= 10^6 * 2^23), rounded half to even on the exact remainder; X starts at floor(log10 2^(e + 23)), which
// is the value's own decimal exponent or one below it, and moves up when the rounded digits reach 10^6.  Supported: +-0 and
// 2^-17 <= |v| < 2^39; everything else (smaller magnitudes, larger ones, inf, nan) is refused, as fixed_of refuses.
struct G6 {
    uint32_t q;       // the significant digits, trailing zeros dropped (0 for +-0)
    int nsig;         // how many
    int X;            // decimal exponent of the first digit
    bool neg, ok;
};

NPH_HD uint64_t pow10_u64(int n) { uint64_t p = 1; for (int i = 0; i < n; ++i) p *= 10u; return p; }

// round_half_even(m * 2^e * 10^P) for m < 2^24, 2^-17 <= m * 2^e < 2^39, -6 <= P <= 11
NPH_HD uint64_t g6_scaled(uint64_t m, int e, int P)
{
    if (P >= 0) {                                          // then e < 0: a value with e >= 0 is at least 2^23 > 10^6
        const uint64_t x = m * pow10_u64(P);
        return e >= 0 ? x << e : shift_round(x, -e);
    }
    const uint64_t N = e >= 0 ? m << e : m, D = pow10_u64(-P) << (e >= 0 ? 0 : -e);
    uint64_t q = N / D;
    const uint64_t rem2 = 2u * (N - q * D);
    if (rem2 > D || (rem2 == D && (q & 1))) q += 1;
    return q;
}

NPH_HD G6 g6_of(float v)
{
    uint32_t bits;
    memcpy(&bits, &v, 4);
    const uint32_t expo = (bits >> 23) & 0xff;
    G6 g;
    g.neg = (bits >> 31) != 0;
    g.q = 0; g.nsig = 1; g.X = 0;
    g.ok = (bits << 1) == 0 || (expo >= 127 - 17 && expo < 127 + 39);
    if (!g.ok || (bits << 1) == 0) return g;
    const uint64_t m = (bits & 0x7fffff) | 0x800000;
    const int e = (int)expo - 150;
    int X = ((e + 23) * 1233) >> 12;                       // floor((e + 23) * log10 2) for |e + 23| <= 40
    uint64_t q = g6_scaled(m, e, 5 - X);
    while (q >= 1000000u) { X += 1; q = g6_scaled(m, e, 5 - X); }
    int nsig = 6;
    while (nsig > 1 && q % 10u == 0) { q /= 10u; --nsig; }
    g.q = (uint32_t)q; g.nsig = nsig; g.X = X;
    return g;
}

NPH_HD int g6_len(const G6& g)
{
    const int sign = g.neg ? 1 : 0;
    if (g.X < -4 || g.X >= 6) return sign + g.nsig + (g.nsig > 1 ? 1 : 0) + 4;              // d[.ddd]e+XX
    if (g.X >= 0) return sign + (g.X + 1) + (g.nsig > g.X + 1 ? 1 + g.nsig - (g.X + 1) : 0);
    return sign + 2 + (-g.X - 1) + g.nsig;                                                  // 0.000ddd
}

NPH_HD char* put_g6(char* o, const G6& g)
{
    if (g.neg) *o++ = '-';
    char d[6];
    uint32_t q = g.q;
    for (int i = g.nsig - 1; i >= 0; --i) { d[i] = (char)('0' + (int)(q % 10u)); q /= 10u; }
    if (g.X < -4 || g.X >= 6) {
        *o++ = d[0];
        if (g.nsig > 1) { *o++ = '.'; for (int i = 1; i < g.nsig; ++i) *o++ = d[i]; }
        *o++ = 'e';
        const int ax = g.X < 0 ? -g.X : g.X;
        *o++ = g.X < 0 ? '-' : '+';
        *o++ = (char)('0' + ax / 10); *o++ = (char)('0' + ax % 10);
    } else if (g.X >= 0) {
        for (int i = 0; i <= g.X; ++i) *o++ = i < g.nsig ? d[i] : '0';
        if (g.nsig > g.X + 1) { *o++ = '.'; for (int i = g.X + 1; i < g.nsig; ++i) *o++ = d[i]; }
    } else {
        *o++ = '0'; *o++ = '.';
        for (int i = 0; i < -g.X - 1; ++i) *o++ = '0';
        for (int i = 0; i < g.nsig; ++i) *o++ = d[i];
    }
    return o;
}

// the value must be in the domain (g6_of(v).ok)
NPH_HD char* put_g6(char* o, float v) { return put_g6(o, g6_of(v)); }

// ---- eventalign.tsv ------------------------------------------------------------------------------------------------
// One row of the reference's emit_event_alignment_tsv (src/alignment/nanopolish_eventalign.cpp:398-484):
// "%s\t%d\t%s\t%zu|%s\t%c\t" contig, position, reference_kmer, read_idx | read_name (-n), strand;
// "%d\t%.2lf\t%.3lf\t%.5lf\t" event_index, event_level_mean, event_stdv, event_length;
// "%s\t%.2lf\t%.2lf\t%.2lf" model_kmer, model_mean, model_stdv, standardized_level;
// with --signal-index "\t%zu\t%zu" start_idx, end_idx; with --samples "\t" and the event's scaled samples, "%g" joined by ','.
// Every step of the arithmetic is one IEEE operation in the reference's types (built without FMA contraction on both sides).

// what a row needs of its read strand
struct EaRead {
    double scale, shift, drift, var, sqrt_var;             // SquiggleScalings; sqrt_var = sqrt(var)
    double sample_rate;
    uint64_t sample_start_time;
};

NPH_HD double ea_sqrt(double v)
{
#ifdef __CUDA_ARCH__
    return __dsqrt_rn(v);
#else
    return std::sqrt(v);
#endif
}

struct EaRowNums {
    float event_mean, model_mean, model_stdv, standard_level;   // the values (the C library's to print when ok is false)
    Fixed mean, stdv, dur, mmean, mstdv, stdl;                  // "%.2lf" "%.3lf" "%.5lf" "%.2lf" "%.2lf" "%.2lf"
    int std_inf;                                                // standardized_level: 0 finite, 1 "inf", -1 "-inf" ('B' states)
    uint64_t start_idx, end_idx;                                // --signal-index / --samples
    bool ok;                                                    // every number formats here; false: the C library's row
};

// ev_mean: the event's unscaled mean; level: its drift-scaled level (get_drift_scaled_level, read with --scale-events only);
// level_mean / level_stdv: the model's state for model_kmer (not read for a 'B' state); sample_idx: fill start_idx / end_idx
NPH_HD EaRowNums ea_row_numbers(float ev_mean, float level, float ev_stdv, float ev_duration, double start_time, char state,
                                double level_mean, double level_stdv, const EaRead& rd, bool scale_events, bool sample_idx)
{
    EaRowNums r;
    r.event_mean = ev_mean; r.model_mean = 0.0f; r.model_stdv = 0.0f;
#ifdef __CUDA_ARCH__
    if (scale_events) {
        // get_fully_scaled_level (squiggle_read.h:149-171): scale reads to the model, unscaled model parameters
        r.event_mean = (float)__ddiv_rn(__dsub_rn((double)level, rd.shift), rd.scale);
        if (state != 'B') { r.model_mean = (float)level_mean; r.model_stdv = (float)level_stdv; }
    } else if (state != 'B') {
        // get_scaled_gaussian_from_pore_model_state (squiggle_read.h:217-226): scale the model to the reads
        r.model_mean = (float)__dadd_rn(__dmul_rn(rd.scale, level_mean), rd.shift);
        r.model_stdv = (float)__dmul_rn(level_stdv, rd.var);
    }
    // float difference over a double product, narrowed to float (a 'B' state divides by zero)
    r.standard_level = (float)__ddiv_rn((double)__fsub_rn(r.event_mean, r.model_mean), __dmul_rn(rd.sqrt_var, (double)r.model_stdv));
#else
    if (scale_events) {
        const double centred = (double)level - rd.shift;
        r.event_mean = (float)(centred / rd.scale);
        if (state != 'B') { r.model_mean = (float)level_mean; r.model_stdv = (float)level_stdv; }
    } else if (state != 'B') {
        const double scaled = rd.scale * level_mean;
        r.model_mean = (float)(scaled + rd.shift);
        r.model_stdv = (float)(level_stdv * rd.var);
    }
    const float diff = r.event_mean - r.model_mean;
    const double denom = rd.sqrt_var * (double)r.model_stdv;
    r.standard_level = (float)((double)diff / denom);
#endif
    r.mean = fixed_of<2>(r.event_mean);
    r.stdv = fixed_of<3>(ev_stdv);
    r.dur = fixed_of<5>(ev_duration);
    r.mmean = fixed_of<2>(r.model_mean);
    r.mstdv = fixed_of<2>(r.model_stdv);
    uint32_t sbits;
    memcpy(&sbits, &r.standard_level, 4);
    const bool s_inf = (sbits << 1) == 0xff000000u;       // 0 / 0 gives a NaN whose printed sign is the host FPU's: not ok
    r.std_inf = !s_inf ? 0 : (sbits >> 31) ? -1 : 1;
    r.stdl = fixed_of<2>(r.standard_level);
    r.ok = r.mean.ok && r.stdv.ok && r.dur.ok && r.mmean.ok && r.mstdv.ok && (r.stdl.ok || s_inf);
    r.start_idx = 0; r.end_idx = 0;
    if (sample_idx) {
        // get_event_sample_idx (squiggle_read.cpp:393-428): size_t arithmetic
#ifdef __CUDA_ARCH__
        const double t0 = __dmul_rn(start_time, rd.sample_rate);
        const double t1 = __dmul_rn(__dadd_rn(start_time, (double)ev_duration), rd.sample_rate);
#else
        const double t0 = start_time * rd.sample_rate;
        const double end_time = start_time + (double)ev_duration;
        const double t1 = end_time * rd.sample_rate;
#endif
        const double lim = 9223372036854775808.0;          // 2^63: the conversion to size_t is defined below it
        if (t0 >= 0.0 && t0 < lim && t1 >= 0.0 && t1 < lim) {
            r.start_idx = (uint64_t)t0 - rd.sample_start_time;
            r.end_idx = (uint64_t)t1 - rd.sample_start_time;
        } else {
            r.ok = false;
        }
    }
    return r;
}

// get_scaled_samples_for_event's sample i (squiggle_read.cpp:399-416)
NPH_HD float ea_scaled_sample(float raw, uint64_t i, const EaRead& rd)
{
#ifdef __CUDA_ARCH__
    const double t = __ddiv_rn((double)(rd.sample_start_time + i), rd.sample_rate);
    double s = __dsub_rn((double)raw, rd.shift);
    s = __dsub_rn(s, __dmul_rn(__dsub_rn(t, __ddiv_rn((double)rd.sample_start_time, rd.sample_rate)), rd.drift));
    return (float)__ddiv_rn(s, rd.scale);
#else
    const double t = (double)(rd.sample_start_time + i) / rd.sample_rate;
    double s = (double)raw - rd.shift;
    const double elapsed = t - (double)rd.sample_start_time / rd.sample_rate;
    const double drifted = elapsed * rd.drift;
    s -= drifted;
    s /= rd.scale;
    return (float)s;
#endif
}

// The k-mer columns of the record at offset pos of a reference of n characters (upper case, ambiguity codes resolved) and its
// reverse complement rc_ref: reference_kmer is the k characters at pos, clipped at the end as substr clips; model_kmer is what
// HMMInputSequence::get_kmer hands the model: the same k-mer, for rc reads rc_ref's k-mer at n - pos - k, k times 'N' for a
// 'B' state.  pos + k <= n for every record of an alignment window.
struct EaKmers { const char* ref_kmer; uint32_t ref_kmer_len; const char* model_kmer; /* nullptr: k times 'N' */ };

NPH_HD EaKmers ea_kmers_at(const char* ref, const char* rc_ref, size_t n, size_t pos, uint32_t k, bool rc, char state)
{
    EaKmers km;
    const size_t len = pos <= n ? (k < n - pos ? k : n - pos) : 0;
    km.ref_kmer = ref + (len ? pos : 0);
    km.ref_kmer_len = (uint32_t)len;
    km.model_kmer = state == 'B' ? nullptr : rc ? rc_ref + (n - pos - k) : ref + pos;
    return km;
}

struct EaRow {
    const char* contig; uint32_t contig_len;
    int ref_position;
    EaKmers kmers; uint32_t k;
    const char* name; uint32_t name_len;          // -n; nullptr: read_idx as "%zu"
    uint64_t read_idx;
    char strand;                                   // 't' or 'c'
    int event_idx;
    bool signal_index;
};

// the row up to and excluding the sample column and the newline; r.ok must hold
NPH_HD uint32_t ea_row_len(const EaRow& w, const EaRowNums& r)
{
    uint32_t n = w.contig_len + 1u + (uint32_t)int_len(w.ref_position) + 1u + w.kmers.ref_kmer_len + 1u +
                 (w.name ? w.name_len : (uint32_t)ndigits(w.read_idx)) + 3u + (uint32_t)int_len(w.event_idx) + 1u +
                 (uint32_t)fixed_len<2>(r.mean) + 1u + (uint32_t)fixed_len<3>(r.stdv) + 1u + (uint32_t)fixed_len<5>(r.dur) + 1u + w.k + 1u +
                 (uint32_t)fixed_len<2>(r.mmean) + 1u + (uint32_t)fixed_len<2>(r.mstdv) + 1u +
                 (r.std_inf == 0 ? (uint32_t)fixed_len<2>(r.stdl) : r.std_inf > 0 ? 3u : 4u);
    if (w.signal_index) n += 2u + (uint32_t)ndigits(r.start_idx) + (uint32_t)ndigits(r.end_idx);
    return n;
}

NPH_HD char* put_ea_row(char* o, const EaRow& w, const EaRowNums& r)
{
    o = put_bytes(o, w.contig, w.contig_len); *o++ = '\t';
    o = put_int(o, w.ref_position); *o++ = '\t';
    o = put_bytes(o, w.kmers.ref_kmer, w.kmers.ref_kmer_len); *o++ = '\t';
    o = w.name ? put_bytes(o, w.name, w.name_len) : put_u64(o, w.read_idx);
    *o++ = '\t'; *o++ = w.strand; *o++ = '\t';
    o = put_int(o, w.event_idx); *o++ = '\t';
    o = put_fixed<2>(o, r.mean); *o++ = '\t';
    o = put_fixed<3>(o, r.stdv); *o++ = '\t';
    o = put_fixed<5>(o, r.dur); *o++ = '\t';
    if (w.kmers.model_kmer) o = put_bytes(o, w.kmers.model_kmer, w.k);
    else for (uint32_t i = 0; i < w.k; ++i) *o++ = 'N';
    *o++ = '\t';
    o = put_fixed<2>(o, r.mmean); *o++ = '\t';
    o = put_fixed<2>(o, r.mstdv); *o++ = '\t';
    if (r.std_inf == 0) o = put_fixed<2>(o, r.stdl);
    else { if (r.std_inf < 0) *o++ = '-'; *o++ = 'i'; *o++ = 'n'; *o++ = 'f'; }
    if (w.signal_index) { *o++ = '\t'; o = put_u64(o, r.start_idx); *o++ = '\t'; o = put_u64(o, r.end_idx); }
    return o;
}

} // namespace nph_tsv
