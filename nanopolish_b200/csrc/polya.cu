// polya.cu — nanopolish polya on the device: poly(A) tail segmentation and length of a batch of reads in one call
// (src/nanopolish_polya_estimator.cpp; the per-read part of estimate_polya_for_single_read, :786-813), and nanopolish
// detect-polyi, its sibling for poly(I) tails (src/nanopolish_detect_polyi.cpp; dpi_estimate_polya_for_single_read, :1061-1095).
//
// One CTA per read, reads launched longest first.  Warp 0 walks the 6-state Viterbi of SegmentationHMM (:372-463) over the
// read's samples on one lane; warps 1..3 compute the six emission log-probabilities (:259-306) of the NEXT tile of samples
// into the other half of a double buffer in shared memory, so the eight expf / logf per sample stay off the walk.  Before the
// walk the whole CTA computes the read rate (:564-599) by a radix selection of the median per-k-mer duration.  After it the
// walking lane applies segment_squiggle's sentinel rule (:500-506), estimate_polya_length (:638-662) and the QC (:672-722).
//
// No trace is stored.  The reference backtracks p[n-1] = T, p[j] = bptr[j][p[j+1]] for j = n-2 .. 1 (the pointer table of
// step j, one step early against textbook Viterbi), p[0] = START, and segment_squiggle then only needs four "last index of a
// label pair" values and a CLIFF count.  So the walk carries, for each state s, the summary of the path p[0..j] that the
// backtrack would produce if p[j+1] were s; step j composes it with bptr[j] (a select per field), and after step n-2 the
// summary of s = TRANSCRIPT is segment_squiggle's answer.  The path's order S -> L -> A -> (P <-> C) -> T leaves 16 live
// fields (a state's chains can only have passed the boundaries before it).  Row n-1 of the Viterbi is never read.
//
// Every floating-point operation is spelled as the reference rounds it (float for the HMM, double for the length and QC;
// max is std::max, (a < b) ? b : a; the backpointer rules use strict < in the reference's precedence), and expf / logf are
// glibc's (libm_exact.cuh).
//
// detect-polyi is the same kernel instantiated with kPolyi (DESIGN §15).  Its segmentation HMM (DPISegmentationHMM,
// :177-518) differs from polya's only in the POLYA emission, an even mixture of two Gaussians (:291-295).  After the walk the
// whole CTA runs BernoulliHMM::segmentation (:728-756) over the tail's samples in two passes through the same double buffer:
// warps 1..3 scale the samples tile by tile while lane 0 takes their sequential float mean; then warps 1..3 compute each
// centred sample's log-likelihood-ratio bit tile by tile while lane 0 walks the 2-state Viterbi one tile behind.  Its labels
// are I..I A..A (A is absorbing), so the walk folds the backtrack into one index: the first A of the path that ends in A.
#include "nph_internal.cuh"
#include "libm_exact.cuh"

#include <cmath>
#include <type_traits>
#include <vector>

namespace {

constexpr int kTile = 256;            // samples per emission tile
constexpr int kEmitWarps = 3;
constexpr int kThreads = 32 * (1 + kEmitWarps);
enum { ST_S = 0, ST_L, ST_A, ST_P, ST_C, ST_T, N_ST };
// G_P1 exists in detect-polyi's table only
enum { G_S = 0, G_L, G_A0, G_A1, G_P, G_T0, G_T1, G_P1 };
template <bool kPolyi> constexpr int n_gauss = kPolyi ? G_P1 + 1 : G_P1;

// The reference's emission parameters (:232-250; detect_polyi.cpp:233-255 adds P1), before scaling
__constant__ const float k_gauss[G_P1 + 1][2] = {
    {70.2737f, 3.7743f}, {110.973f, 5.237f}, {79.347f, 8.3702f}, {63.3126f, 2.7464f},
    {108.883f, 3.257f}, {79.679f, 6.966f}, {105.784f, 16.022f}, {108.498f, 5.257f}};

template <int NG>
struct Gauss {
    float mean[NG], stdv[NG], log_stdv[NG], coef[NG];   // coef = inv_sqrt_2pi / stdv, as normal_pdf forms it
    float log_inv_sqrt_2pi;
};

template <bool kPolyi> using TailResult = typename std::conditional<kPolyi, nph_polyi_result, nph_polya_result>::type;

template <bool kPolyi>
struct PolyaParams {
    const float* raw;
    const float* dur;
    const nph_event_range* b2e;
    const nph_polya_job* jobs;
    const uint32_t* order;
    TailResult<kPolyi>* out;
    float log_inv_sqrt_2pi;           // (float)log(0.3989422804014327) (hmm/nanopolish_emissions.h:43), host libm
};

// normal_pdf (emissions.h:19-24): inv_sqrt_2pi / stdv * exp(-0.5f * a * a)
template <int NG>
__device__ __forceinline__ float normal_pdf(float x, const Gauss<NG>& g, int k)
{
    const float a = __fdiv_rn(__fsub_rn(x, g.mean[k]), g.stdv[k]);
    return __fmul_rn(g.coef[k], nph_expf(__fmul_rn(__fmul_rn(-0.5f, a), a)));
}
// log_normal_pdf (emissions.h:51-55): log_inv_sqrt_2pi - log_stdv + (-0.5f * a * a)
template <int NG>
__device__ __forceinline__ float log_normal_pdf(float x, const Gauss<NG>& g, int k)
{
    const float a = __fdiv_rn(__fsub_rn(x, g.mean[k]), g.stdv[k]);
    return __fadd_rn(__fsub_rn(g.log_inv_sqrt_2pi, g.log_stdv[k]), __fmul_rn(__fmul_rn(-0.5f, a), a));
}

// emit_log_proba of all six states (:259-306; detect_polyi.cpp:263-312)
template <bool kPolyi>
__device__ __forceinline__ void emissions(float x, const Gauss<n_gauss<kPolyi>>& g, float e[N_ST])
{
    const float xx = (x > 200.0f || x < 40.0f) ? 100.0f : x;
    e[ST_S] = nph_logf(__fadd_rn(__fmul_rn(0.50f, normal_pdf(xx, g, G_S)), __fmul_rn(0.50f, 0.00476f)));
    e[ST_L] = log_normal_pdf(xx, g, G_L);
    e[ST_A] = nph_logf(__fadd_rn(__fmul_rn(0.874f, normal_pdf(xx, g, G_A0)), __fmul_rn(0.126f, normal_pdf(xx, g, G_A1))));
    if constexpr (kPolyi)
        e[ST_P] = nph_logf(__fadd_rn(__fmul_rn(0.500f, normal_pdf(xx, g, G_P)), __fmul_rn(0.500f, normal_pdf(xx, g, G_P1))));
    else
        e[ST_P] = log_normal_pdf(xx, g, G_P);
    e[ST_C] = (xx > 70.0f && xx < 140.0f) ? -4.2485f : -INFINITY;
    e[ST_T] = nph_logf(__fadd_rn(__fmul_rn(0.346f, normal_pdf(xx, g, G_T0)), __fmul_rn(0.654f, normal_pdf(xx, g, G_T1))));
}

// the transition log-probabilities (:313-326): logf of the float probabilities, -inf for zeros
__device__ __forceinline__ float log_prob(float p) { return p > 0.00f ? nph_logf(p) : -INFINITY; }

__device__ __forceinline__ float smax(float a, float b) { return (a < b) ? b : a; }   // std::max

// segment_squiggle's sentinel rule (:500-506): a boundary left at its initial value moves all three to the read's end
__device__ __forceinline__ void sentinel_rule(uint64_t& ld, uint64_t& ad, uint64_t& pa, uint32_t n)
{
    if (ld == 1 || ad == 2 || pa == 3) { ld = (uint64_t)n - 3; ad = (uint64_t)n - 2; pa = (uint64_t)n - 1; }
}

// BernoulliHMM's bit of one scaled tail sample (detect_polyi.cpp:663-671): recentred on 108, clamped like the segmentation,
// then log normal_pdf under the UNSCALED poly(I) and poly(A) Gaussians (:563-564, :581-603); (lI / lA) > 1, so the NaN of
// -inf / -inf (both densities underflow) is 0
__device__ __forceinline__ float unscaled_pdf(float x, float mean, float stdv)
{
    const float a = __fdiv_rn(__fsub_rn(x, mean), stdv);
    return __fmul_rn(__fdiv_rn((float)0.3989422804014327, stdv), nph_expf(__fmul_rn(__fmul_rn(-0.5f, a), a)));
}
__device__ __forceinline__ bool bernoulli_bit(float y, float mean)
{
    const float s = __fadd_rn(__fsub_rn(y, mean), 108.000f);
    const float xx = (s > 200.0f || s < 40.0f) ? 100.0f : s;
    const float lI = nph_logf(unscaled_pdf(xx, 108.498f, 5.257f));
    const float lA = nph_logf(unscaled_pdf(xx, 108.883f, 3.257f));
    return __fdiv_rn(lI, lA) > 1.0f;
}

// total order of doubles as unsigned keys (the median's radix selection)
__device__ __forceinline__ uint64_t dkey(double d)
{
    const uint64_t u = (uint64_t)__double_as_longlong(d);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double dunkey(uint64_t k)
{
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

template <bool kPolyi>
__global__ void __launch_bounds__(kThreads) polya_kernel(const PolyaParams<kPolyi> p)
{
    __shared__ float s_em[2][N_ST][kTile];
    __shared__ Gauss<n_gauss<kPolyi>> s_g;
    __shared__ uint32_t s_hist[256];
    __shared__ uint32_t s_sel, s_rank;
    __shared__ double s_rate;

    const uint32_t jid = p.order[blockIdx.x];
    const nph_polya_job jb = p.jobs[jid];
    const int tid = threadIdx.x, warp = tid >> 5;
    const uint32_t n = jb.n_samples;
    const float* x = p.raw + jb.sample_off;

    // ---- per-read constants (:310-354): (float)scale, shift, var; mean' = shift + scale*mean, stdv' = var*stdv ----
    if (tid < n_gauss<kPolyi>) {
        const float scale = (float)jb.scale, shift = (float)jb.shift, var = (float)jb.var;
        const float sd = __fmul_rn(var, k_gauss[tid][1]);
        s_g.mean[tid] = __fadd_rn(shift, __fmul_rn(scale, k_gauss[tid][0]));
        s_g.stdv[tid] = sd;
        s_g.log_stdv[tid] = nph_logf(sd);
        s_g.coef[tid] = __fdiv_rn((float)0.3989422804014327, sd);
        if (tid == 0) s_g.log_inv_sqrt_2pi = p.log_inv_sqrt_2pi;
    }

    // ---- read rate (:564-599): durations per k-mer in FP64, summed in event order; element [n/2] of the sorted list ----
    {
        const nph_event_range* map = p.b2e + jb.rank_off;
        const float* dur = p.dur + jb.event_off;
        const uint32_t nk = jb.n_kmers;
        uint64_t prefix = 0, mask = 0;
        if (tid == 0) s_rank = nk / 2;
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int b = tid; b < 256; b += kThreads) s_hist[b] = 0;
            __syncthreads();
            for (uint32_t i = tid; i < nk; i += kThreads) {
                const nph_event_range r = map[i];
                double d = 0.0;
                if (r.start != -1)
                    for (int32_t e = r.start; e <= r.stop; ++e) d = __dadd_rn(d, (double)dur[e]);
                const uint64_t key = dkey(d);
                if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                uint32_t k = s_rank, b = 0;
                for (; b < 255 && s_hist[b] <= k; ++b) k -= s_hist[b];
                s_sel = b; s_rank = k;
            }
            __syncthreads();
            prefix |= (uint64_t)s_sel << shift;
            mask |= 255ull << shift;
        }
        if (tid == 0) s_rate = __ddiv_rn(1.0, dunkey(prefix));
    }

    // ---- emissions of tile t into buffer t & 1: step i uses sample i, row 0 uses the LAST sample (:385-386) ----
    // Only steps 0 .. n-2 are needed: row n-1's scores and pointers are never read by the backtrack.
    const uint32_t n_steps = n - 1;
    const uint32_t n_tiles = (n_steps + kTile - 1) / kTile;
    auto fill = [&](uint32_t t) {
        float (*em)[kTile] = s_em[t & 1];
        for (uint32_t o = tid - 32; o < kTile; o += 32 * kEmitWarps) {
            const uint32_t i = t * kTile + o;
            if (i >= n_steps) break;
            float e[N_ST];
            emissions<kPolyi>(x[i == 0 ? n - 1 : i], s_g, e);
#pragma unroll
            for (int s = 0; s < N_ST; ++s) em[s][o] = e[s];
        }
    };
    if (warp > 0) fill(0);
    __syncthreads();

    // the walk's state (warp 0, lane 0): scores, and the path summaries (see the file comment).  Field names: <slot><field>
    // with fields s(tart) l(eader) a(dapter) p(olya) c(liffs); absent fields are still their sentinels {0, 1, 2, 3, 0}.
    float vS = 0.f, vL = 0.f, vA = 0.f, vP = 0.f, vC = 0.f, vT = 0.f;
    uint32_t Ls = 0, As = 0, Al = 1, Ps = 0, Pl = 1, Pa = 2, Pc = 0, Cs = 0, Cl = 1, Ca = 2, Cc = 0;
    uint32_t Ts = 0, Tl = 1, Ta = 2, Tp = 3, Tc = 0;
    float lSS = 0.f, lSL = 0.f, lLL = 0.f, lLA = 0.f, lAA = 0.f, lAP = 0.f, lPP = 0.f, lPC = 0.f, lPT = 0.f, lCP = 0.f, lCC = 0.f, lTT = 0.f;
    if (tid == 0) {
        lSS = log_prob(0.10f); lSL = log_prob(0.90f); lLL = log_prob(0.90f); lLA = log_prob(0.10f);
        lAA = log_prob(0.95f); lAP = log_prob(0.05f); lPP = log_prob(0.89f); lPC = log_prob(0.01f); lPT = log_prob(0.10f);
        lCP = log_prob(0.99f); lCC = log_prob(0.01f); lTT = log_prob(1.00f);
    }

    for (uint32_t t = 0; t < n_tiles; ++t) {
        if (tid == 0) {
            const float (*em)[kTile] = s_em[t & 1];
            const uint32_t i0 = t * kTile, i1 = min(n_steps, i0 + kTile);
            uint32_t i = i0;
            if (i == 0) {
                // row 0: log_start_probs (logf(1) = 0 for START, -inf for LEADER) + emissions of samples[n-1]
                vS = __fadd_rn(log_prob(1.00f), em[ST_S][0]);
                vL = __fadd_rn(-INFINITY, em[ST_L][0]);
                vA = vP = vC = vT = -INFINITY;
                i = 1;
            }
            for (; i < i1; ++i) {
                const uint32_t o = i - i0;
                const float s_to_s = __fadd_rn(vS, lSS), s_to_l = __fadd_rn(vS, lSL);
                const float l_to_l = __fadd_rn(vL, lLL), l_to_a = __fadd_rn(vL, lLA);
                const float a_to_a = __fadd_rn(vA, lAA), a_to_p = __fadd_rn(vA, lAP);
                const float p_to_p = __fadd_rn(vP, lPP), p_to_c = __fadd_rn(vP, lPC), p_to_t = __fadd_rn(vP, lPT);
                const float c_to_c = __fadd_rn(vC, lCC), c_to_p = __fadd_rn(vC, lCP);
                const float t_to_t = __fadd_rn(vT, lTT);
                vS = __fadd_rn(s_to_s, em[ST_S][o]);
                vL = __fadd_rn(smax(l_to_l, s_to_l), em[ST_L][o]);
                vA = __fadd_rn(smax(a_to_a, l_to_a), em[ST_A][o]);
                vP = __fadd_rn(smax(p_to_p, smax(a_to_p, c_to_p)), em[ST_P][o]);
                vC = __fadd_rn(smax(c_to_c, p_to_c), em[ST_C][o]);
                vT = __fadd_rn(smax(p_to_t, t_to_t), em[ST_T][o]);
                // backpointers of step i (:411-444) folded into the summaries; i <= n-2 always holds here
                const bool bL_is_L = s_to_l < l_to_l;
                const bool bA_is_A = l_to_a < a_to_a;
                const bool bP_is_P = (a_to_p < p_to_p) && (c_to_p < p_to_p);
                const bool bP_is_A = !bP_is_P && (p_to_p < a_to_p) && (c_to_p < a_to_p);
                const bool bC_is_C = p_to_c < c_to_c;
                const bool bT_is_T = p_to_t < t_to_t;
                // T <- T | P (P -> T at i)
                if (!bT_is_T) { Ts = Ps; Tl = Pl; Ta = Pa; Tp = i; Tc = Pc; }
                // C <- C (one more cliff) | P; P <- P | A (A -> P at i) | C (one more cliff): both read the old P and C
                const uint32_t oPs = Ps, oPl = Pl, oPa = Pa, oPc = Pc;
                if (!bP_is_P) {
                    if (bP_is_A) { Ps = As; Pl = Al; Pa = i; Pc = 0; }
                    else         { Ps = Cs; Pl = Cl; Pa = Ca; Pc = Cc + 1; }
                }
                if (bC_is_C) Cc = Cc + 1;
                else { Cs = oPs; Cl = oPl; Ca = oPa; Cc = oPc; }
                // A <- A | L (L -> A at i); L <- L | S (S -> L at i)
                if (!bA_is_A) { As = Ls; Al = i; }
                if (!bL_is_L) Ls = i;
            }
        } else if (warp > 0 && t + 1 < n_tiles) {
            fill(t + 1);
        }
        __syncthreads();
    }

    // ---- detect-polyi: BernoulliHMM::segmentation(sr, adapter + 1, polya) (detect_polyi.cpp:728-756) ----
    int32_t b_polyi = -1, b_polya = -1;   // BernoulliSegmentation {-1, -1}: not found (lane 0)
    if constexpr (kPolyi) {
        __shared__ uint32_t s_b0, s_m;
        __shared__ float s_mean;
        if (tid == 0) {
            uint64_t ld = Tl, ad = Ta, pa = Tp;
            sentinel_rule(ld, ad, pa, n);
            // int start / stop: exact, as the host refuses n >= 2^31; polya >= adapter + 1 always
            s_b0 = (uint32_t)(ad + 1);
            s_m = (uint32_t)(pa - (ad + 1));
        }
        __syncthreads();
        const uint32_t b0 = s_b0, m = s_m;
        if (m >= 100) {                                        // stop - start < 100: not found (:732-734)
            constexpr uint32_t kFlat = N_ST * kTile;           // one half of the double buffer, as one flat tile
            const uint32_t n_ft = (m + kFlat - 1) / kFlat;
            // pass 0: (x - shift) / scale in double with the unrounded scalings, narrowed to float (:737-740); pass 1: the bit
            auto fill = [&](uint32_t t, bool bits, float mean) {
                float* buf = &s_em[t & 1][0][0];
                for (uint32_t o = tid - 32; o < kFlat; o += 32 * kEmitWarps) {
                    const uint32_t i = t * kFlat + o;
                    if (i >= m) break;
                    const float y = __double2float_rn(__ddiv_rn(__dsub_rn((double)x[b0 + i], jb.shift), jb.scale));
                    buf[o] = bits ? (bernoulli_bit(y, mean) ? 1.0f : 0.0f) : y;
                }
            };
            // pass 0: instance_mean, a sequential float sum divided by (float)size (:655-659)
            if (warp > 0) fill(0, false, 0.0f);
            __syncthreads();
            float sum = 0.0f;
            for (uint32_t t = 0; t < n_ft; ++t) {
                if (tid == 0) {
                    const float* buf = &s_em[t & 1][0][0];
                    const uint32_t o1 = min(kFlat, m - t * kFlat);
                    for (uint32_t o = 0; o < o1; ++o) sum = __fadd_rn(sum, buf[o]);
                } else if (warp > 0 && t + 1 < n_ft) {
                    fill(t + 1, false, 0.0f);
                }
                __syncthreads();
            }
            if (tid == 0) s_mean = __fdiv_rn(sum, __uint2float_rn(m));
            __syncthreads();
            const float mean = s_mean;
            // pass 1: BernoulliHMM::viterbi (:678-725).  first_a is the first A of the backtracked path ending in A: the
            // backpointer of step i into A is I iff a2a < i2a, and the backtrack reads those of steps 1 .. m-2 (regions[0]
            // stays I, so a path in A at step 1 starts A there)
            if (warp > 0) fill(0, true, mean);
            __syncthreads();
            float vI = 0.0f, vA = 0.0f, lII = 0.0f, lIA = 0.0f, lAA = 0.0f, eI1 = 0.0f, eI0 = 0.0f, eA1 = 0.0f, eA0 = 0.0f;
            uint32_t first_a = 1;
            if (tid == 0) {
                lII = log_prob(0.90f); lIA = log_prob(0.10f); lAA = log_prob(1.00f);
                eI1 = nph_logf(0.72304f); eI0 = nph_logf(__fsub_rn(1.0f, 0.72304f));
                eA1 = nph_logf(0.92154f); eA0 = nph_logf(__fsub_rn(1.0f, 0.92154f));
            }
            for (uint32_t t = 0; t < n_ft; ++t) {
                if (tid == 0) {
                    const float* buf = &s_em[t & 1][0][0];
                    const uint32_t i0 = t * kFlat, o1 = min(kFlat, m - i0);
                    uint32_t o = 0;
                    if (t == 0) {
                        // row 0: log_start_probs {logf(1), -inf} + the emissions of bit 0
                        vI = __fadd_rn(log_prob(1.00f), buf[0] != 0.0f ? eI1 : eI0);
                        vA = -INFINITY;
                        o = 1;
                    }
                    for (; o < o1; ++o) {
                        const uint32_t i = i0 + o;
                        const bool one = buf[o] != 0.0f;
                        const float i2i = __fadd_rn(vI, lII), i2a = __fadd_rn(vI, lIA), a2a = __fadd_rn(vA, lAA);
                        vI = __fadd_rn(i2i, one ? eI1 : eI0);
                        vA = __fadd_rn(smax(i2a, a2a), one ? eA1 : eA0);
                        if (a2a < i2a && i + 1 < m) first_a = i + 1;
                    }
                } else if (warp > 0 && t + 1 < n_ft) {
                    fill(t + 1, true, mean);
                }
                __syncthreads();
            }
            // the last row's state is A iff vI < vA (:710-716); labels I..I A..A give polyi = polya - 1
            if (vI < vA) { b_polya = (int32_t)first_a; b_polyi = (int32_t)first_a - 1; }
            else         { b_polyi = (int32_t)m - 1; }
        }
    }

    if (tid != 0) return;
    // ---- segment_squiggle's result (:474-507), estimate_polya_length, QC (size_t arithmetic as in the reference) ----
    uint64_t st = Ts, ld = Tl, ad = Ta, pa = Tp;
    sentinel_rule(ld, ad, pa, n);
    const double rate = s_rate;
    const double polya_duration = __ddiv_rn(__ull2double_rn(pa - (ad + 1)), jb.sample_rate);
    const double len = __dadd_rn(__dmul_rn(polya_duration, rate), -5.0);
    const double polya_length = (0.0 < len) ? len : 0.0;                 // std::max(0.0, len): NaN gives 0
    const double n_adapter = __ull2double_rn((ad + 1) - ld), n_polya = __ull2double_rn(pa - (ad + 1));
    const double adapter_length = __dmul_rn(__ddiv_rn(__ull2double_rn(ad - (ld - 1)), jb.sample_rate), rate);
    int32_t qc = NPH_POLYA_PASS;
    if (n_adapter < 200.0 || n_polya < 200.0) qc = NPH_POLYA_NOREGION;
    else if (adapter_length > 300.0) qc = NPH_POLYA_ADAPTER;
    else if (jb.suffix_clip > 200) qc = NPH_POLYA_SUFFCLIP;
    nph_polya_result r;
    r.start = st; r.leader = ld; r.adapter = ad; r.polya = pa; r.cliffs = Tc;
    r.read_rate = rate; r.polya_length = polya_length; r.qc = qc; r.reserved = 0;
    if constexpr (kPolyi) {
        // post_boolhmm_detetection_qc(segmentation, (int)(polya - (adapter + 1))) (detect_polyi.cpp:973-997, :1095)
        const int32_t region_length = (int32_t)(pa - (ad + 1));
        const bool polyi_found = b_polyi > 200;
        const bool polya_found = b_polya > 0 && region_length - b_polya > 200;
        nph_polyi_result q;
        q.seg = r; q.polyi_last = b_polyi; q.polya_first = b_polya; q.reserved = 0;
        q.detected = polyi_found ? (polya_found ? NPH_POLYI_A_PLUS_I : NPH_POLYI_POLYI_ONLY)
                                 : (polya_found ? NPH_POLYI_POLYA_ONLY : NPH_POLYI_NONE);
        p.out[jid] = q;
    } else {
        p.out[jid] = r;
    }
}

// Both entry points: job validation, the failed-load results, longest-first order, the d_polya carve, the uploads and the launch
template <bool kPolyi>
int polya_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_polya_job* jobs, size_t n_jobs,
                const float* ev_duration, size_t n_events_total, const nph_event_range* base_to_event, size_t n_ranks_total,
                TailResult<kPolyi>* results_out)
{
    using Result = TailResult<kPolyi>;
    if (!ctx) return NPH_ERR_INVALID;
    if (n_jobs == 0) return NPH_OK;
    if (!jobs || !results_out) return NPH_ERR_INVALID;
    std::vector<uint32_t> live;
    std::vector<uint32_t> len;
    for (size_t j = 0; j < n_jobs; ++j) {
        const nph_polya_job& jb = jobs[j];
        if (!jb.loaded || jb.n_events == 0) continue;         // events[0].empty(): READ_FAILED_LOAD (:762)
        if (!raw || !ev_duration || !base_to_event) return NPH_ERR_INVALID;
        if (kPolyi && jb.n_samples >= (1u << 31)) return NPH_ERR_INVALID;   // BernoulliHMM::segmentation's int start / stop
        if (jb.n_samples < 2 || !nph_slice_ok(jb.sample_off, jb.n_samples, n_samples_total) ||
            !nph_kmers_ok(jb.rank_off, jb.n_kmers, n_ranks_total) || !nph_slice_ok(jb.event_off, jb.n_events, n_events_total))
            return NPH_ERR_INVALID;
        for (uint32_t k = 0; k < jb.n_kmers; ++k) {
            const nph_event_range r = base_to_event[jb.rank_off + k];
            if (r.start != -1 && !(r.start >= 0 && r.start <= r.stop && (uint32_t)r.stop < jb.n_events)) return NPH_ERR_INVALID;
            // a NaN duration in a mapped span: the reference's sort of the per-k-mer durations has no defined order
            if (r.start != -1)
                for (int32_t e = r.start; e <= r.stop; ++e)
                    if (std::isnan(ev_duration[jb.event_off + e])) return NPH_ERR_INVALID;
        }
        live.push_back((uint32_t)j);
        len.push_back(jb.n_samples);
    }
    for (size_t j = 0; j < n_jobs; ++j) {
        nph_polya_result r{};
        r.read_rate = -1.0; r.polya_length = -1.0; r.qc = NPH_POLYA_READ_FAILED_LOAD;
        if constexpr (kPolyi) results_out[j] = nph_polyi_result{r, -1, -1, -1, 0};
        else results_out[j] = r;
    }
    if (live.empty()) { nph_timing_events(ctx, 0); return NPH_OK; }
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));

    // longest read first: it sets the batch's latency
    const std::vector<uint32_t> by_len = nph_longest_first(len);
    std::vector<uint32_t> order(live.size());
    for (size_t t = 0; t < live.size(); ++t) order[t] = live[by_len[t]];

    float* d_raw; float* d_dur; nph_event_range* d_b2e; nph_polya_job* d_jobs; uint32_t* d_order; Result* d_out;
    NPH_TRY(nph_carve(ctx, ctx->d_polya, [&](NphArena& a) {
        d_raw = a.take<float>(n_samples_total);
        d_dur = a.take<float>(n_events_total);
        d_b2e = a.take<nph_event_range>(n_ranks_total);
        d_jobs = a.take<nph_polya_job>(n_jobs);
        d_order = a.take<uint32_t>(order.size());
        d_out = a.take<Result>(n_jobs);
    }));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_raw, raw, sizeof(float) * n_samples_total, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_dur, ev_duration, sizeof(float) * n_events_total, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_b2e, base_to_event, sizeof(nph_event_range) * n_ranks_total, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_jobs, jobs, sizeof(nph_polya_job) * n_jobs, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_order, order.data(), sizeof(uint32_t) * order.size(), cudaMemcpyHostToDevice, ctx->stream));

    PolyaParams<kPolyi> pp;
    pp.raw = d_raw; pp.dur = d_dur; pp.b2e = d_b2e; pp.jobs = d_jobs; pp.order = d_order; pp.out = d_out;
    pp.log_inv_sqrt_2pi = (float)std::log(0.3989422804014327);
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    polya_kernel<kPolyi><<<(unsigned)order.size(), kThreads, 0, ctx->stream>>>(pp);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    std::vector<Result> res(n_jobs);
    NPH_CUDA(ctx, cudaMemcpyAsync(res.data(), d_out, sizeof(Result) * n_jobs, cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // order[] and res must outlive the copies
    for (uint32_t j : live) results_out[j] = res[j];
    nph_timing_events(ctx, 1);
    return NPH_OK;
}

} // namespace

extern "C" int nph_polya_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_polya_job* jobs, size_t n_jobs,
                               const float* ev_duration, size_t n_events_total, const nph_event_range* base_to_event, size_t n_ranks_total,
                               nph_polya_result* results_out)
{
    return polya_batch<false>(ctx, raw, n_samples_total, jobs, n_jobs, ev_duration, n_events_total, base_to_event, n_ranks_total,
                              results_out);
}

extern "C" int nph_detect_polyi_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_polya_job* jobs, size_t n_jobs,
                                      const float* ev_duration, size_t n_events_total, const nph_event_range* base_to_event,
                                      size_t n_ranks_total, nph_polyi_result* results_out)
{
    return polya_batch<true>(ctx, raw, n_samples_total, jobs, n_jobs, ev_duration, n_events_total, base_to_event, n_ranks_total,
                             results_out);
}
