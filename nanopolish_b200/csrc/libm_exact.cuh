// libm_exact.cuh — expf and logf that return glibc's bits, on the host and on the device.
//
// The reference calls libm's expf / logf (through exp() and std::log() on float arguments) for every raw sample in the
// poly(A) segmentation HMM (src/nanopolish_polya_estimator.cpp:259-306, hmm/nanopolish_emissions.h:19-24).  glibc (2.28 and
// later, x86-64 and aarch64) computes both in double arithmetic with small tables — the algorithms of Arm's
// optimized-routines (MIT licence), sysdeps/ieee754/flt-32/e_expf.c and e_logf.c — and is NOT correctly rounded: about one
// float in 10^4 differs from the correctly rounded result.  A correctly rounded device function would therefore disagree
// with the reference on about 10^-3 of all samples.  Instead these are the same double-precision algorithms, operation for
// operation, with every multiply-add written as one explicit fma, which is how glibc's x86-64 FMA build (the variant an
// FMA-capable CPU runs) contracts them.  Each step is a single IEEE double operation, so the host build and the device
// build round identically.
//
// The claim is checked exhaustively, not argued: tests/cuda/check_libm_exact.cu compares nph_expf with the C library's expf
// on every float <= 0 (and -0, -inf, NaN) and nph_logf with logf on every float >= 0, on the host (CPU test) and on the
// device against the host libm of the GPU machine (GPU test).  A libm with another algorithm fails those checks loudly.
//
// Domains used by the poly(A) kernel (csrc/polya.cu): expf of (-0.5f*a)*a <= 0 (or NaN), logf of a non-negative mixture.
// Positive expf arguments and negative logf arguments are outside the checked domains and must not be passed.
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>

#if defined(__CUDA_ARCH__)
#define NPH_LX_FMA(a, b, c) __fma_rn((a), (b), (c))
#define NPH_LX_MUL(a, b) __dmul_rn((a), (b))
#define NPH_LX_ADD(a, b) __dadd_rn((a), (b))
#define NPH_LX_SUB(a, b) __dsub_rn((a), (b))
#else
#define NPH_LX_FMA(a, b, c) fma((a), (b), (c))
#define NPH_LX_MUL(a, b) ((a) * (b))
#define NPH_LX_ADD(a, b) ((a) + (b))
#define NPH_LX_SUB(a, b) ((a) - (b))
#endif

#if defined(__CUDACC__)
#define NPH_LX_HD __host__ __device__ __forceinline__
#else
#define NPH_LX_HD inline
#endif

namespace nph_libm {

NPH_LX_HD uint32_t f2u(float x)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__float_as_uint(x);
#else
    uint32_t u; memcpy(&u, &x, 4); return u;
#endif
}
NPH_LX_HD float u2f(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float x; memcpy(&x, &u, 4); return x;
#endif
}
NPH_LX_HD uint64_t d2u(double x)
{
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
NPH_LX_HD double u2d(uint64_t u)
{
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double x; memcpy(&x, &u, 8); return x;
#endif
}

// 2^(i/32) for i = 0..31, each as its double's bit pattern minus i << 47 (so that adding k << 47 scales by 2^(k/32))
#define NPH_EXP2F_TAB { \
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, \
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, \
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull, \
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, \
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull, \
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull, \
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, \
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull }

// logf's 16 subintervals of [0x3f330000, 0x3fb30000): {1/c, log(c)} with c near each centre
#define NPH_LOGF_TAB { \
    0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2, 0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2, \
    0x1.49539f0f010b0p+0, -0x1.01eae7f513a67p-2, 0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3, \
    0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3, 0x1.25e227b0b8ea0p+0, -0x1.1aa2bc79c8100p-3, \
    0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4, 0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4, \
    0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5, 0x1.0p+0, 0x0.0p+0, \
    0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5, 0x1.ca4b31f026aa0p-1, 0x1.c5e53aa362eb4p-4, \
    0x1.b2036576afce6p-1, 0x1.526e57720db08p-3, 0x1.9c2d163a1aa2dp-1, 0x1.bc2860d224770p-3, \
    0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2, 0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2 }

#if defined(__CUDACC__)
__constant__ const uint64_t k_exp2f_tab_dev[32] = NPH_EXP2F_TAB;
__constant__ const double k_logf_tab_dev[32] = NPH_LOGF_TAB;
#endif
static const uint64_t k_exp2f_tab_host[32] = NPH_EXP2F_TAB;
static const double k_logf_tab_host[32] = NPH_LOGF_TAB;

NPH_LX_HD uint64_t exp2f_tab(uint32_t i)
{
#if defined(__CUDA_ARCH__)
    return k_exp2f_tab_dev[i];
#else
    return k_exp2f_tab_host[i];
#endif
}
NPH_LX_HD double logf_tab(uint32_t i)
{
#if defined(__CUDA_ARCH__)
    return k_logf_tab_dev[i];
#else
    return k_logf_tab_host[i];
#endif
}

} // namespace nph_libm

// expf(x) for x <= 0 (any such float, -inf and NaN included): glibc's e_expf.c.
//   x*32/ln2 = k + r, |r| <= 1/2;  exp(x) = 2^(k/32) * 2^(r/32) ~= s * (C0 r^3 + C1 r^2 + C2 r + 1)
NPH_LX_HD float nph_expf(float x)
{
    using namespace nph_libm;
    const uint32_t abstop = (f2u(x) >> 20) & 0x7ff;
    if (abstop >= 0x42b) {                       // |x| >= 88 or NaN (0x42b = top12(88.0f))
        if (f2u(x) == 0xff800000u) return 0.0f;  // -inf
        if (abstop >= 0x7f8) return x + x;       // NaN
        if (x < -0x1.9fe368p6f) return 0.0f;     // below log(2^-150): underflows to +0
    }
    const double xd = (double)x;
    const double shift = 0x1.8p+52, invln2n = 0x1.71547652b82fep+5;
    double kd = NPH_LX_FMA(invln2n, xd, shift);  // round(x*32/ln2) in the low bits
    const uint64_t ki = d2u(kd);
    kd = NPH_LX_SUB(kd, shift);
    const double r = NPH_LX_FMA(invln2n, xd, -kd);
    uint64_t t = exp2f_tab((uint32_t)(ki % 32));
    t += ki << 47;
    const double s = u2d(t);
    const double z = NPH_LX_FMA(0x1.c6af84b912394p-20, r, 0x1.ebfce50fac4f3p-13);
    const double r2 = NPH_LX_MUL(r, r);
    double y = NPH_LX_FMA(0x1.62e42ff0c52d6p-6, r, 1.0);
    y = NPH_LX_FMA(z, r2, y);
    y = NPH_LX_MUL(y, s);
    return (float)y;
}

// logf(x) for x >= 0 (any such float, +inf and NaN included): glibc's e_logf.c.
//   x = 2^k z, z in [0x3f330000, 2*0x3f330000);  log(x) = log1p(z/c - 1) + log(c) + k ln2
NPH_LX_HD float nph_logf(float x)
{
    using namespace nph_libm;
    uint32_t ix = f2u(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {
        if (ix * 2 == 0) return -INFINITY;                       // +-0
        if (ix == 0x7f800000u) return x;                          // +inf
        if ((ix & 0x80000000u) || ix * 2 >= 0xff000000u) return (x - x) / (x - x);   // negative or NaN
        ix = f2u(x * 0x1p23f);                                    // subnormal: normalise (exact)
        ix -= 23u << 23;
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const uint32_t i = (tmp >> 19) % 16;
    const int32_t k = (int32_t)tmp >> 23;
    const uint32_t iz = ix - (tmp & 0xff800000u);
    const double invc = logf_tab(2 * i), logc = logf_tab(2 * i + 1);
    const double z = (double)u2f(iz);
    const double ln2 = 0x1.62e42fefa39efp-1;
    const double r = NPH_LX_FMA(z, invc, -1.0);
    const double y0 = NPH_LX_FMA((double)k, ln2, logc);
    const double r2 = NPH_LX_MUL(r, r);
    double y = NPH_LX_FMA(0x1.5575b0be00b6ap-2, r, -0x1.ffffef20a4123p-2);
    y = NPH_LX_FMA(-0x1.00ea348b88334p-2, r2, y);
    y = NPH_LX_FMA(y, r2, NPH_LX_ADD(y0, r));
    return (float)y;
}
