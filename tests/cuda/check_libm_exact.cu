// check_libm_exact.cu — nph_expf / nph_logf (csrc/libm_exact.cuh) against the C library's expf / logf on EVERY float of
// their domains: expf on all 2^31 bit patterns with the sign bit set (-0 .. -inf and the negative NaNs) plus +0, logf on all
// 2^31 patterns without it (+0 .. +inf and the positive NaNs).  NaN results compare equal to NaN.
//   --host    the host build of the two functions (no device needed)
//   --device  the device build, computed on GPU 0 in chunks, against this machine's libm
// Prints "expf: N bad, logf: M bad" and exits 0 only if both are 0.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "libm_exact.cuh"

// the C library's functions, called through pointers so that nothing is folded at compile time
static float (*volatile g_expf)(float) = expf;
static float (*volatile g_logf)(float) = logf;

static inline bool same(float a, float b)
{
    uint32_t ua, ub;
    memcpy(&ua, &a, 4); memcpy(&ub, &b, 4);
    return ua == ub || (std::isnan(a) && std::isnan(b));
}

// pattern of the i-th float of a domain: expf takes 0x80000000 + i (i < 2^31) and +0 last; logf takes i
static inline uint32_t pattern(int fn, uint64_t i) { return fn == 0 ? (i < 0x80000000ull ? 0x80000000u + (uint32_t)i : 0u) : (uint32_t)i; }
static const uint64_t kDomain[2] = {0x80000001ull, 0x80000000ull};

static long long report(const char* name, int fn, uint64_t i, float got, float want, long long bad)
{
    if (bad < 5) {
        uint32_t u = pattern(fn, i);
        float x; memcpy(&x, &u, 4);
        printf("  %s(%a) = %a, libm %a\n", name, x, got, want);
    }
    return 1;
}

static int run_host()
{
    long long bad[2] = {0, 0};
    for (int fn = 0; fn < 2; ++fn) {
        long long b = 0;
        #pragma omp parallel for reduction(+:b) schedule(static, 1 << 16)
        for (long long i = 0; i < (long long)kDomain[fn]; ++i) {
            const uint32_t u = pattern(fn, (uint64_t)i);
            float x; memcpy(&x, &u, 4);
            const float got = fn == 0 ? nph_expf(x) : nph_logf(x);
            const float want = fn == 0 ? g_expf(x) : g_logf(x);
            if (!same(got, want)) {
                #pragma omp critical
                b += report(fn == 0 ? "expf" : "logf", fn, (uint64_t)i, got, want, b);
            }
        }
        bad[fn] = b;
    }
    printf("host: expf: %lld bad, logf: %lld bad\n", bad[0], bad[1]);
    return bad[0] == 0 && bad[1] == 0 ? 0 : 1;
}

__global__ void eval_kernel(int fn, uint64_t first, uint32_t n, float* out)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint64_t i = first + j;
        const uint32_t u = fn == 0 ? (i < 0x80000000ull ? 0x80000000u + (uint32_t)i : 0u) : (uint32_t)i;
        const float x = __uint_as_float(u);
        out[j] = fn == 0 ? nph_expf(x) : nph_logf(x);
    }
}

#define CK(call) do { cudaError_t e = (call); if (e != cudaSuccess) { printf("CUDA error %s at %s\n", cudaGetErrorString(e), #call); return 2; } } while (0)

static int run_device()
{
    const uint32_t chunk = 1u << 27;
    float* d = nullptr;
    CK(cudaMalloc(&d, sizeof(float) * chunk));
    std::vector<float> h(chunk);
    long long bad[2] = {0, 0};
    for (int fn = 0; fn < 2; ++fn) {
        long long b = 0;
        for (uint64_t first = 0; first < kDomain[fn]; first += chunk) {
            const uint32_t n = (uint32_t)std::min<uint64_t>(chunk, kDomain[fn] - first);
            eval_kernel<<<132 * 16, 256>>>(fn, first, n, d);
            CK(cudaGetLastError());
            CK(cudaMemcpy(h.data(), d, sizeof(float) * n, cudaMemcpyDeviceToHost));
            #pragma omp parallel for reduction(+:b) schedule(static, 1 << 16)
            for (long long j = 0; j < (long long)n; ++j) {
                const uint32_t u = pattern(fn, first + (uint64_t)j);
                float x; memcpy(&x, &u, 4);
                const float want = fn == 0 ? g_expf(x) : g_logf(x);
                if (!same(h[j], want)) {
                    #pragma omp critical
                    b += report(fn == 0 ? "expf" : "logf", fn, first + (uint64_t)j, h[j], want, b);
                }
            }
        }
        bad[fn] = b;
    }
    CK(cudaFree(d));
    printf("device: expf: %lld bad, logf: %lld bad\n", bad[0], bad[1]);
    return bad[0] == 0 && bad[1] == 0 ? 0 : 1;
}

int main(int argc, char** argv)
{
    if (argc > 1 && !strcmp(argv[1], "--host")) return run_host();
    if (argc > 1 && !strcmp(argv[1], "--device")) return run_device();
    printf("usage: %s --host | --device\n", argv[0]);
    return 2;
}
