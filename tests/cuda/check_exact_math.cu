// check_exact_math.cu — GPU self-check of nanopolish_b200/csrc/exact_math.cuh (test infrastructure).
//   * div_by_cached_rcp(a, b, RN(1/b)) must equal __fdiv_rn(a, b) bit for bit
//   * lsum(a, b) must equal a literal transcription of p7_FLogsum (src/common/logsum.h:55-66)
// Usage: check_exact_math [n_million_pairs]   -> prints mismatch counts, exit code 0 iff both are 0.
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "../../nanopolish_b200/csrc/exact_math.cuh"

__device__ __forceinline__ uint32_t rng_next(uint64_t& s)
{
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    uint32_t x = (uint32_t)(s >> 33) ^ (uint32_t)(s >> 13);
    return x * 2654435761u;
}

__global__ void check_div(unsigned long long* bad, unsigned long long per_thread, uint64_t seed)
{
    uint64_t s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    unsigned long long local = 0;
    for (unsigned long long i = 0; i < per_thread; ++i) {
        const uint32_t r0 = rng_next(s), r1 = rng_next(s), sel = rng_next(s);
        float a, b;
        // numerator: event level minus model level
        switch (sel & 3) {
            case 0: a = ((int)(r0 >> 8) - (1 << 23)) * (200.0f / (1 << 23)); break;               // uniform [-200, 200)
            case 1: a = __int_as_float(((r0 & 0x80000000u)) | ((107u + (r0 >> 8) % 30u) << 23) | (r1 & 0x7fffffu)); break; // 2^-20..2^9, any mantissa
            case 2: a = __fsub_rn(60.0f + (r0 >> 8) * (70.0f / (1 << 24)), 60.0f + (r1 >> 8) * (70.0f / (1 << 24))); break; // difference of two levels
            default: a = (r0 & 1) ? 0.0f : __int_as_float((r0 & 0x80000000u) | 0x3f800000u | (r1 & 0x7fffffu)); break;
        }
        // divisor: scaled model stdv
        const uint32_t m = r1 >> 9;
        switch ((sel >> 2) & 7) {
            case 0: b = 0.3f + (r1 >> 8) * (20.0f / (1 << 24)); break;
            case 1: b = __int_as_float(((119u + (r0 % 17u)) << 23) | m); break;                  // 2^-8..2^8 any mantissa
            case 2: b = __int_as_float(((119u + (r0 % 17u)) << 23) | 0x7fffffu); break;          // all-ones mantissa
            case 3: b = __int_as_float(((119u + (r0 % 17u)) << 23) | (0x7fffffu - (m & 7u))); break; // near all-ones
            case 4: b = __int_as_float(((119u + (r0 % 17u)) << 23) | (m & 7u)); break;            // near a power of two
            case 5: b = 1.0f + (m & 0xffff) * 1.1920929e-7f; break;
            default: b = (float)(1.2 + (r1 >> 8) * (4.6 / (1 << 24))) * (float)(0.9 + (r0 >> 8) * (0.4 / (1 << 24))); break; // stdv*var like the data
        }
        const float y = __frcp_rn(b);
        const float q = div_by_cached_rcp(a, b, y);
        const float w = __fdiv_rn(a, b);
        if (__float_as_int(q) != __float_as_int(w)) ++local;
    }
    if (local) atomicAdd(bad, local);
}

__device__ float ref_logsum(float a, float b, const float* tbl)
{
    const float mx = a > b ? a : b;
    const float mn = a < b ? a : b;
    if (mn == -INFINITY || (mx - mn) >= 15.7f) return mx;
    return mx + tbl[(int)((mx - mn) * 1000.f)];
}

__global__ void check_lsum(unsigned long long* bad, unsigned long long per_thread, uint64_t seed, const float* tbl_g, uint32_t bias)
{
    extern __shared__ float s_tbl[];
    for (int i = threadIdx.x; i <= NPH_LOGSUM_CUT; i += blockDim.x) s_tbl[i] = tbl_g[i];
    __syncthreads();
    const LogsumTable tb = make_logsum_table(s_tbl, bias);
    uint64_t s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    unsigned long long local = 0;
    for (unsigned long long i = 0; i < per_thread; ++i) {
        const uint32_t r0 = rng_next(s), r1 = rng_next(s), sel = rng_next(s);
        float a = -(r0 >> 8) * (2000.0f / (1 << 24));
        float b;
        switch (sel & 7) {
            case 0: b = -INFINITY; break;
            case 1: b = a; break;
            case 2: b = a - 15.7f; break;
            case 3: b = a - (15.69f + (r1 >> 8) * (0.02f / (1 << 24))); break;      // straddles the cut-off
            case 4: b = a + (r1 >> 8) * (0.002f / (1 << 24)); break;                  // tiny differences
            case 5: b = __int_as_float(__float_as_int(a) + (int)(r1 % 64u) - 32); break; // neighbouring floats
            default: b = a + ((int)(r1 >> 8) - (1 << 23)) * (20.0f / (1 << 23)); break;
        }
        if ((sel & 0x700) == 0x700) a = -INFINITY;
        float x = a, y = b;
        if (sel & 8) { x = b; y = a; }
        if (x != x || y != y) continue;   // NaN is not a log-probability (case 5 can step off -0.0)
        const float got = lsum(x, y, tb);
        const float want = ref_logsum(x, y, tbl_g);
        if (__float_as_int(got) != __float_as_int(want) && !(got == 0.0f && want == 0.0f)) ++local;
    }
    if (local) atomicAdd(bad, local);
}

int main(int argc, char** argv)
{
    const unsigned long long millions = argc > 1 ? strtoull(argv[1], nullptr, 10) : 2000;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { fprintf(stderr, "no CUDA device\n"); return 2; }
    unsigned long long* d_bad; cudaMalloc(&d_bad, 128); cudaMemset(d_bad, 0, 128);
    std::vector<float> tbl(NPH_LOGSUM_CUT + 1);
    for (int i = 0; i < NPH_LOGSUM_CUT; ++i) tbl[i] = (float)log(1. + exp((double)-i / 1000.f));
    tbl[NPH_LOGSUM_CUT] = 0.0f;
    float* d_tbl; cudaMalloc(&d_tbl, tbl.size() * sizeof(float));
    cudaMemcpy(d_tbl, tbl.data(), tbl.size() * sizeof(float), cudaMemcpyHostToDevice);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = sms * 4, threads = 256;
    const unsigned long long per_thread = millions * 1000000ull / ((unsigned long long)blocks * threads) + 1;
    check_div<<<blocks, threads>>>(d_bad, per_thread, 12345);
    const size_t smem = sizeof(float) * (NPH_LOGSUM_CUT + 1);
    cudaFuncSetAttribute(check_lsum, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    check_lsum<<<sms, 512, smem>>>(d_bad + 1, per_thread / 4 + 1, 777, d_tbl, NPH_LOGSUM_ADDR_BIAS);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(e)); return 3; }
    unsigned long long bad[2];
    cudaMemcpy(bad, d_bad, 16, cudaMemcpyDeviceToHost);
    printf("division: %llu pairs, %llu mismatches\nlogsum: %llu pairs, %llu mismatches\n",
           per_thread * blocks * threads, bad[0], (per_thread / 4 + 1) * sms * 512ull, bad[1]);
    return (bad[0] | bad[1]) ? 1 : 0;
}
