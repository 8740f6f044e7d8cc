// check_lsum_saturated.cu — GPU self-check of lsum_sat (nanopolish_b200/csrc/exact_math.cuh, test infrastructure).
//   lsum_sat(a, b) on the forward kernel's 16385-entry table must equal, bit for bit, a literal transcription of
//   p7_FLogsum (src/common/logsum.h:55-66) and the clamped 8-instruction lsum on the same table.
// Usage: check_lsum_saturated [n_million_pairs]   -> prints the mismatch counts, exit code 0 iff both are 0.
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

__device__ float ref_logsum(float a, float b, const float* tbl)
{
    const float mx = a > b ? a : b;
    const float mn = a < b ? a : b;
    if (mn == -INFINITY || (mx - mn) >= 15.7f) return mx;
    return mx + tbl[(int)((mx - mn) * 1000.f)];
}

__device__ bool same(float got, float want) { return __float_as_int(got) == __float_as_int(want) || (got == 0.0f && want == 0.0f); }

__global__ void check(unsigned long long* bad, unsigned long long per_thread, uint64_t seed, const float* tbl_g)
{
    extern __shared__ float s_tbl[];
    for (int i = threadIdx.x; i < NPH_LOGSUM_TBL_LEN; i += blockDim.x) s_tbl[i] = tbl_g[i];
    __syncthreads();
    const LogsumTable tb_sat = make_logsum_table(s_tbl, NPH_LOGSUM_SAT_ADDR_BIAS);
    const LogsumTable tb_cut = make_logsum_table(s_tbl, NPH_LOGSUM_ADDR_BIAS);
    uint64_t s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    unsigned long long bad_ref = 0, bad_cut = 0;
    for (unsigned long long i = 0; i < per_thread; ++i) {
        const uint32_t r0 = rng_next(s), r1 = rng_next(s), sel = rng_next(s);
        float a = -(r0 >> 8) * (2000.0f / (1 << 24));
        float b;
        switch (sel & 15) {
            case 0: b = -INFINITY; break;
            case 1: b = a; break;
            case 2: b = a - 15.7f; break;
            case 3: b = a - (15.69f + (r1 >> 8) * (0.02f / (1 << 24))); break;      // straddles the cut-off
            case 4: b = a + (r1 >> 8) * (0.002f / (1 << 24)); break;                  // tiny differences
            case 5: b = __int_as_float(__float_as_int(a) + (int)(r1 % 64u) - 32); break; // neighbouring floats
            case 6: b = a - (15.6f + (r1 >> 8) * (0.9f / (1 << 24))); break;         // cut-off to past the saturated index (16.384)
            case 7: a = -INFINITY; b = -INFINITY; break;                                // difference NaN
            case 8:                                                                     // exact differences: 15.7f, 16.384f and their neighbours
                a = (r0 & 1) ? 0.0f : -0.25f;                                           // a - d is exact: |a - d| < 16 for d near 15.7, < 32 near 16.4
                b = a - __int_as_float(__float_as_int((r0 & 2) ? 16.384f : 15.7f) + (int)(r1 % 64u) - 32);
                break;
            case 9:                                                                     // subnormal and tiny normal differences
                a = __int_as_float(0x80000000u | (r1 & 0x01ffffffu));                  // -0 .. -2^-124: subnormal or tiny normal
                b = __int_as_float(__float_as_int(a) + (int)(r0 % 4096u) - 2048);
                break;
            default: b = a + ((int)(r1 >> 8) - (1 << 23)) * (20.0f / (1 << 23)); break;
        }
        if ((sel & 0x700) == 0x700) a = -INFINITY;
        float x = a, y = b;
        if (sel & 8) { x = b; y = a; }
        if (x != x || y != y) continue;   // NaN is not a log-probability (cases 5 and 9 can step past a zero)
        const float got = lsum_sat(x, y, tb_sat);
        if (!same(got, ref_logsum(x, y, tbl_g))) ++bad_ref;
        if (!same(got, lsum(x, y, tb_cut))) ++bad_cut;
    }
    if (bad_ref) atomicAdd(bad, bad_ref);
    if (bad_cut) atomicAdd(bad + 1, bad_cut);
}

int main(int argc, char** argv)
{
    const unsigned long long millions = argc > 1 ? strtoull(argv[1], nullptr, 10) : 500;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { fprintf(stderr, "no CUDA device\n"); return 2; }
    unsigned long long* d_bad; cudaMalloc(&d_bad, 16); cudaMemset(d_bad, 0, 16);
    std::vector<float> tbl(NPH_LOGSUM_TBL_LEN, 0.0f);   // built as nph_api.cu builds it: entries from NPH_LOGSUM_CUT on stay 0.0f
    for (int i = 0; i < NPH_LOGSUM_CUT; ++i) tbl[i] = (float)log(1. + exp((double)-i / 1000.f));
    float* d_tbl; cudaMalloc(&d_tbl, tbl.size() * sizeof(float));
    cudaMemcpy(d_tbl, tbl.data(), tbl.size() * sizeof(float), cudaMemcpyHostToDevice);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int threads = 512;
    const unsigned long long per_thread = millions * 1000000ull / ((unsigned long long)sms * threads) + 1;
    const size_t smem = sizeof(float) * NPH_LOGSUM_TBL_LEN;
    cudaFuncSetAttribute(check, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    check<<<sms, threads, smem>>>(d_bad, per_thread, 4242, d_tbl);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(e)); return 3; }
    unsigned long long bad[2];
    cudaMemcpy(bad, d_bad, 16, cudaMemcpyDeviceToHost);
    printf("saturated logsum: %llu pairs, %llu mismatches against the reference, %llu mismatches against the clamped form\n",
           per_thread * sms * threads, bad[0], bad[1]);
    return (bad[0] | bad[1]) ? 1 : 0;
}
