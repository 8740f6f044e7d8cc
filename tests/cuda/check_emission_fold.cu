// check_emission_fold.cu — GPU self-check of add_neg_half_square (nanopolish_b200/csrc/exact_math.cuh, test infrastructure).
//   add_neg_half_square(cc, a) must equal the reference's literal cc + (-0.5f*a)*a (emissions.h:54) bit for bit, with a
//   formed as the forward kernel forms it: a = (x - mu) / sigma over the operand ranges of check_exact_math.cu
// Usage: check_emission_fold [n_million_pairs]   -> prints the mismatch count, exit code 0 iff it is 0.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../../nanopolish_b200/csrc/exact_math.cuh"

__device__ __forceinline__ uint32_t rng_next(uint64_t& s)
{
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    uint32_t x = (uint32_t)(s >> 33) ^ (uint32_t)(s >> 13);
    return x * 2654435761u;
}

__global__ void check_fold(unsigned long long* bad, unsigned long long per_thread, uint64_t seed)
{
    uint64_t s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    unsigned long long local = 0;
    for (unsigned long long i = 0; i < per_thread; ++i) {
        const uint32_t r0 = rng_next(s), r1 = rng_next(s), r2 = rng_next(s), sel = rng_next(s);
        float num, b;
        // numerator: event level minus model level (check_exact_math.cu's cases)
        switch (sel & 3) {
            case 0: num = ((int)(r0 >> 8) - (1 << 23)) * (200.0f / (1 << 23)); break;
            case 1: num = __int_as_float(((r0 & 0x80000000u)) | ((107u + (r0 >> 8) % 30u) << 23) | (r1 & 0x7fffffu)); break;
            case 2: num = __fsub_rn(60.0f + (r0 >> 8) * (70.0f / (1 << 24)), 60.0f + (r1 >> 8) * (70.0f / (1 << 24))); break;
            default: num = (r0 & 1) ? 0.0f : __int_as_float((r0 & 0x80000000u) | 0x3f800000u | (r1 & 0x7fffffu)); break;
        }
        const uint32_t m = r1 >> 9;
        switch ((sel >> 2) & 7) {
            case 0: b = 0.3f + (r1 >> 8) * (20.0f / (1 << 24)); break;
            case 1: b = __int_as_float(((119u + (r0 % 17u)) << 23) | m); break;
            case 2: b = __int_as_float(((119u + (r0 % 17u)) << 23) | 0x7fffffu); break;
            case 3: b = __int_as_float(((119u + (r0 % 17u)) << 23) | (0x7fffffu - (m & 7u))); break;
            case 4: b = __int_as_float(((119u + (r0 % 17u)) << 23) | (m & 7u)); break;
            case 5: b = 1.0f + (m & 0xffff) * 1.1920929e-7f; break;
            default: b = (float)(1.2 + (r1 >> 8) * (4.6 / (1 << 24))) * (float)(0.9 + (r0 >> 8) * (0.4 / (1 << 24))); break;
        }
        const float a = __fdiv_rn(num, b);
        // cc = log(1/sqrt(2 pi)) - log(sigma'): the data's range, any float in [-64, 64], exact zero, and small magnitudes
        float cc;
        switch ((sel >> 5) & 3) {
            case 0: cc = __fsub_rn(-0.9189385f, (float)((int)(r2 >> 8) - (1 << 23)) * (6.0f / (1 << 23))); break;
            case 1: cc = __int_as_float((r2 & 0x80000000u) | ((100u + (r2 >> 8) % 33u) << 23) | (r0 & 0x7fffffu)); break;
            case 2: cc = (r2 & 1) ? 0.0f : -0.0f; break;
            default: cc = __int_as_float((r2 & 0x80000000u) | ((1u + (r2 >> 8) % 60u) << 23) | (r1 & 0x7fffffu)); break;
        }
        const float got = add_neg_half_square(cc, a);
        const float want = __fadd_rn(cc, __fmul_rn(__fmul_rn(-0.5f, a), a));
        if (__float_as_int(got) != __float_as_int(want)) ++local;
    }
    if (local) atomicAdd(bad, local);
}

int main(int argc, char** argv)
{
    const unsigned long long millions = argc > 1 ? strtoull(argv[1], nullptr, 10) : 2000;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { fprintf(stderr, "no CUDA device\n"); return 2; }
    unsigned long long* d_bad; cudaMalloc(&d_bad, sizeof(unsigned long long)); cudaMemset(d_bad, 0, sizeof(unsigned long long));
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = sms * 4, threads = 256;
    const unsigned long long per_thread = millions * 1000000ull / ((unsigned long long)blocks * threads) + 1;
    check_fold<<<blocks, threads>>>(d_bad, per_thread, 4242);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(e)); return 3; }
    unsigned long long bad = 0;
    cudaMemcpy(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost);
    printf("emission fold: %llu pairs, %llu mismatches\n", per_thread * blocks * threads, bad);
    return bad ? 1 : 0;
}
