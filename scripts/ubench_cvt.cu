// throughput of the conversion / FP64 instructions the event detector leans on (warp instructions per clock per SM sub-partition)
#include <cstdio>
#include <cuda_runtime.h>
#define N_ITER 4096
template <int OP> __global__ void k(float* out, float seed, long long* clk)
{
    float f0 = seed + threadIdx.x, f1 = f0 + 1.f, f2 = f0 + 2.f, f3 = f0 + 3.f;
    double d0 = f0, d1 = f1, d2 = f2, d3 = f3;
    unsigned u0 = __float_as_uint(f0), u1 = u0 + 1, u2 = u0 + 2, u3 = u0 + 3;
    const long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < N_ITER; ++i) {
        if (OP == 0) {          // F2F.F64.F32 + F2F.F32.F64 round trip (2 conversions per chain step)
            d0 = (double)f0; d1 = (double)f1; d2 = (double)f2; d3 = (double)f3;
            asm volatile("" : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3));
            f0 = (float)d0; f1 = (float)d1; f2 = (float)d2; f3 = (float)d3;
            asm volatile("" : "+f"(f0), "+f"(f1), "+f"(f2), "+f"(f3));
        } else if (OP == 1) {   // DADD
            d0 = __dadd_rn(d0, d1); d1 = __dadd_rn(d1, d2); d2 = __dadd_rn(d2, d3); d3 = __dadd_rn(d3, d0);
        } else if (OP == 2) {   // DFMA
            d0 = __fma_rn(d0, d1, d2); d1 = __fma_rn(d1, d2, d3); d2 = __fma_rn(d2, d3, d0); d3 = __fma_rn(d3, d0, d1);
        } else if (OP == 3) {   // integer float->double widening (normal numbers): 4 ALU ops per value
            unsigned h0 = (u0 & 0x80000000u) | ((u0 >> 3) & 0x0fffffffu), l0 = u0 << 29; h0 += 0x38000000u;
            unsigned h1 = (u1 & 0x80000000u) | ((u1 >> 3) & 0x0fffffffu), l1 = u1 << 29; h1 += 0x38000000u;
            d0 = __dadd_rn(d0, __hiloint2double((int)h0, (int)l0)); d1 = __dadd_rn(d1, __hiloint2double((int)h1, (int)l1));
            u0 += 7; u1 += 11;
        } else if (OP == 4) {   // MUFU.RSQ64H
            d0 = rsqrt(d0) + 1.0; d1 = rsqrt(d1) + 1.0;
        }
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = f0 + f1 + f2 + f3 + (float)(d0 + d1 + d2 + d3) + (float)(u0 + u1 + u2 + u3);
    if (threadIdx.x == 0 && blockIdx.x == 0) *clk = t1 - t0;
}
template <int OP> void run(const char* name, int per_iter)
{
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float* out; long long* clk; cudaMalloc(&out, sms * 1024 * 4); cudaMalloc(&clk, 8);
    for (int warps = 4; warps <= 32; warps *= 2) {          // warps per SM (1..8 per sub-partition)
        k<OP><<<sms, warps * 32>>>(out, 1.5f, clk); cudaDeviceSynchronize();
        k<OP><<<sms, warps * 32>>>(out, 1.5f, clk); cudaDeviceSynchronize();
        long long c; cudaMemcpy(&c, clk, 8, cudaMemcpyDeviceToHost);
        printf("%-28s warps/SMSP %d : %.3f warp-instr/clk/SMSP\n", name, warps / 4, (double)per_iter * N_ITER * (warps / 4) / (double)c);
    }
}
int main()
{
    run<0>("F2F f32<->f64 (8/iter)", 8);
    run<1>("DADD (4/iter)", 4);
    run<2>("DFMA (4/iter)", 4);
    run<3>("int widen + DADD (2 values)", 2);
    run<4>("rsqrt(double)+DADD (2)", 2);
    return 0;
}
