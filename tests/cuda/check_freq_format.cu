// check_freq_format — the methylated_frequency column of the per-site frequency table: tsv_format.cuh's fixed_of<3> / put_fixed<3>
// against snprintf("%.3f") of the double m / n for every 0 <= m <= n, 1 <= n <= 5000 (exact ties such as 1/16 = 0.0625 round to
// even: "0.062"), and fixed2_of / put_fixed2 against snprintf("%.2lf") on the same doubles (its results must not move); the same
// inputs through the device copies of the functions.
// Build: nvcc -O2 -gencode arch=compute_90a,code=sm_90a -I nanopolish_b200/csrc tests/cuda/check_freq_format.cu -o build/checks/check_freq_format
// Usage: check_freq_format [--host-only]
#include "tsv_format.cuh"
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <cuda_runtime.h>

using namespace nph_tsv;

constexpr int kMaxN = 5000;
constexpr int kStride = 32;          // bytes per formatted value

// out[i]: "%.3f" then "%.2lf" of v[i], each NUL terminated in its own kStride bytes; ok[i] = 0 when a length disagrees
__global__ void fmt_kernel(const double* v, size_t n, char* out3, char* out2, unsigned char* ok)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const Fixed f3 = fixed_of<3>(v[i]);
        const Fixed2 f2 = fixed2_of(v[i]);
        char* e3 = put_fixed<3>(out3 + kStride * i, f3); *e3 = 0;
        char* e2 = put_fixed2(out2 + kStride * i, f2); *e2 = 0;
        ok[i] = f3.ok && f2.ok && (int)(e3 - (out3 + kStride * i)) == fixed_len<3>(f3) && (int)(e2 - (out2 + kStride * i)) == fixed2_len(f2);
    }
}

int main(int argc, char** argv)
{
    const bool host_only = argc > 1 && std::string(argv[1]) == "--host-only";
    std::vector<double> v;
    for (int n = 1; n <= kMaxN; ++n)
        for (int m = 0; m <= n; ++m) v.push_back((double)m / (double)n);
    size_t bad = 0;
    char ref[64], got[64];
    for (double d : v) {
        const Fixed f3 = fixed_of<3>(d);
        char* e = put_fixed<3>(got, f3); *e = 0;
        snprintf(ref, sizeof ref, "%.3f", d);
        if (!f3.ok || strcmp(ref, got) != 0 || (int)strlen(got) != fixed_len<3>(f3)) { ++bad; if (bad < 10) printf("host %%.3f mismatch %a: %s vs %s\n", d, got, ref); }
        const Fixed2 f2 = fixed2_of(d);
        e = put_fixed2(got, f2); *e = 0;
        snprintf(ref, sizeof ref, "%.2lf", d);
        if (!f2.ok || strcmp(ref, got) != 0 || (int)strlen(got) != fixed2_len(f2)) { ++bad; if (bad < 10) printf("host %%.2lf mismatch %a: %s vs %s\n", d, got, ref); }
    }
    printf("host: %zu values, %zu bad\n", v.size(), bad);
    if (!host_only) {
        const size_t n = v.size();
        double* dv; char* d3; char* d2; unsigned char* dok;
        if (cudaMalloc(&dv, 8 * n) != cudaSuccess) { printf("no device\n"); return 2; }
        cudaMalloc(&d3, kStride * n); cudaMalloc(&d2, kStride * n); cudaMalloc(&dok, n);
        cudaMemcpy(dv, v.data(), 8 * n, cudaMemcpyHostToDevice);
        fmt_kernel<<<1024, 256>>>(dv, n, d3, d2, dok);
        std::vector<char> o3(kStride * n), o2(kStride * n);
        std::vector<unsigned char> ok(n);
        if (cudaMemcpy(o3.data(), d3, kStride * n, cudaMemcpyDeviceToHost) != cudaSuccess) { printf("kernel failed\n"); return 2; }
        cudaMemcpy(o2.data(), d2, kStride * n, cudaMemcpyDeviceToHost);
        cudaMemcpy(ok.data(), dok, n, cudaMemcpyDeviceToHost);
        size_t dbad = 0;
        for (size_t i = 0; i < n; ++i) {
            snprintf(ref, sizeof ref, "%.3f", v[i]);
            snprintf(got, sizeof got, "%.2lf", v[i]);
            if (!ok[i] || strcmp(ref, &o3[kStride * i]) != 0 || strcmp(got, &o2[kStride * i]) != 0) {
                ++dbad;
                if (dbad < 10) printf("device mismatch %a: %s / %s vs %s / %s\n", v[i], &o3[kStride * i], &o2[kStride * i], ref, got);
            }
        }
        printf("device: %zu bad\n", dbad);
        bad += dbad;
        cudaFree(dv); cudaFree(d3); cudaFree(d2); cudaFree(dok);
    }
    printf(bad ? "FAILED\n" : "ok\n");
    return bad ? 1 : 0;
}
