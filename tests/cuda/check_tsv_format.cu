// check_tsv_format — tsv_format.cuh against the C library: printf("%.2lf") on random and adversarial doubles (values the
// call-methylation rows hold: float scores widened and their differences; exact halves at the second decimal; tiny, huge,
// negative zero), and %d on the integer range; the same inputs through the device copies of the functions.
// Build: nvcc -O2 -gencode arch=compute_90a,code=sm_90a -I nanopolish_b200/csrc tests/cuda/check_tsv_format.cu -o build/checks/check_tsv_format
// Usage: check_tsv_format [--host-only]
#include "tsv_format.cuh"
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <string>
#include <vector>
#include <random>
#include <cuda_runtime.h>

using namespace nph_tsv;

__global__ void fmt_kernel(const double* v, size_t n, char* out /* 40 bytes per value */, unsigned char* ok)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const Fixed2 f = fixed2_of(v[i]);
        ok[i] = f.ok ? 1 : 0;
        char* o = out + 40 * i;
        char* e = f.ok ? put_fixed2(o, f) : o;
        *e = 0;
        if (f.ok && (int)(e - o) != fixed2_len(f)) ok[i] = 2;
    }
}

int main(int argc, char** argv)
{
    const bool host_only = argc > 1 && std::string(argv[1]) == "--host-only";
    std::vector<double> v;
    std::mt19937_64 rng(12345);
    std::uniform_real_distribution<double> u(-400.0, 50.0);
    for (int i = 0; i < 2000000; ++i) {
        const float a = (float)u(rng), b = (float)u(rng);
        v.push_back((double)a); v.push_back((double)a - (double)b);
    }
    for (int i = -200000; i <= 200000; ++i) { v.push_back(i / 200.0); v.push_back(i * 0.005); v.push_back(std::nextafter(i * 0.005, 1e9)); v.push_back(std::nextafter(i * 0.005, -1e9)); }
    for (int e = -1080; e <= 70; ++e) { v.push_back(std::ldexp(1.0, e)); v.push_back(-std::ldexp(1.7, e)); v.push_back(std::ldexp(1.0 - 1e-16, e)); }
    for (int i = 0; i < 1000000; ++i) { uint64_t b = rng(); double d; memcpy(&d, &b, 8); v.push_back(d); }
    v.push_back(0.0); v.push_back(-0.0); v.push_back(INFINITY); v.push_back(-INFINITY); v.push_back(NAN); v.push_back(4503599627370496.0); v.push_back(4503599627370495.5);
    size_t bad = 0, refused = 0;
    char ref[512], got[64];
    for (double d : v) {
        const Fixed2 f = fixed2_of(d);
        if (!f.ok) { ++refused; if (std::isfinite(d) && std::fabs(d) < 4503599627370496.0) { ++bad; if (bad < 10) printf("refused %a\n", d); } continue; }
        snprintf(ref, sizeof ref, "%.2lf", d);
        char* e = put_fixed2(got, f); *e = 0;
        if (strcmp(ref, got) != 0 || (int)strlen(got) != fixed2_len(f)) { ++bad; if (bad < 10) printf("host mismatch %a: %s vs %s\n", d, got, ref); }
    }
    for (long long i = -2147483647LL - 1; i <= 2147483647LL; i += 104729) {
        snprintf(ref, sizeof ref, "%d", (int)i);
        char* e = put_int(got, (int)i); *e = 0;
        if (strcmp(ref, got) != 0 || (int)strlen(got) != int_len((int)i)) { ++bad; if (bad < 10) printf("int mismatch %lld: %s\n", i, got); }
    }
    printf("host: %zu values, %zu refused, %zu bad\n", v.size(), refused, bad);
    if (!host_only) {
        double* dv; char* dout; unsigned char* dok;
        const size_t n = v.size();
        if (cudaMalloc(&dv, 8 * n) != cudaSuccess) { printf("no device\n"); return 2; }
        cudaMalloc(&dout, 40 * n); cudaMalloc(&dok, n);
        cudaMemcpy(dv, v.data(), 8 * n, cudaMemcpyHostToDevice);
        fmt_kernel<<<1024, 256>>>(dv, n, dout, dok);
        std::vector<char> out(40 * n); std::vector<unsigned char> ok(n);
        if (cudaMemcpy(out.data(), dout, 40 * n, cudaMemcpyDeviceToHost) != cudaSuccess) { printf("kernel failed\n"); return 2; }
        cudaMemcpy(ok.data(), dok, n, cudaMemcpyDeviceToHost);
        size_t dbad = 0;
        for (size_t i = 0; i < n; ++i) {
            const Fixed2 f = fixed2_of(v[i]);
            if (!f.ok) { if (ok[i] != 0) ++dbad; continue; }
            snprintf(ref, sizeof ref, "%.2lf", v[i]);
            if (ok[i] != 1 || strcmp(ref, &out[40 * i]) != 0) { ++dbad; if (dbad < 10) printf("device mismatch %a: %s vs %s\n", v[i], &out[40 * i], ref); }
        }
        printf("device: %zu bad\n", dbad);
        bad += dbad;
    }
    printf(bad ? "FAILED\n" : "ok\n");
    return bad ? 1 : 0;
}
