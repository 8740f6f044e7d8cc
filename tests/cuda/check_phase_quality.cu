// check_phase_quality.cu — phase-reads' call and quality step (nph_phase_quality, csrc/exact_math.cuh) on the host and on the device.
//
// Inputs: ties, +-inf and NaN scores, score differences on a fine grid across the log-sum table (0 .. 20, both orders, two
// offsets), the floats on and next to the table's 15.7 cut-off, and for every q = 0 .. 31 the first score difference whose q
// reaches it with its two float neighbours.
//   --host    prints "ref_bits alt_bits call q_char" per input from the host (tests/test_phase_quality.py compares them with the
//             restatement in tests/phase_restatement.py)
//   --device  runs the same inputs on the device, prints the host lines and then "mismatches N" (host against device)
#include "exact_math.cuh"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

std::vector<float> g_tbl;

float bits_to_float(uint32_t b) { float f; std::memcpy(&f, &b, 4); return f; }
uint32_t float_bits(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }

// the host's q of (ref = 0, alt = -d) before truncation, for the bisection
double q_of(float d)
{
    const float ref = 0.f, alt = -d;
    const float mx = ref, dd = mx - alt;
    const double ls = !(dd < 15.7f) ? mx : mx + g_tbl[(int)(dd * 1000.f)];
    return -10.0 * ((double)alt - ls) / 2.302585092994045684;
}

std::vector<float2> inputs()
{
    std::vector<float2> v;
    const float inf = INFINITY, nan = NAN;
    const float specials[] = {0.f, -0.f, -1.5f, -1234.5678f, inf, -inf, nan, -3.0e38f, 3.0e38f};
    for (float a : specials) for (float b : specials) v.push_back(make_float2(a, b));
    for (float base : {0.f, -1234.5678f}) {
        for (int i = 0; i <= 40000; ++i) {
            const float d = (float)i * 0.0005f;
            v.push_back(make_float2(base, base - d));
            v.push_back(make_float2(base - d, base));
        }
    }
    const float cut = 15.7f;
    for (float d : {nextafterf(cut, 0.f), cut, nextafterf(cut, 100.f)}) {
        v.push_back(make_float2(0.f, -d));
        v.push_back(make_float2(-d, 0.f));
        v.push_back(make_float2(-100.f, -100.f - d));
    }
    for (int n = 0; n <= 31; ++n) {
        uint32_t lo = 0, hi = float_bits(40.f);              // q(0) = 3.01..., q(40) > 30: the first d with q >= n
        if (q_of(bits_to_float(lo)) >= n) hi = lo;
        while (hi - lo > 1) { const uint32_t m = lo + (hi - lo) / 2; if (q_of(bits_to_float(m)) >= n) hi = m; else lo = m; }
        for (uint32_t b : {hi - 1, hi, hi + 1}) {
            const float d = bits_to_float(b);
            v.push_back(make_float2(0.f, -d));
            v.push_back(make_float2(-d, 0.f));
        }
    }
    return v;
}

__global__ void device_quality(const float2* in, size_t n, const float* tbl, NphPhaseCall* out)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = nph_phase_quality(in[i].x, in[i].y, 'C', 'T', tbl);
}

} // namespace

int main(int argc, char** argv)
{
    const bool device = argc > 1 && std::strcmp(argv[1], "--device") == 0;
    g_tbl.assign(16000, 0.f);
    for (int i = 0; i < 16000; ++i) g_tbl[i] = (float)log(1. + exp((double)-i / 1000.f));       // p7_FLogsumInit
    const std::vector<float2> in = inputs();
    std::vector<NphPhaseCall> host(in.size());
    for (size_t i = 0; i < in.size(); ++i) {
        host[i] = nph_phase_quality(in[i].x, in[i].y, 'C', 'T', g_tbl.data());
        std::printf("%08x %08x %c %d\n", float_bits(in[i].x), float_bits(in[i].y), host[i].call, (int)host[i].q_char);
    }
    if (!device) return 0;
    float2* d_in; float* d_tbl; NphPhaseCall* d_out;
    if (cudaMalloc(&d_in, sizeof(float2) * in.size()) != cudaSuccess || cudaMalloc(&d_tbl, sizeof(float) * g_tbl.size()) != cudaSuccess ||
        cudaMalloc(&d_out, sizeof(NphPhaseCall) * in.size()) != cudaSuccess) { std::printf("cuda error\n"); return 2; }
    cudaMemcpy(d_in, in.data(), sizeof(float2) * in.size(), cudaMemcpyHostToDevice);
    cudaMemcpy(d_tbl, g_tbl.data(), sizeof(float) * g_tbl.size(), cudaMemcpyHostToDevice);
    device_quality<<<64, 256>>>(d_in, in.size(), d_tbl, d_out);
    std::vector<NphPhaseCall> dev(in.size());
    if (cudaMemcpy(dev.data(), d_out, sizeof(NphPhaseCall) * in.size(), cudaMemcpyDeviceToHost) != cudaSuccess) { std::printf("cuda error\n"); return 2; }
    size_t bad = 0;
    for (size_t i = 0; i < in.size(); ++i) bad += dev[i].call != host[i].call || dev[i].q_char != host[i].q_char;
    std::printf("mismatches %zu\n", bad);
    cudaFree(d_in); cudaFree(d_tbl); cudaFree(d_out);
    return bad ? 1 : 0;
}
