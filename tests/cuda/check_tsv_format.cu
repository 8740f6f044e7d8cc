// check_tsv_format — tsv_format.cuh against the C library, on the host and through the device copies of the same functions:
//   doubles at "%.0lf" .. "%.3lf": the values call-methylation rows hold (float scores widened and their differences), exact
//     halves at the second decimal, every binade, random bit patterns, refusals at 2^52, non-finite values, +-0;
//   every m / n with n <= 5000 at "%.3f" and "%.2lf" (the frequency table's column and the row's numbers);
//   floats at "%.0lf" .. "%.5lf": raw bit patterns, scaled 16-bit integers, decimal ties and their neighbours, refusals at 2^39;
//   put_int / put_i64 against "%d" / "%lld" (host);
//   put_meth_row / meth_row_len against the reference's "%s\t%c\t%d\t%d\t%s\t%.2lf\t%.2lf\t%.2lf\t%d\t%d\t%s\n";
//   row_numbers' sequence column, including seq_ok = false for a group that starts k - 2 bases into its record.
// Build: nvcc -O2 -gencode arch=compute_90a,code=sm_90a -I nanopolish_b200/csrc tests/cuda/check_tsv_format.cu -o build/checks/check_tsv_format
// Usage: check_tsv_format [--host-only]
#include "tsv_format.cuh"
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <climits>
#include <string>
#include <vector>
#include <random>
#include <cuda_runtime.h>

using namespace nph_tsv;

constexpr int kStride = 32;          // bytes per formatted number
constexpr int kRowStride = 1024;     // bytes per formatted row

static bool g_device = true;
static size_t g_values = 0, g_refused = 0, g_bad = 0, g_dbad = 0;

static void section_end(size_t dbad)
{
    if (g_device) printf(", device %zu bad", dbad);
    printf("\n");
}

#define BAD(counter, ...) do { if (++(counter) < 10) printf(__VA_ARGS__); } while (0)

template <typename T>
static std::vector<T> from_device(const T* d, size_t n)
{
    std::vector<T> h(n);
    if (cudaMemcpy(h.data(), d, sizeof(T) * n, cudaMemcpyDeviceToHost) != cudaSuccess) { printf("device copy failed\n"); exit(2); }
    return h;
}

template <typename T>
static T* to_device(const std::vector<T>& h)
{
    T* d = nullptr;
    if (cudaMalloc(&d, sizeof(T) * (h.size() ? h.size() : 1)) != cudaSuccess) { printf("no device\n"); exit(2); }
    cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice);
    return d;
}

// ---- numbers ------------------------------------------------------------------------------------------------------

// out[i]: the text of v[i] in its own kStride bytes, NUL terminated; ok[i]: 0 refused, 1 formatted, 2 length disagrees
template <int N, typename T>
__global__ void fixed_kernel(const T* v, size_t n, char* out, unsigned char* ok)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const Fixed f = fixed_of<N>(v[i]);
        char* o = out + kStride * i;
        char* e = f.ok ? put_fixed<N>(o, f) : o;
        *e = 0;
        ok[i] = !f.ok ? 0 : (int)(e - o) == fixed_len<N>(f) ? 1 : 2;
    }
}

// fixed_of<N> / put_fixed<N> / fixed_len<N> == snprintf("%.Nlf") of every value below `limit`, refusal of everything else
template <int N, typename T>
static void check_fixed(const char* what, const std::vector<T>& v, double limit)
{
    const char fmt[] = {'%', '.', (char)('0' + N), 'l', 'f', 0};
    char ref[512], got[64];
    size_t refused = 0, bad = 0;
    for (const T x : v) {
        const Fixed f = fixed_of<N>(x);
        if (!f.ok) {
            ++refused;
            if (std::isfinite((double)x) && std::fabs((double)x) < limit) BAD(bad, "%s: refused %a\n", what, (double)x);
            continue;
        }
        snprintf(ref, sizeof ref, fmt, (double)x);
        char* e = put_fixed<N>(got, f); *e = 0;
        if (strcmp(ref, got) != 0 || (int)strlen(got) != fixed_len<N>(f)) BAD(bad, "%s: host %a: %s vs %s\n", what, (double)x, got, ref);
    }
    size_t dbad = 0;
    if (g_device) {
        const size_t n = v.size();
        T* dv = to_device(v);
        char* dout; unsigned char* dok;
        cudaMalloc(&dout, kStride * n); cudaMalloc(&dok, n);
        fixed_kernel<N, T><<<1024, 256>>>(dv, n, dout, dok);
        const std::vector<char> out = from_device(dout, kStride * n);
        const std::vector<unsigned char> ok = from_device(dok, n);
        for (size_t i = 0; i < n; ++i) {
            if (!fixed_of<N>(v[i]).ok) { if (ok[i] != 0) BAD(dbad, "%s: device formatted refused %a\n", what, (double)v[i]); continue; }
            snprintf(ref, sizeof ref, fmt, (double)v[i]);
            if (ok[i] != 1 || strcmp(ref, &out[kStride * i]) != 0) BAD(dbad, "%s: device %a: %s vs %s\n", what, (double)v[i], &out[kStride * i], ref);
        }
        cudaFree(dv); cudaFree(dout); cudaFree(dok);
    }
    printf("  %-28s %8zu values, %7zu refused, host %zu bad", what, v.size(), refused, bad);
    section_end(dbad);
    g_values += v.size(); g_refused += refused; g_bad += bad; g_dbad += dbad;
}

static void check_ints()
{
    char ref[64], got[64];
    size_t bad = 0, n = 0;
    for (long long i = -2147483647LL - 1; i <= 2147483647LL; i += 104729, ++n) {
        snprintf(ref, sizeof ref, "%d", (int)i);
        char* e = put_int(got, (int)i); *e = 0;
        if (strcmp(ref, got) != 0 || (int)strlen(got) != int_len((int)i)) BAD(bad, "int %lld: %s\n", i, got);
    }
    std::mt19937_64 rng(7);
    std::vector<long long> w = {LLONG_MIN, LLONG_MIN + 1, LLONG_MAX, -1, 0, 1, 9, 10, -10};
    for (int i = 0; i < 200000; ++i) w.push_back((long long)(rng() >> (rng() % 64)) * ((i & 1) ? -1 : 1));
    for (const long long x : w) {
        snprintf(ref, sizeof ref, "%lld", x);
        char* e = put_i64(got, (int64_t)x); *e = 0;
        if (strcmp(ref, got) != 0) BAD(bad, "i64 %lld: %s\n", x, got);
    }
    n += w.size();
    printf("  %-28s %8zu values, host %zu bad\n", "%d, %lld", n, bad);
    g_values += n; g_bad += bad;
}

// ---- rows ---------------------------------------------------------------------------------------------------------

struct RowCase {
    uint32_t contig_off, contig_len, name_off, name_len, seq_off, seq_len;
    char strand;
    int start, end, strands, n_motif;
    double sum_m, sum_u;
};

__host__ __device__ MethRow row_of(const RowCase& c, const char* pool)
{
    return MethRow{pool + c.contig_off, c.contig_len, c.strand, c.start, c.end, pool + c.name_off, c.name_len,
                   fixed_of<2>(c.sum_m - c.sum_u), fixed_of<2>(c.sum_m), fixed_of<2>(c.sum_u), c.strands, c.n_motif, pool + c.seq_off, c.seq_len};
}

// out[i]: the row of case i in its own kRowStride bytes, NUL terminated; len[i]: meth_row_len, or -1 where put_meth_row disagrees
__global__ void row_kernel(const RowCase* cases, size_t n, const char* pool, char* out, int* len)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const MethRow r = row_of(cases[i], pool);
        char* o = out + kRowStride * i;
        char* e = put_meth_row(o, r);
        *e = 0;
        len[i] = (int)(e - o) == (int)meth_row_len(r) ? (int)meth_row_len(r) : -1;
    }
}

static void check_rows()
{
    std::mt19937_64 rng(99);
    std::string pool;
    auto add = [&](const std::string& s) { const uint32_t off = (uint32_t)pool.size(); pool += s; return off; };
    const std::vector<std::string> contigs = {"chr20", "GL000220.1", "c", std::string(180, 'X')};
    const std::vector<std::string> names = {"", "r", "5a8a4b1f-e0f5-4a6e-9b5e-0c3c1d2f0e11", std::string(300, 'n')};
    std::uniform_real_distribution<float> score(-400.0f, 50.0f);
    std::vector<RowCase> cases;
    std::vector<std::string> want;
    for (int i = 0; i < 40000; ++i) {
        RowCase c;
        const std::string& contig = contigs[rng() % contigs.size()];
        const std::string& name = names[rng() % names.size()];
        std::string seq(rng() % 80, 'A');
        for (char& b : seq) b = "ACGTN"[rng() % 5];
        c.contig_off = add(contig); c.contig_len = (uint32_t)contig.size();
        c.name_off = add(name); c.name_len = (uint32_t)name.size();
        c.seq_off = add(seq); c.seq_len = (uint32_t)seq.size();
        c.strand = (rng() & 1) ? '-' : '+';
        const int span = (int)(rng() % 300);
        switch (i % 4) {
        case 0: c.start = (int)(rng() % 250000000); break;
        case 1: c.start = -(int)(rng() % 100000); break;                 // negative positions
        case 2: c.start = INT_MIN + (int)(rng() % 1000); break;
        default: c.start = INT_MAX - 300 - (int)(rng() % 1000); break;
        }
        c.end = c.start + span;
        c.strands = 1 + (int)(rng() & 1);
        c.n_motif = (i % 97 == 0) ? INT_MAX - (int)(rng() % 10) : 1 + (int)(rng() % 12);
        // the writer's sums: one float and the other strand's 0.0, or two floats; -0.0f on both strands prints "-0.00"
        const float m0 = i % 101 == 0 ? -0.0f : score(rng), u0 = i % 103 == 0 ? -0.0f : score(rng);
        const float m1 = c.strands == 2 ? (i % 101 == 0 ? -0.0f : score(rng)) : 0.0f, u1 = c.strands == 2 ? (i % 103 == 0 ? -0.0f : score(rng)) : 0.0f;
        c.sum_m = (double)m0 + (double)m1; c.sum_u = (double)u0 + (double)u1;
        cases.push_back(c);
        char ref[2048];
        snprintf(ref, sizeof ref, "%s\t%c\t%d\t%d\t%s\t%.2lf\t%.2lf\t%.2lf\t%d\t%d\t%s\n", contig.c_str(), c.strand, c.start, c.end, name.c_str(),
                 c.sum_m - c.sum_u, c.sum_m, c.sum_u, c.strands, c.n_motif, seq.c_str());
        want.push_back(ref);
    }
    size_t bad = 0, dbad = 0;
    std::vector<char> got(kRowStride);
    for (size_t i = 0; i < cases.size(); ++i) {
        const MethRow r = row_of(cases[i], pool.data());
        char* e = put_meth_row(got.data(), r);
        const std::string s(got.data(), e);
        if (s != want[i] || meth_row_len(r) != s.size()) BAD(bad, "row %zu: host %s vs %s", i, s.c_str(), want[i].c_str());
    }
    if (g_device) {
        const size_t n = cases.size();
        RowCase* dc = to_device(cases);
        char* dpool = to_device(std::vector<char>(pool.begin(), pool.end()));
        char* dout; int* dlen;
        cudaMalloc(&dout, (size_t)kRowStride * n); cudaMalloc(&dlen, sizeof(int) * n);
        row_kernel<<<256, 128>>>(dc, n, dpool, dout, dlen);
        const std::vector<char> out = from_device(dout, (size_t)kRowStride * n);
        const std::vector<int> len = from_device(dlen, n);
        for (size_t i = 0; i < n; ++i) {
            const char* s = &out[(size_t)kRowStride * i];
            if (len[i] != (int)want[i].size() || want[i] != s) BAD(dbad, "row %zu: device %s vs %s", i, s, want[i].c_str());
        }
        cudaFree(dc); cudaFree(dpool); cudaFree(dout); cudaFree(dlen);
    }
    printf("  %-28s %8zu values, host %zu bad", "methylation_calls.tsv rows", cases.size(), bad);
    section_end(dbad);
    g_values += cases.size(); g_bad += bad; g_dbad += dbad;
}

// ---- row_numbers --------------------------------------------------------------------------------------------------

struct SeqCase { nph_meth_site ms; nph_meth_record R; uint32_t k; bool ok; uint32_t b, len; bool m_neg; };

__global__ void seq_kernel(const SeqCase* c, size_t n, RowNums* out)
{
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = row_numbers(c[i].ms, c[i].R, c[i].k);
}

static void check_row_numbers()
{
    std::vector<SeqCase> cases;
    auto add = [&](int start_in_record, int span, uint32_t ref_len, uint32_t k, float ll_m, bool ok, uint32_t b, uint32_t len, bool m_neg) {
        SeqCase c{};
        c.R.ref_start_pos = 1000; c.R.ref_len = ref_len;
        c.ms.start_position = 1000 + start_in_record; c.ms.end_position = c.ms.start_position + span;
        c.ms.ll_methylated = ll_m; c.ms.ll_unmethylated = -3.25f; c.ms.n_motif = 1;
        c.k = k; c.ok = ok; c.b = b; c.len = len; c.m_neg = m_neg;
        cases.push_back(c);
    };
    for (uint32_t k = 5; k <= 6; ++k) {
        add((int)k - 2, 0, 500, k, -1.5f, false, 0, 0, true);                 // starts k - 2 bases in: the column would begin at -1
        add((int)k - 1, 0, 500, k, -1.5f, true, 0, 2 * k - 1, true);          // k - 1 bases in: begins at the record's first base
        add(100, 4, 500, k, 2.0f, true, 100 - k + 1, 4 + 2 * k - 1, false);
        add(495, 3, 500, k, 2.0f, true, 495 - k + 1, 500 - (495 - k + 1), false);   // cut at the end of the record
        add(200, 0, 500, k, -0.0f, true, 200 - k + 1, 2 * k - 1, false);      // -0.0f + the other strand's 0.0 prints "0.00"
    }
    size_t bad = 0, dbad = 0;
    auto same = [](const SeqCase& c, const RowNums& r) {
        return r.seq_ok == c.ok && (!c.ok || (r.seq_b == c.b && r.seq_len == c.len)) && r.m.ok && r.m.neg == c.m_neg && r.u.ok && r.u.neg;
    };
    for (size_t i = 0; i < cases.size(); ++i)
        if (!same(cases[i], row_numbers(cases[i].ms, cases[i].R, cases[i].k))) BAD(bad, "row_numbers case %zu: host\n", i);
    if (g_device) {
        SeqCase* dc = to_device(cases);
        RowNums* dout; cudaMalloc(&dout, sizeof(RowNums) * cases.size());
        seq_kernel<<<1, 64>>>(dc, cases.size(), dout);
        const std::vector<RowNums> got = from_device(dout, cases.size());
        for (size_t i = 0; i < cases.size(); ++i) if (!same(cases[i], got[i])) BAD(dbad, "row_numbers case %zu: device\n", i);
        cudaFree(dc); cudaFree(dout);
    }
    printf("  %-28s %8zu values, host %zu bad", "row_numbers sequence column", cases.size(), bad);
    section_end(dbad);
    g_values += cases.size(); g_bad += bad; g_dbad += dbad;
}

int main(int argc, char** argv)
{
    g_device = !(argc > 1 && std::string(argv[1]) == "--host-only");
    std::mt19937_64 rng(12345);

    std::vector<double> v;
    std::uniform_real_distribution<double> u(-400.0, 50.0);
    for (int i = 0; i < 2000000; ++i) {
        const float a = (float)u(rng), b = (float)u(rng);
        v.push_back((double)a); v.push_back((double)a - (double)b);
    }
    for (int i = -200000; i <= 200000; ++i) { v.push_back(i / 200.0); v.push_back(i * 0.005); v.push_back(std::nextafter(i * 0.005, 1e9)); v.push_back(std::nextafter(i * 0.005, -1e9)); }
    for (int e = -1080; e <= 70; ++e) { v.push_back(std::ldexp(1.0, e)); v.push_back(-std::ldexp(1.7, e)); v.push_back(std::ldexp(1.0 - 1e-16, e)); }
    for (int i = 0; i < 1000000; ++i) { uint64_t b = rng(); double d; memcpy(&d, &b, 8); v.push_back(d); }
    v.push_back(0.0); v.push_back(-0.0); v.push_back(INFINITY); v.push_back(-INFINITY); v.push_back(NAN); v.push_back(4503599627370496.0); v.push_back(4503599627370495.5);
    const double kDoubleLimit = 4503599627370496.0;      // 2^52
    check_fixed<2>("double %.2lf", v, kDoubleLimit);
    std::vector<double> few(v.begin(), v.begin() + 400000);   // the other precisions on scores and differences ...
    few.insert(few.end(), v.end() - 1000000 - 7, v.end());   // ... random bit patterns, specials
    check_fixed<0>("double %.0lf", few, kDoubleLimit);
    check_fixed<1>("double %.1lf", few, kDoubleLimit);
    check_fixed<3>("double %.3lf", few, kDoubleLimit);

    std::vector<double> ratios;
    for (int n = 1; n <= 5000; ++n)
        for (int m = 0; m <= n; ++m) ratios.push_back((double)m / (double)n);
    check_fixed<3>("m / n %.3f", ratios, kDoubleLimit);
    check_fixed<2>("m / n %.2lf", ratios, kDoubleLimit);

    // floats: raw bit patterns; scaled 16-bit integers (often exact ties at a printed digit) and their upper neighbours;
    // decimal ties (q + 0.5) / 1000 rounded to float and their neighbours; specials
    std::vector<float> f;
    for (int i = 0; i < 400000; ++i) { const uint32_t b = (uint32_t)rng(); float x; memcpy(&x, &b, 4); f.push_back(x); }
    for (int i = 0; i < 400000; ++i) {
        const uint64_t x = rng();
        const float q = (float)((int)(x & 0xffff) - 32768) / (float)(1 << ((x >> 16) & 15));
        f.push_back((x >> 20) & 1 ? std::nextafterf(q, 1e9f) : q);
    }
    for (int i = 0; i < 400000; ++i) {
        const uint64_t x = rng();
        const float t = (float)(((double)(x & 0xfffff) + 0.5) / 1000.0);
        const float w = (x >> 20) % 3 == 0 ? t : (x >> 20) % 3 == 1 ? std::nextafterf(t, 1e9f) : std::nextafterf(t, -1e9f);
        f.push_back((x >> 40) & 1 ? -w : w);
    }
    const float kFloatLimit = 549755813888.0f;           // 2^39
    for (const float s : {0.0f, -0.0f, INFINITY, -INFINITY, NAN, 1e-45f, -1e-45f, 1.17549435e-38f, kFloatLimit, -kFloatLimit,
                          std::nextafterf(kFloatLimit, 0.0f), -std::nextafterf(kFloatLimit, 0.0f), 3.4028235e38f})
        f.push_back(s);
    check_fixed<0>("float %.0lf", f, kFloatLimit);
    check_fixed<1>("float %.1lf", f, kFloatLimit);
    check_fixed<2>("float %.2lf", f, kFloatLimit);
    check_fixed<3>("float %.3lf", f, kFloatLimit);
    check_fixed<4>("float %.4lf", f, kFloatLimit);
    check_fixed<5>("float %.5lf", f, kFloatLimit);

    check_ints();
    check_rows();
    check_row_numbers();

    printf("host: %zu values, %zu refused, %zu bad\n", g_values, g_refused, g_bad);
    if (g_device) printf("device: %zu bad\n", g_dbad);
    const size_t bad = g_bad + g_dbad;
    printf(bad ? "FAILED\n" : "ok\n");
    return bad ? 1 : 0;
}
