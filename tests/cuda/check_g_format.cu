// check_g_format — the "%g" formatter and the eventalign.tsv row of tsv_format.cuh against the C library:
//   --host:   put_g6 / g6_len == snprintf("%g") on EVERY float of the supported domain (+-0 and 2^-17 <= |v| < 2^39, both signs,
//             about 9.4e8 values, OpenMP over the binades) and refusal of every float outside it;
//             ea_row_numbers / ea_row_len / put_ea_row / ea_scaled_sample against snprintf with the reference's format strings
//             on seeded random rows: forward and rc k-mers, 'B' states (inf, -inf, and the refused 0 / 0), --scale-events,
//             --signal-index, names and read indices;
//   --device: the same functions compiled for the device, on every 61st float of the domain and its edges, and on the same rows.
// Build: nvcc -O3 -fmad=false -Xcompiler -fopenmp -gencode arch=compute_90a,code=sm_90a -I nanopolish_b200/csrc tests/cuda/check_g_format.cu
#include "tsv_format.cuh"
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <random>
#include <string>
#include <vector>
#include <cuda_runtime.h>

using namespace nph_tsv;

static bool in_domain(uint32_t bits)
{
    const uint32_t mag = bits & 0x7fffffffu, expo = mag >> 23;
    return mag == 0 || (expo >= 127 - 17 && expo < 127 + 39);
}

// 0: fine; 1: wrong refusal; 2: wrong text or length
static int check_one(uint32_t bits)
{
    float v;
    memcpy(&v, &bits, 4);
    const G6 g = g6_of(v);
    if (g.ok != in_domain(bits)) return 1;
    if (!g.ok) return 0;
    char got[32], ref[32];
    char* e = put_g6(got, g);
    *e = 0;
    snprintf(ref, sizeof ref, "%g", (double)v);
    return (strcmp(got, ref) == 0 && (int)(e - got) == g6_len(g)) ? 0 : 2;
}

static size_t host_numbers()
{
    size_t bad = 0, checked = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : bad, checked)
    for (int hi = 0; hi < 512; ++hi) {                       // sign and exponent
        const uint32_t base = (uint32_t)hi << 23;
        const bool inside = in_domain(base | 1u);
        // outside the domain only the refusal is at stake: every 7th mantissa
        for (uint32_t m = 0; m < (1u << 23); m += inside ? 1u : 7u) {
            const int rc = check_one(base | m);
            if (rc) {
                bad += 1;
                if (bad < 5) { float v; const uint32_t b = base | m; memcpy(&v, &b, 4); printf("bad (%d): %08x %a\n", rc, b, (double)v); }
            }
            checked += 1;
        }
    }
    printf("  %%g host: %zu values, %zu bad\n", checked, bad);
    return bad;
}

// ---- rows ---------------------------------------------------------------------------------------------------------
struct RowCase {
    float ev_mean, level, stdv, duration;
    double start_time, level_mean, level_stdv;
    EaRead rd;
    char state;
    uint8_t rc, scale_events, signal_index, named;
    int ref_position, event_idx;
    uint32_t pos, n, k, contig_off, contig_len, name_off, name_len, ref_off;      // ref and rc_ref: n characters at ref_off / ref_off + n
    uint64_t read_idx;
    float raw[4];                                                                // four raw samples at indices 0 .. 3
};

__host__ __device__ static int format_case(const RowCase& c, const char* pool, char* out, float* scaled4)
{
    const EaRowNums r = ea_row_numbers(c.ev_mean, c.level, c.stdv, c.duration, c.start_time, c.state, c.level_mean, c.level_stdv, c.rd,
                                       c.scale_events != 0, c.signal_index != 0);
    for (int i = 0; i < 4; ++i) scaled4[i] = ea_scaled_sample(c.raw[i], (uint64_t)i, c.rd);
    if (!r.ok) return -1;
    EaRow w;
    w.contig = pool + c.contig_off; w.contig_len = c.contig_len;
    w.ref_position = c.ref_position;
    w.kmers = ea_kmers_at(pool + c.ref_off, pool + c.ref_off + c.n, c.n, c.pos, c.k, c.rc != 0, c.state);
    w.k = c.k;
    w.name = c.named ? pool + c.name_off : nullptr; w.name_len = c.name_len;
    w.read_idx = c.read_idx;
    w.strand = 't';
    w.event_idx = c.event_idx;
    w.signal_index = c.signal_index != 0;
    char* e = put_ea_row(out, w, r);
    *e = 0;
    return (int)(e - out) == (int)ea_row_len(w, r) ? (int)(e - out) : -2;
}

constexpr int kRowStride = 512;

__global__ void row_kernel(const RowCase* cases, size_t n, const char* pool, char* out, int* len, float* scaled)
{
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) len[i] = format_case(cases[i], pool, out + kRowStride * i, scaled + 4 * i);
}

struct Rows { std::vector<RowCase> cases; std::string pool; std::vector<std::string> want; std::vector<float> scaled; };

static Rows make_rows()
{
    Rows R;
    std::mt19937_64 rng(20240611);
    auto add = [&](const std::string& s) { const uint32_t off = (uint32_t)R.pool.size(); R.pool += s; return off; };
    const std::vector<std::string> contigs = {"chr20", "GL000220.1", "c"};
    const std::vector<std::string> names = {"r", "5a8a4b1f-e0f5-4a6e-9b5e-0c3c1d2f0e11", std::string(90, 'n')};
    std::uniform_real_distribution<double> u01(0.0, 1.0);
    for (int i = 0; i < 60000; ++i) {
        RowCase c{};
        const std::string& contig = contigs[rng() % contigs.size()];
        const std::string& name = names[rng() % names.size()];
        c.k = 5 + (uint32_t)(rng() & 1);
        c.n = 40 + (uint32_t)(rng() % 60);
        std::string ref(c.n, 'A'), rc_ref(c.n, 'A');
        for (uint32_t j = 0; j < c.n; ++j) { const int b = (int)(rng() % 4); ref[j] = "ACGT"[b]; rc_ref[c.n - 1 - j] = "TGCA"[b]; }
        c.contig_off = add(contig); c.contig_len = (uint32_t)contig.size();
        c.name_off = add(name); c.name_len = (uint32_t)name.size();
        c.ref_off = add(ref); add(rc_ref);
        c.pos = (uint32_t)(rng() % (c.n - c.k + 1));
        c.ref_position = (int)(rng() % 250000000) + (int)c.pos;
        c.event_idx = (int)(rng() % 2000000);
        c.read_idx = i % 50 == 0 ? ~(uint64_t)0 : rng() % 100000;        // read_idx -1 prints as size_t
        c.named = (uint8_t)(rng() & 1); c.rc = (uint8_t)(rng() & 1);
        c.scale_events = (uint8_t)((rng() >> 3) & 1); c.signal_index = (uint8_t)((rng() >> 4) & 1);
        c.state = i % 9 == 0 ? 'B' : 'M';
        c.ev_mean = (float)(40.0 + 110.0 * u01(rng));
        if (i % 9 == 0 && i % 2 == 0) c.ev_mean = -c.ev_mean;           // -inf at a 'B' state
        if (i % 999 == 0) { c.ev_mean = 0.0f; c.state = 'B'; c.scale_events = 0; }   // 0 / 0: refused
        c.level = (float)(c.ev_mean - 0.3 * u01(rng));
        c.stdv = (float)(0.3 + 4.0 * u01(rng));
        c.duration = (float)((double)(3 + rng() % 60) / 4000.0);
        c.start_time = 3000.0 * u01(rng);
        c.level_mean = 50.0 + 90.0 * u01(rng); c.level_stdv = 0.8 + 3.0 * u01(rng);
        c.rd.scale = 0.8 + 0.4 * u01(rng); c.rd.shift = -15.0 + 30.0 * u01(rng); c.rd.drift = 1e-3 * (u01(rng) - 0.5);
        c.rd.var = 0.7 + 0.8 * u01(rng); c.rd.sqrt_var = std::sqrt(c.rd.var);
        c.rd.sample_rate = 4000.0; c.rd.sample_start_time = i % 3 == 0 ? 0 : rng() % 100000;
        for (float& s : c.raw) s = (float)(60.0 + 80.0 * u01(rng));
        R.cases.push_back(c);

        // the reference's statements (eventalign.cpp:431-460, squiggle_read.h:149-171, 217-226, squiggle_read.cpp:393-428)
        float event_mean = c.ev_mean, model_mean = 0.0, model_stdv = 0.0;
        if (c.scale_events) {
            event_mean = (float)((c.level - c.rd.shift) / c.rd.scale);
            if (c.state != 'B') { model_mean = (float)c.level_mean; model_stdv = (float)c.level_stdv; }
        } else if (c.state != 'B') {
            model_mean = (float)(c.rd.scale * c.level_mean + c.rd.shift);
            model_stdv = (float)(c.level_stdv * c.rd.var);
        }
        const float standard_level = (float)((event_mean - model_mean) / (sqrt(c.rd.var) * model_stdv));
        const std::string ref_kmer = ref.substr(c.pos, c.k);
        const std::string model_kmer = c.state == 'B' ? std::string(c.k, 'N') : c.rc ? rc_ref.substr(c.n - c.pos - c.k, c.k) : ref_kmer;
        char buf[1024];
        int o = snprintf(buf, sizeof buf, "%s\t%d\t%s\t", contig.c_str(), c.ref_position, ref_kmer.c_str());
        if (c.named) o += snprintf(buf + o, sizeof buf - o, "%s\t%c\t", name.c_str(), 't');
        else o += snprintf(buf + o, sizeof buf - o, "%zu\t%c\t", (size_t)c.read_idx, 't');
        o += snprintf(buf + o, sizeof buf - o, "%d\t%.2lf\t%.3lf\t%.5lf\t", c.event_idx, event_mean, c.stdv, c.duration);
        o += snprintf(buf + o, sizeof buf - o, "%s\t%.2lf\t%.2lf\t%.2lf", model_kmer.c_str(), model_mean, model_stdv, standard_level);
        if (c.signal_index) {
            const size_t a = (size_t)(c.start_time * c.rd.sample_rate) - c.rd.sample_start_time;
            const size_t b = (size_t)((c.start_time + (double)c.duration) * c.rd.sample_rate) - c.rd.sample_start_time;
            o += snprintf(buf + o, sizeof buf - o, "\t%zu\t%zu", a, b);
        }
        R.want.push_back(std::isnan(standard_level) ? std::string() : std::string(buf));       // "": refused
        for (int s = 0; s < 4; ++s) {
            const double t = (c.rd.sample_start_time + (uint64_t)s) / c.rd.sample_rate;
            double v = c.raw[s] - c.rd.shift;
            v -= (t - (c.rd.sample_start_time / c.rd.sample_rate)) * c.rd.drift;
            v /= c.rd.scale;
            R.scaled.push_back((float)v);
        }
    }
    return R;
}

static size_t compare_rows(const Rows& R, const char* where, const char* out, const int* len, const float* scaled)
{
    size_t bad = 0, refused = 0, infs = 0;
    for (size_t i = 0; i < R.cases.size(); ++i) {
        const bool same_samples = memcmp(scaled + 4 * i, R.scaled.data() + 4 * i, 16) == 0;
        if (R.want[i].empty()) {
            refused += 1;
            if (len[i] != -1 || !same_samples) { if (++bad < 5) printf("%s row %zu: a 0 / 0 row was not refused\n", where, i); }
            continue;
        }
        infs += R.want[i].find("inf") != std::string::npos;
        if (len[i] != (int)R.want[i].size() || R.want[i] != out + kRowStride * i || !same_samples)
            if (++bad < 5) printf("%s row %zu (%d): %s\n   vs %s\n", where, i, len[i], out + kRowStride * i, R.want[i].c_str());
    }
    printf("  rows %s: %zu rows (%zu with inf, %zu refused), %zu bad\n", where, R.cases.size(), infs, refused, bad);
    return bad + (infs == 0) + (refused == 0);
}

static size_t host_rows(const Rows& R)
{
    std::vector<char> out((size_t)kRowStride * R.cases.size());
    std::vector<int> len(R.cases.size());
    std::vector<float> scaled(4 * R.cases.size());
    for (size_t i = 0; i < R.cases.size(); ++i) len[i] = format_case(R.cases[i], R.pool.data(), &out[kRowStride * i], &scaled[4 * i]);
    return compare_rows(R, "host", out.data(), len.data(), scaled.data());
}

// ---- device -------------------------------------------------------------------------------------------------------
constexpr int kNumStride = 16;

__global__ void g6_kernel(const uint32_t* bits, size_t n, char* out, signed char* len)
{
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v;
    memcpy(&v, &bits[i], 4);
    const G6 g = g6_of(v);
    if (!g.ok) { len[i] = -1; return; }
    char* e = put_g6(out + kNumStride * i, g);
    *e = 0;
    len[i] = (int)(e - (out + kNumStride * i)) == g6_len(g) ? (signed char)g6_len(g) : (signed char)-2;
}

#define CK(call) do { if ((call) != cudaSuccess) { printf("no device: %s\n", #call); return 2; } } while (0)

static int device_checks(const Rows& R)
{
    std::vector<uint32_t> bits;
    for (uint64_t b = 0; b < (1ull << 32); b += 61) bits.push_back((uint32_t)b);
    for (uint32_t s = 0; s < 2; ++s)
        for (uint32_t ex : {0u, 1u, 109u, 110u, 111u, 165u, 166u, 254u, 255u})
            for (uint32_t m : {0u, 1u, 0x7fffffu}) bits.push_back(s << 31 | ex << 23 | m);
    const size_t n = bits.size();
    uint32_t* dbits; char* dout; signed char* dlen;
    CK(cudaMalloc(&dbits, 4 * n)); CK(cudaMalloc(&dout, (size_t)kNumStride * n)); CK(cudaMalloc(&dlen, n));
    CK(cudaMemcpy(dbits, bits.data(), 4 * n, cudaMemcpyHostToDevice));
    g6_kernel<<<(unsigned)((n + 255) / 256), 256>>>(dbits, n, dout, dlen);
    std::vector<char> out((size_t)kNumStride * n);
    std::vector<signed char> len(n);
    CK(cudaMemcpy(out.data(), dout, out.size(), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(len.data(), dlen, n, cudaMemcpyDeviceToHost));
    size_t bad = 0;
    char ref[32];
    for (size_t i = 0; i < n; ++i) {
        float v;
        memcpy(&v, &bits[i], 4);
        if (!in_domain(bits[i])) { if (len[i] != -1 && ++bad < 5) printf("device formatted %08x\n", bits[i]); continue; }
        snprintf(ref, sizeof ref, "%g", (double)v);
        if ((len[i] != (int)strlen(ref) || strcmp(ref, &out[kNumStride * i]) != 0) && ++bad < 5) printf("device %08x: %s vs %s\n", bits[i], &out[kNumStride * i], ref);
    }
    printf("  %%g device: %zu values, %zu bad\n", n, bad);
    cudaFree(dbits); cudaFree(dout); cudaFree(dlen);

    const size_t nr = R.cases.size();
    RowCase* dc; char* dpool; char* drow; int* drl; float* dsc;
    CK(cudaMalloc(&dc, sizeof(RowCase) * nr)); CK(cudaMalloc(&dpool, R.pool.size())); CK(cudaMalloc(&drow, (size_t)kRowStride * nr));
    CK(cudaMalloc(&drl, sizeof(int) * nr)); CK(cudaMalloc(&dsc, 16 * nr));
    CK(cudaMemcpy(dc, R.cases.data(), sizeof(RowCase) * nr, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dpool, R.pool.data(), R.pool.size(), cudaMemcpyHostToDevice));
    row_kernel<<<(unsigned)((nr + 127) / 128), 128>>>(dc, nr, dpool, drow, drl, dsc);
    std::vector<char> rows((size_t)kRowStride * nr);
    std::vector<int> rl(nr);
    std::vector<float> sc(4 * nr);
    CK(cudaMemcpy(rows.data(), drow, rows.size(), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rl.data(), drl, sizeof(int) * nr, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(sc.data(), dsc, 16 * nr, cudaMemcpyDeviceToHost));
    bad += compare_rows(R, "device", rows.data(), rl.data(), sc.data());
    cudaFree(dc); cudaFree(dpool); cudaFree(drow); cudaFree(drl); cudaFree(dsc);
    return bad ? 1 : 0;
}

int main(int argc, char** argv)
{
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode != "--host" && mode != "--device" && mode != "--host-rows") { printf("usage: check_g_format --host | --host-rows | --device\n"); return 2; }
    const Rows R = make_rows();
    int rc;
    if (mode == "--device") rc = device_checks(R);
    else rc = (host_rows(R) + (mode == "--host" ? host_numbers() : 0)) ? 1 : 0;
    printf(rc ? "FAILED\n" : "ok\n");
    return rc;
}
