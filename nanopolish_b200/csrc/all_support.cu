// all_support.cu — `nanopolish variants --calculate-all-support` on the device: the A/C/G/T read support of every called variant
// in one call.
//
// Replaces, for every (variant, read, base) at once, the scoring loop of
//   annotate_variants_with_all_support        ref: src/common/nanopolish_variant.cpp:801-859
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_event_subsequence, shared
//                                             with variant screening and homopolymer fixing)
//   Haplotype::apply_variant on the window    ref: src/nanopolish_haplotype.cpp:33-75 (decided on the host, per variant)
//   profile_hmm_score of the four haplotypes (K1, unchanged)
//
// Kernels, in the count -> scan -> fill -> emit -> score -> fold shape of homopolymer.cu:
//   sup_pairs_kernel<false>  a warp per variant, the records 32 at a time: the window's event sequences
//   (nph_scan_exclusive: each variant's first pair; one read-back sizes everything below)
//   sup_pairs_kernel<true>   the same walk, writing the pairs {record, e1, e2} in record order
//   sup_emit_kernel          thread per (pair, base): the k-mer ranks of the edited window, strand-resolved, and one nph_hmm_job
//   K1 (nph_score_device_jobs)
//   sup_fold_kernel          thread per pair: the table log-sum of the four scores in the reference's order, and the four
//                            differences score - log-sum in double
// exp, the fold over reads in record order and the division run on the host with the host's libm (DESIGN: glibc's double exp is
// not correctly rounded, and unlike expf / logf in libm_exact.cuh it cannot be checked exhaustively).
#include "nph_internal.cuh"
#include "exact_math.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kBases = 4;                            // the haplotypes of "ACGT"

struct SupPair { uint32_t record; int32_t e1, e2; };

// per variant, what the kernels need: the window's first base as an offset into the region reference, and the length of the
// reference allele apply_variant replaces (-1: it does not apply, every haplotype is the window)
struct SupVariant { int32_t win_off; int32_t del; };

struct SupArgs {
    const nph_meth_record* records;
    const int32_t* dense;
    const int32_t* first_valid;
    const SupVariant* variants;
    const uint8_t* ref;                              // the region reference
    int32_t region_start, flank;
    uint32_t n_records, n_variants;
};

// FILL = false: per variant the number of event sequences; FILL = true: the pairs
template <bool FILL>
__global__ void __launch_bounds__(kThreads) sup_pairs_kernel(const SupArgs a, uint64_t* __restrict__ n_pairs, const uint64_t* __restrict__ pair_off,
                                                             SupPair* __restrict__ pairs)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t vi = warp; vi < a.n_variants; vi += n_warps) {
        const int cs = a.region_start + a.variants[vi].win_off, ce = cs + 2 * a.flank;
        uint64_t n = 0;
        SupPair* out = FILL ? pairs + pair_off[vi] : nullptr;
        for (uint32_t base = 0; base < a.n_records; base += 32) {
            const uint32_t r = base + lane;
            int e1 = 0, e2 = 0;
            bool in = false;
            if (r < a.n_records) {
                const nph_meth_record R = a.records[r];
                in = nph_event_subsequence(R, a.dense + R.ref_off, a.first_valid[r], cs, ce, e1, e2);
            }
            const unsigned m = __ballot_sync(kFull, in);
            if (FILL && in) out[n + __popc(m & ((1u << lane) - 1u))] = SupPair{r, e1, e2};
            n += __popc(m);
        }
        if (!FILL && lane == 0) n_pairs[vi] = n;
    }
}

// base v of haplotype b of a variant: the window with its reference allele replaced by b at offset flank when apply_variant succeeds
__device__ __forceinline__ uint8_t sup_base(const SupArgs& a, const SupVariant& V, int b, int v)
{
    if (V.del < 0 || v < a.flank) return a.ref[V.win_off + v];
    if (v == a.flank) return (uint8_t)"ACGT"[b];
    return a.ref[V.win_off + v + V.del - 1];
}

// thread per (pair, base): job t = pair * 4 + base, ranks at kmer_stride per job
__global__ void sup_emit_kernel(const SupArgs a, const SupPair* __restrict__ pairs, const uint32_t* __restrict__ pair_variant, uint64_t n_pairs,
                                uint32_t kmer_stride, uint32_t k, uint8_t flags, nph_hmm_job* __restrict__ jobs, uint32_t* __restrict__ ranks)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_pairs * kBases) return;
    const uint64_t p = t / kBases;
    const int b = (int)(t % kBases);
    const SupPair P = pairs[p];
    const SupVariant V = a.variants[pair_variant[p]];
    const nph_meth_record R = a.records[P.record];
    const int len = 2 * a.flank + 1 - (V.del < 0 ? 0 : V.del - 1);
    const int nk = len - (int)k + 1;
    uint32_t* rk = ranks + t * kmer_stride;
    // HMMInputSequence::get_kmer_rank(q, k, rc) of the DNA alphabet (nph_dna_kmer_ranks, one k-mer at a time)
    for (int q = 0; q < nk; ++q) {
        uint8_t c[8];
        for (int i = 0; i < (int)k; ++i) c[i] = nph_dna_code(sup_base(a, V, b, q + i));
        uint32_t fw, rc;
        nph_dna_kmer_ranks(c, 0, (int)k, fw, rc);
        rk[q] = R.rc ? rc : fw;
    }
    nph_hmm_job jb;
    jb.rank_off = t * kmer_stride; jb.read = R.read; jb.model_id = R.model_id;
    jb.event_start = (uint32_t)P.e1; jb.event_stop = (uint32_t)P.e2; jb.n_kmers = (uint32_t)nk;
    jb.stride = R.rc ? -1 : 1;                    // EventAlignmentRecord::stride agrees with rc for every read the HMM accepts
    jb.rc = R.rc; jb.flags = flags; jb.reserved = 0;
    jobs[t] = jb;
}

// thread per pair: sum = s[0], then sum = add_logs(s[hi], sum) (p7_FLogsum on floats: the double overload narrows), and
// diff[hi] = double(s[hi]) - double(sum), the argument of the reference's exp
__global__ void sup_fold_kernel(const float* __restrict__ scores, uint64_t n_pairs, const float* __restrict__ tbl, double* __restrict__ diff)
{
    const uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    float s[kBases];
    for (int hi = 0; hi < kBases; ++hi) s[hi] = scores[p * kBases + hi];
    float sum = s[0];
    for (int hi = 1; hi < kBases; ++hi) sum = nph_flogsum(s[hi], sum, tbl);
    for (int hi = 0; hi < kBases; ++hi) diff[p * kBases + hi] = __dsub_rn((double)s[hi], (double)sum);
}

// the nph_support_variant checks, and apply_variant's outcome on the unedited window: window.substr(flank, len) == ref_seq, where
// substr clamps at the window's end (so a reference allele longer than flank + 1 bases never matches)
int check_variants(nph_ctx* ctx, const nph_support_variant* variants, size_t n_variants, const char* ref_seqs, size_t n_seq_bytes,
                   const nph_support_params& p, const char* ref, size_t n_ref, std::vector<SupVariant>& dev)
{
    const int64_t region_end = (int64_t)p.region_start + (int64_t)n_ref - 1;
    dev.resize(n_variants);
    for (size_t i = 0; i < n_variants; ++i) {
        const nph_support_variant& v = variants[i];
        const std::string at = "variant " + std::to_string(i) + ": ";
        if (!nph_slice_ok(v.ref_seq_off, v.ref_seq_len, n_seq_bytes)) { ctx->last_error = at + "ref_seq outside ref_seqs"; return NPH_ERR_INVALID; }
        const int64_t cs = (int64_t)v.ref_position - p.flank, ce = (int64_t)v.ref_position + p.flank;
        if (cs < p.region_start || ce > region_end) {
            ctx->last_error = at + "calling window [" + std::to_string(cs) + ", " + std::to_string(ce) + "] outside the region [" +
                              std::to_string(p.region_start) + ", " + std::to_string(region_end) + "] (substr_by_reference asserts)";
            return NPH_ERR_INVALID;
        }
        const size_t off = (size_t)(cs - p.region_start);
        const bool applies = v.ref_seq_len <= (uint32_t)p.flank + 1 && std::memcmp(ref + off + p.flank, ref_seqs + v.ref_seq_off, v.ref_seq_len) == 0;
        dev[i] = SupVariant{(int32_t)off, applies ? (int32_t)v.ref_seq_len : -1};
    }
    return NPH_OK;
}

} // namespace

extern "C" int nph_all_support_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                     const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                     const char* ref_bases, size_t n_ref_bases,
                                     const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                     const nph_meth_record* records, size_t n_records,
                                     const nph_support_params* params, const char* ref_seqs, size_t n_seq_bytes,
                                     const nph_support_variant* variants, size_t n_variants, double indel_bias,
                                     nph_support_result* out, nph_support_counts* counts_out)
{
    if (!ctx || !params || (n_variants && (!variants || !out)) || (n_seq_bytes && !ref_seqs)) return NPH_ERR_INVALID;
    if (n_records && (!records || !first_event || (n_deltas_total && !event_deltas))) return NPH_ERR_INVALID;
    if (!ref_bases || !ev_start_time) return NPH_ERR_INVALID;
    if (n_ref_bases < 1 || n_ref_bases > 0x7fffffffu || (int64_t)params->region_start + (int64_t)n_ref_bases - 1 > INT32_MAX) return NPH_ERR_INVALID;
    const nph_support_params p = *params;
    if (p.k < 1 || p.k > 8) { ctx->last_error = "k outside 1..8"; return NPH_ERR_INVALID; }
    if (p.flank < 0 || (int64_t)p.flank + 1 < (int64_t)p.k) { ctx->last_error = "flank + 1 below k (a haplotype without a k-mer)"; return NPH_ERR_INVALID; }
    if (p.alignment_flags & ~(NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP)) { ctx->last_error = "unknown alignment_flags"; return NPH_ERR_INVALID; }
    std::vector<SupVariant> dev;
    NPH_TRY(check_variants(ctx, variants, n_variants, ref_seqs, n_seq_bytes, p, ref_bases, n_ref_bases, dev));
    nph_support_counts cnt{};
    cnt.n_variants = n_variants;
    if (counts_out) *counts_out = cnt;
    if (n_variants == 0) { nph_timing_staged(ctx, 0.f, 0); return NPH_OK; }
    nph_ctx::SupportState& ss = ctx->sup;
    const auto run = [&]() -> int {
        NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
        // records index the event deltas, as screening's do
        NPH_TRY(nph_event_records_load(ctx, ss.ev, ref_bases, n_ref_bases, n_deltas_total, true, event_deltas, first_event, nullptr, 0,
                                       records, n_records, 0x3fffffffu, [&](size_t r, const nph_meth_record& R) {
            const DevModel& mod = ctx->models[R.model_id];
            if (mod.k == p.k && mod.alphabet_size == 4) return NPH_OK;
            ctx->last_error = "record " + std::to_string(r) + ": its model is not a nucleotide model of k = " + std::to_string(p.k);
            return NPH_ERR_INVALID;
        }));
        cudaStream_t st = ctx->stream;
        SupVariant* d_vars; uint64_t* d_n; uint64_t* d_off; uint64_t* d_scratch;
        NPH_TRY(nph_carve(ctx, ss.d_counts, [&](NphArena& c) {
            d_vars = c.take<SupVariant>(n_variants);
            d_n = c.take<uint64_t>(n_variants);
            d_off = c.take<uint64_t>(n_variants + 1);
            d_scratch = c.take<uint64_t>(nph_scan_scratch(n_variants));
        }));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_vars, dev.data(), sizeof(SupVariant) * n_variants, cudaMemcpyHostToDevice, st));
        const int32_t* dense;
        const int32_t* first_valid;
        NPH_TRY(nph_event_records_expand(ctx, ss.ev, &dense, &first_valid));
        const SupArgs a{ss.ev.d_records.p, dense, first_valid, d_vars, ss.ev.d_ref.p, p.region_start, p.flank, (uint32_t)n_records,
                        (uint32_t)n_variants};
        const int grid = (int)std::min<size_t>((n_variants + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 8);
        sup_pairs_kernel<false><<<grid, kThreads, 0, st>>>(a, d_n, nullptr, nullptr);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_scan_exclusive(ctx, d_n, (uint32_t)n_variants, d_off, d_scratch));
        std::vector<uint64_t> off(n_variants + 1);
        NPH_CUDA(ctx, cudaMemcpyAsync(off.data(), d_off, sizeof(uint64_t) * (n_variants + 1), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));                     // the one read-back that sizes the pair and job arrays
        const uint64_t n_pairs = off[n_variants];
        cnt.n_pairs = n_pairs;
        const uint64_t n_jobs = n_pairs * kBases;
        std::vector<double> h_diff(n_jobs);
        std::vector<SupPair> h_pairs(n_pairs);
        float kernel_ms = 0.f;
        int launches = 4;
        if (n_pairs) {
            std::vector<uint32_t> pair_variant(n_pairs);
            for (size_t i = 0; i < n_variants; ++i) std::fill(pair_variant.begin() + off[i], pair_variant.begin() + off[i + 1], (uint32_t)i);
            SupPair* d_pairs; uint32_t* d_pair_variant; double* d_diff;
            NPH_TRY(nph_carve(ctx, ss.d_pairs, [&](NphArena& c) {
                d_pairs = c.take<SupPair>(n_pairs);
                d_pair_variant = c.take<uint32_t>(n_pairs);
                d_diff = c.take<double>(n_jobs);
            }));
            NPH_CUDA(ctx, cudaMemcpyAsync(d_pair_variant, pair_variant.data(), sizeof(uint32_t) * n_pairs, cudaMemcpyHostToDevice, st));
            sup_pairs_kernel<true><<<grid, kThreads, 0, st>>>(a, nullptr, d_off, d_pairs);
            NPH_CUDA(ctx, cudaGetLastError());
            // every job gets room for the longest haplotype: the window plus one base (an empty reference allele that applies)
            const uint32_t kmer_stride = 2u * (uint32_t)p.flank + 2u - p.k + 1u;
            NPH_TRY(nph_reserve(ctx, ctx->d_ranks, (size_t)(n_jobs * kmer_stride)));
            NPH_TRY(nph_score_device_jobs(ctx, (size_t)n_jobs, (size_t)(n_jobs * kmer_stride), indel_bias, [&]() -> int {
                sup_emit_kernel<<<(unsigned)((n_jobs + 127) / 128), 128, 0, st>>>(a, d_pairs, d_pair_variant, n_pairs, kmer_stride, p.k,
                                                                                (uint8_t)p.alignment_flags, ctx->d_jobs.p, ctx->d_ranks.p);
                NPH_CUDA(ctx, cudaGetLastError());
                return NPH_OK;
            }));
            int nl = 0;
            if (nph_last_kernel_ms(ctx, &kernel_ms, &nl) == NPH_OK) launches += nl + 2;
            sup_fold_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, st>>>(ctx->d_scores.p, n_pairs, ctx->d_logsum.p, d_diff);
            NPH_CUDA(ctx, cudaGetLastError());
            NPH_CUDA(ctx, cudaMemcpyAsync(h_pairs.data(), d_pairs, sizeof(SupPair) * n_pairs, cudaMemcpyDeviceToHost, st));
            NPH_CUDA(ctx, cudaMemcpyAsync(h_diff.data(), d_diff, sizeof(double) * n_jobs, cudaMemcpyDeviceToHost, st));
            NPH_CUDA(ctx, cudaStreamSynchronize(st));
        }
        // the reference's host arithmetic on what the device found: per variant, in record order, support[hi] += exp(diff), then the
        // division by the number of event sequences (0 / 0 with none: a NaN, as the reference prints it)
        const auto t0 = std::chrono::steady_clock::now();
        for (size_t i = 0; i < n_variants; ++i) {
            double support[kBases] = {0.0, 0.0, 0.0, 0.0};
            for (uint64_t q = off[i]; q < off[i + 1]; ++q)
                for (int hi = 0; hi < kBases; ++hi) support[hi] += exp(h_diff[q * kBases + hi]);
            const size_t n = (size_t)(off[i + 1] - off[i]);
            for (int hi = 0; hi < kBases; ++hi) out[i].support[hi] = support[hi] / n;
            out[i].n_reads = (uint32_t)n;
            out[i].applied = dev[i].del >= 0 ? 1u : 0u;
        }
        cnt.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        cnt.n_jobs = n_jobs;
        for (uint64_t q = 0; q < n_pairs; ++q)
            cnt.n_dp_rows += (uint64_t)kBases * (uint64_t)((h_pairs[q].e1 > h_pairs[q].e2 ? h_pairs[q].e1 - h_pairs[q].e2 : h_pairs[q].e2 - h_pairs[q].e1) + 1);
        nph_timing_staged(ctx, kernel_ms, launches);
        return NPH_OK;
    };
    NPH_TRY(run());
    if (counts_out) *counts_out = cnt;
    return NPH_OK;
}
