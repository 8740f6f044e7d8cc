// homopolymer.cu — the likelihoods of `nanopolish variants --fix-homopolymers` on the device, for every calling window of a
// haplotype in one call.
//
// Replaces, for every (window, read, candidate length L = 3..9) at once, the scoring loop of
//   fix_homopolymers                          ref: src/nanopolish_call_variants.cpp:541-780 (the loop :624-683)
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_window_reads)
//   DurationModel::generate_aligned_durations ref: src/hmm/nanopolish_duration_model.cpp:17-40
//   profile_hmm_score / profile_hmm_align on the variant sequence (K1 and K3, unchanged)
// The haplotype scan, the calling ranges, the call and its application stay with the caller: a window arrives as its calling
// sequence and the offsets the reference derives from the haplotype (nph_hp_window).
//
// Kernels, after the window-read walk of window_reads.cu (count -> scan -> fill: each window's event sequences, TotalReads, and
// of those the ones the reference scores, abs(e_start - e_stop) >= 10, with the largest event span):
//   hp_emit_kernel          thread per (pair, L) of a chunk: the k-mer ranks of the variant sequence, strand-resolved, and ONE
//                           nph_hmm_job — the forward and the Viterbi call of the reference are the same triple
//   K1 (nph_score_device_jobs), then K3 on the same jobs (nph_viterbi_chunks, which runs the emit and K1 per chunk)
//   hp_duration_kernel      a warp per job: sum_duration over the path, slot by slot in path order, slots ascending
// The log-gamma terms and the fold in record order run on the host with the host's libm (DESIGN: glibc's double log and
// lgamma are not correctly rounded, and unlike expf / logf in libm_exact.cuh they cannot be checked exhaustively).
#include "nph_internal.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kL = NPH_HP_LENGTHS;
constexpr int kMinEvents = 10;                       // abs(e_start - e_stop) < 10 skips the read (:637)
constexpr double kShape = 2.461964;                  // GammaParameters::shape (:643)
constexpr double kMinDuration = 0.00025;             // MIN_DURATION, src/hmm/nanopolish_duration_model.h:17

struct HpArgs {
    const nph_meth_record* records;
    const nph_hp_window* windows;
    const uint8_t* seqs;
};

// base v of the variant sequence of length L (the calling sequence with the homopolymer erased or extended at edit_offset, :650-655)
// as a DNA code
__device__ __forceinline__ uint8_t hp_variant_code(const nph_hp_window& w, const uint8_t* __restrict__ seq, int L, int v)
{
    const int at = (int)w.edit_offset, diff = L - (int)w.hp_length;
    if (v < at) return nph_dna_code(seq[v]);
    if (diff > 0 && v < at + diff) return nph_dna_code((uint8_t)w.hp_base);
    return nph_dna_code(seq[v - diff]);
}

// thread per (pair, L) of the chunk [p0, p0 + n_pairs): job p * 7 + (L - 3), ranks at kmer_stride per job
__global__ void hp_emit_kernel(const HpArgs a, const NphWinPair* __restrict__ pairs, const uint32_t* __restrict__ pair_window, uint64_t p0,
                               uint64_t n_pairs, uint32_t kmer_stride, nph_hmm_job* __restrict__ jobs, uint32_t* __restrict__ ranks)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_pairs * kL) return;
    const uint64_t pl = t / kL;
    const int L = NPH_HP_MIN_LENGTH + (int)(t % kL);
    const NphWinPair P = pairs[p0 + pl];
    const nph_hp_window W = a.windows[pair_window[p0 + pl]];
    const nph_meth_record R = a.records[P.record];
    const uint8_t* seq = a.seqs + W.seq_off;
    const int k = (int)W.k;
    const int nk = (int)W.seq_len + L - (int)W.hp_length - k + 1;
    nph_window_ranks([&](int v) { return hp_variant_code(W, seq, L, v); }, nk, k, R.rc, ranks + t * kmer_stride);
    nph_hmm_job jb = nph_window_job(R, P, 0);     // alignment_flags = 0 (:543)
    jb.rank_off = t * kmer_stride; jb.model_id = R.model_id; jb.n_kmers = (uint32_t)nk;
    jobs[t] = jb;
}

// a warp per job: slots k0 + 2 .. k0 + L + 1 of generate_aligned_durations (each the durations of the path's non-K states of that
// k-mer, added in path order in double), summed ascending; *no_path set where K3 found none (the reference asserts)
__global__ void __launch_bounds__(kThreads) hp_duration_kernel(const HpArgs a, const NphWinPair* __restrict__ pairs,
                                                               const uint32_t* __restrict__ pair_window, uint64_t p0, uint64_t n_jobs,
                                                               const nph_align_state* __restrict__ states, const uint64_t* __restrict__ states_off,
                                                               const uint32_t* __restrict__ n_states, const DevRead* __restrict__ reads,
                                                               const float* __restrict__ duration, double* __restrict__ sum_out,
                                                               unsigned int* __restrict__ no_path)
{
    const int lane = threadIdx.x & 31;
    const uint64_t j = blockIdx.x * (uint64_t)kWarps + (threadIdx.x >> 5);
    if (j >= n_jobs) return;
    const uint64_t pl = j / kL;
    const int L = NPH_HP_MIN_LENGTH + (int)(j % kL);
    const NphWinPair P = pairs[p0 + pl];
    const nph_hp_window W = a.windows[pair_window[p0 + pl]];
    const float* dur = duration + reads[a.records[P.record].read].event_off;
    const nph_align_state* st = states + states_off[j];
    const uint32_t n = n_states[j];
    double slot = 0.0;
    if (lane < L) {
        const uint32_t kmer = W.k0 + 2 + (uint32_t)lane;
        for (uint32_t i = 0; i < n; ++i) {
            const nph_align_state s = st[i];
            if (s.state != 'K' && s.kmer_idx == kmer) slot = __dadd_rn(slot, (double)dur[s.event_idx]);
        }
    }
    double sum = 0.0;
    for (int t = 0; t < L; ++t) sum = __dadd_rn(sum, __shfl_sync(kFull, slot, t));
    if (lane == 0) {
        sum_out[p0 * kL + j] = sum;
        if (n == 0) atomicOr(no_path, 1u);
    }
}

// nph_hp_window checks that need only the window; the model k is checked per record at load
int check_windows(nph_ctx* ctx, const nph_hp_window* windows, size_t n_windows, size_t n_seq_bytes, int32_t region_start, size_t n_ref,
                  uint32_t& max_len)
{
    const int64_t region_end = (int64_t)region_start + (int64_t)n_ref - 1;
    max_len = 0;
    for (size_t i = 0; i < n_windows; ++i) {
        const nph_hp_window& w = windows[i];
        const std::string at = "window " + std::to_string(i) + ": ";
        if (w.k != 6) { ctx->last_error = at + "k != 6 (fix_homopolymers asserts a 6-mer model)"; return NPH_ERR_INVALID; }
        if (w.hp_length < NPH_HP_MIN_LENGTH || w.hp_length > NPH_HP_MAX_LENGTH) { ctx->last_error = at + "hp_length outside 3..9"; return NPH_ERR_INVALID; }
        if (!nph_slice_ok(w.seq_off, w.seq_len, n_seq_bytes)) { ctx->last_error = at + "calling sequence outside calling_seqs"; return NPH_ERR_INVALID; }
        if ((uint64_t)w.edit_offset + w.hp_length > w.seq_len) { ctx->last_error = at + "edit offset outside the calling sequence"; return NPH_ERR_INVALID; }
        // the last duration slot, k0 + L + 1, must be a k-mer of the variant sequence of every L: k0 + L + 2 <= seq_len + L - hp_length - k + 1
        if ((uint64_t)w.k0 + w.hp_length + w.k + 1 > w.seq_len) { ctx->last_error = at + "k0 + L + 2 past the variant sequence's k-mers"; return NPH_ERR_INVALID; }
        if (w.ref_calling_start > w.ref_calling_end || w.ref_calling_start < region_start || (int64_t)w.ref_calling_end > region_end) {
            ctx->last_error = at + "calling range outside the region"; return NPH_ERR_INVALID;
        }
        max_len = std::max(max_len, w.seq_len + NPH_HP_MAX_LENGTH - w.hp_length);
    }
    return NPH_OK;
}

} // namespace

extern "C" int nph_homopolymer_likelihoods_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                                 const float* ev_mean, const double* ev_start_time, const float* ev_duration, size_t n_events_total,
                                                 const char* ref_bases, size_t n_ref_bases,
                                                 const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                                 const nph_meth_record* records, size_t n_records,
                                                 const nph_hp_params* params, const char* calling_seqs, size_t n_seq_bytes,
                                                 const nph_hp_window* windows, size_t n_windows, double indel_bias,
                                                 nph_hp_likelihoods* out, nph_hp_counts* counts_out)
{
    if (!ctx || !params || !out || (n_windows && !windows) || (n_seq_bytes && !calling_seqs)) return NPH_ERR_INVALID;
    if (n_records && (!records || !first_event || (n_deltas_total && !event_deltas))) return NPH_ERR_INVALID;
    if (!ref_bases || !ev_start_time || (n_events_total && !ev_duration)) return NPH_ERR_INVALID;
    if (params->min_flanking_sequence < 7) { ctx->last_error = "min_flanking_sequence below 7"; return NPH_ERR_INVALID; }
    if (n_ref_bases < 1 || n_ref_bases > 0x7fffffffu) return NPH_ERR_INVALID;
    uint32_t max_len = 0;
    NPH_TRY(check_windows(ctx, windows, n_windows, n_seq_bytes, params->region_start, n_ref_bases, max_len));
    for (size_t i = 0; i < n_windows; ++i) out[i] = nph_hp_likelihoods{};
    nph_hp_counts cnt{};
    cnt.n_windows = n_windows;
    if (counts_out) *counts_out = cnt;
    if (n_windows == 0) { nph_timing_staged(ctx, 0.f, 0); return NPH_OK; }
    nph_ctx::HpState& hs = ctx->hp;
    // the reads go up whole before any kernel runs: K3 reads the levels without the forward kernels' wait on a pipelined upload
    const auto load = [&]() -> int {
        NPH_TRY(nph_region_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, ref_bases, n_ref_bases, event_deltas, n_deltas_total,
                                first_event, records, n_records, [&](size_t r, const nph_meth_record& R) {
            const DevModel& mod = ctx->models[R.model_id];
            if (mod.k == 6 && mod.alphabet_size == 4) return NPH_OK;
            ctx->last_error = "record " + std::to_string(r) + ": its model is not a nucleotide 6-mer model";
            return NPH_ERR_INVALID;
        }));
        return nph_reserve(ctx, hs.d_in, sizeof(nph_hp_window) * n_windows + n_seq_bytes + sizeof(float) * n_events_total + 1024);
    };
    const auto run = [&]() -> int {
        NPH_TRY(load());
        cudaStream_t st = ctx->stream;
        NphArena in{hs.d_in.p};
        nph_hp_window* d_windows = in.take<nph_hp_window>(n_windows);
        uint8_t* d_seqs = in.take<uint8_t>(n_seq_bytes);
        float* d_dur = in.take<float>(n_events_total);
        NPH_CUDA(ctx, cudaMemcpyAsync(d_windows, windows, sizeof(nph_hp_window) * n_windows, cudaMemcpyHostToDevice, st));
        if (n_seq_bytes) NPH_CUDA(ctx, cudaMemcpyAsync(d_seqs, calling_seqs, n_seq_bytes, cudaMemcpyHostToDevice, st));
        if (n_events_total) NPH_CUDA(ctx, cudaMemcpyAsync(d_dur, ev_duration, sizeof(float) * n_events_total, cudaMemcpyHostToDevice, st));
        std::vector<int2> bounds(n_windows);
        for (size_t i = 0; i < n_windows; ++i) bounds[i] = make_int2(windows[i].ref_calling_start, windows[i].ref_calling_end);
        NphWindowReads wr;
        NPH_TRY(nph_window_reads(ctx, bounds, kMinEvents, wr));
        const std::vector<uint64_t>& off = wr.off;
        const uint64_t n_pairs = wr.n_pairs();
        for (size_t i = 0; i < n_windows; ++i) { out[i].total_reads = wr.met[i]; out[i].scored_reads = (uint32_t)(off[i + 1] - off[i]); }
        cnt.n_pairs = n_pairs;
        if (n_pairs == 0) { nph_timing_staged(ctx, 0.f, 4); return NPH_OK; }
        const uint64_t n_jobs = n_pairs * kL;
        float* d_fwd; double* d_sum; unsigned int* d_no_path;
        NPH_TRY(nph_carve(ctx, hs.d_jobs, [&](NphArena& c) {
            d_fwd = c.take<float>(n_jobs);
            d_sum = c.take<double>(n_jobs);
            d_no_path = c.take<unsigned int>(1);
        }));
        NPH_CUDA(ctx, cudaMemsetAsync(d_no_path, 0, sizeof(unsigned int), st));
        const HpArgs a{ctx->region.ev.d_records.p, d_windows, d_seqs};
        // chunks of whole pairs (kL jobs each) whose states fit the budget; every job gets room for the batch's largest path
        const uint32_t kmer_stride = max_len - 6 + 1;
        // what nph_last_kernel_ms reports: the forward kernels (timed inside nph_score_device_jobs), the state-offset kernel, K3 and
        // the duration kernel of every chunk; the pair kernels, the scan, the emit kernel and the forward scheduler run outside those windows (in the
        // whole-call time only).  launches counts every launch of the call.
        float kernel_ms = 0.f, vit_ms = 0.f;
        int launches = 6, vit_launches = 0;
        NPH_TRY(nph_viterbi_chunks(ctx, hs.d_states, n_jobs, (uint64_t)params->max_chunk_pairs * kL, kL, kmer_stride, wr.max_rows,
            [&](uint64_t j0, uint64_t nj, uint64_t& first) -> int {
                const uint64_t p0 = j0 / kL, np = nj / kL;
                NPH_TRY(nph_reserve(ctx, ctx->d_ranks, (size_t)(nj * kmer_stride)));
                NPH_TRY(nph_score_device_jobs(ctx, (size_t)nj, (size_t)(nj * kmer_stride), indel_bias, [&]() -> int {
                    hp_emit_kernel<<<(unsigned)((nj + 127) / 128), 128, 0, st>>>(a, wr.d_pairs, wr.d_pair_win, p0, np, kmer_stride,
                                                                                   ctx->d_jobs.p, ctx->d_ranks.p);
                    NPH_CUDA(ctx, cudaGetLastError());
                    return NPH_OK;
                }));
                float ms = 0.f; int nl = 0;
                if (nph_last_kernel_ms(ctx, &ms, &nl) == NPH_OK) { kernel_ms += ms; launches += nl + 1; }
                NPH_CUDA(ctx, cudaMemcpyAsync(d_fwd + j0, ctx->d_scores.p, sizeof(float) * nj, cudaMemcpyDeviceToDevice, st));
                first = 0;                                // each chunk's jobs are emitted from index 0
                return NPH_OK;
            },
            [&](const NphVitChunk& c) -> int {
                hp_duration_kernel<<<(unsigned)((c.n + kWarps - 1) / kWarps), kThreads, 0, st>>>(a, wr.d_pairs, wr.d_pair_win, c.j0 / kL, c.n, c.states,
                                                                                               c.states_off, c.n_states, ctx->d_reads.p, d_dur,
                                                                                               d_sum, d_no_path);
                NPH_CUDA(ctx, cudaGetLastError());
                return NPH_OK;
            },
            &vit_ms, &vit_launches, &cnt.n_chunks));
        kernel_ms += vit_ms;
        launches += vit_launches;
        // the reference's host arithmetic on what the device found: per pair local_avg, per job the log-gamma term, folded per
        // window in record order
        std::vector<NphWinPair> h_pairs(n_pairs);
        std::vector<float> h_fwd(n_jobs);
        std::vector<double> h_sum(n_jobs);
        unsigned int no_path = 0;
        NPH_CUDA(ctx, cudaMemcpyAsync(h_pairs.data(), wr.d_pairs, sizeof(NphWinPair) * n_pairs, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(h_fwd.data(), d_fwd, sizeof(float) * n_jobs, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(h_sum.data(), d_sum, sizeof(double) * n_jobs, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(&no_path, d_no_path, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));
        if (no_path) { ctx->last_error = "profile_hmm_align found no path for a job (the reference asserts)"; return NPH_ERR_INVALID; }
        const auto t0 = std::chrono::steady_clock::now();
        double lgamma_na[kL];
        for (int l = 0; l < kL; ++l) lgamma_na[l] = lgamma((double)(NPH_HP_MIN_LENGTH + l) * kShape);
        for (size_t i = 0; i < n_windows; ++i) {
            const double local_bases = (double)windows[i].seq_len;
            for (uint64_t p = off[i]; p < off[i + 1]; ++p) {
                const NphWinPair& P = h_pairs[p];
                const double* t = ev_start_time + reads[records[P.record].read].event_off;
                // SquiggleRead::get_time: float(start_time[e] - start_time[0]), subtracted in float
                const float ts = (float)(t[P.e1] - t[0]), te = (float)(t[P.e2] - t[0]);
                const double local_time = std::fabs(ts - te);
                const double local_avg = local_time / local_bases;
                const double rate = (1 / local_avg) * kShape;
                const double log_rate = log(rate);
                for (int l = 0; l < kL; ++l) {
                    const uint64_t j = p * kL + l;
                    out[i].event_lik[l] += h_fwd[j];
                    const double x = h_sum[j], na = (double)(NPH_HP_MIN_LENGTH + l) * kShape;
                    // DurationModel::log_gamma_sum (src/hmm/nanopolish_duration_model.cpp:52-58).  The reference adds it only for
                    // PORETYPE_R9 reads (:666); the profile HMM here is the R9 one, so every read of this call is an R9 read
                    // (include/nph.h) and the term is always added
                    const double log_gamma = x > kMinDuration ? (na * log_rate) - lgamma_na[l] + (na - 1) * log(x) - rate * x : 0.0f;
                    out[i].duration_lik[l] += log_gamma;
                }
            }
        }
        cnt.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        cnt.n_jobs = n_jobs;
        for (size_t i = 0; i < n_windows; ++i) cnt.n_dp_rows += 2ull * kL * wr.rows[i];
        nph_timing_staged(ctx, kernel_ms, launches);
        return NPH_OK;
    };
    NPH_TRY(run());
    if (counts_out) *counts_out = cnt;
    return NPH_OK;
}
