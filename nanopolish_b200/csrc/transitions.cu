// transitions.cu — `nanopolish scorereads --train-transitions` on the device: the forward scores of a job batch and the transition
// training counts of the Viterbi paths of the same jobs, in one call.
//
// Replaces, for every segment model_score scores (ref: src/nanopolish_scorereads.cpp:116-203, the training block :190-196):
//   profile_hmm_align(sequence, data) with flags 0            K3, unchanged (nph_viterbi_chunks)
//   TransitionParameters::add_training_from_alignment        ref: src/hmm/nanopolish_transition_parameters.cpp:294-368
//   the binning of TransitionParameters::train              ref: :370-436, get_skip_bin (nanopolish_transition_parameters.h:101-111)
// train() and print() stay with the caller: they need only the per-bin counts (include/nph.h).
//
// Layout:
//   K1 on the jobs (nph_hmm_score_batch_seq: the same upload, scheduler and kernels), which leaves the jobs, their ranks, the read
//   transitions and the flank table on the device
//   K3 on the same jobs in chunks of Viterbi states (nph_viterbi_chunks), and per chunk
//   tt_observe_kernel   a warp per job, lanes striding the path: every count into the block's shared records (integer atomics),
//                       flushed into the group records with 64-bit integer atomics when the block ends
//   one D2H of the records.  No path leaves the device.
#include "nph_internal.cuh"
#include <algorithm>
#include <string>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kWords = (int)(sizeof(nph_transition_counts) / sizeof(uint64_t));      // 81
constexpr int kMatches = 18, kSkips = 20, kTotal = 21, kCount = kTotal + NPH_TT_BINS; // word offsets in nph_transition_counts
static_assert(kWords == kCount + NPH_TT_BINS, "nph_transition_counts layout");

// refusal bits of the flag word
constexpr unsigned kNoPath = 1u, kBadState = 2u, kKmerRange = 4u, kNonFinite = 8u;

struct TtArgs {
    const nph_hmm_job* jobs;         // the device copies: rank_off indexes ranks
    const uint32_t* ranks;
    const DevRead* reads;
    const DevModelView* models;
    const uint8_t* groups;           // nullptr: every job in group 0
    uint32_t n_groups, ignore_edge;
    float log_inv_sqrt_2pi;
    unsigned long long* counts;      // n_groups x kWords
    unsigned int* flags;
};

// statechar2index (nanopolish_transition_parameters.cpp:273-282); -1 where the reference asserts
__device__ __forceinline__ int tt_state_index(char s) { return s == 'M' ? 0 : s == 'B' ? 1 : s == 'K' ? 2 : -1; }

// a warp per job of the chunk [j0, j0 + n); job j0 + i is ctx->d_jobs[j0 + i], its path at states + states_off[i]
__global__ void __launch_bounds__(kThreads) tt_observe_kernel(const TtArgs a, uint64_t j0, uint64_t n, const nph_align_state* __restrict__ states,
                                                              const uint64_t* __restrict__ states_off, const uint32_t* __restrict__ n_states)
{
    extern __shared__ unsigned long long s_cnt[];              // n_groups x kWords
    for (uint32_t i = threadIdx.x; i < a.n_groups * kWords; i += kThreads) s_cnt[i] = 0ull;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    unsigned bad = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)kWarps + (threadIdx.x >> 5); i < n; i += (uint64_t)gridDim.x * kWarps) {
        const uint64_t j = j0 + i;
        const uint32_t m = n_states[i];
        if (m == 0) { bad |= kNoPath; continue; }              // profile_hmm_align asserts
        if (m <= a.ignore_edge) continue;                      // "do nothing if the alignment is too short"
        const nph_hmm_job jb = a.jobs[j];
        const DevRead rd = a.reads[jb.read];
        const DevModelView mv = a.models[jb.model_id];
        const uint32_t* rk = a.ranks + jb.rank_off;
        const nph_align_state* p = states + states_off[i];
        unsigned long long* c = s_cnt + (a.groups ? a.groups[j] : 0) * kWords;
        for (uint32_t pi = lane; pi < m; pi += 32) {
            const nph_align_state cur = p[pi];
            const nph_align_state prv = pi ? p[pi - 1] : cur;
            const int s = tt_state_index(cur.state);
            const int ps = pi ? tt_state_index(prv.state) : 0;   // prev_s starts as 'M'
            if (s < 0 || ps < 0) { bad |= kBadState; continue; }
            const bool kmer_move = pi == 0 || prv.kmer_idx != cur.kmer_idx;
            const int t = ps * 6 + 2 * s + (kmer_move ? 1 : 0);
            const bool interior = pi > a.ignore_edge && pi < m - a.ignore_edge;
            atomicAdd(&c[t], interior ? 2ull : 1ull);              // add_transition_observation, twice inside the edges
            if (s == 0) atomicAdd(&c[kMatches], 1ull);
            if (s == 2) atomicAdd(&c[kSkips], 1ull);
            if (!interior || s == 1) continue;
            const uint32_t from = prv.kmer_idx;
            const uint32_t to = (s == 2 && ps == 0) ? from + 1 : cur.kmer_idx;   // only the first k-mer of a skip after a match
            if (from >= jb.n_kmers || to >= jb.n_kmers) { bad |= kKmerRange; continue; }
            // get_scaled_gaussian_from_pore_model_state's mean: scale * level_mean + shift in FP64, narrowed to float
            const float l1 = nph_scaled_gaussian(mv, rd, rk[from], a.log_inv_sqrt_2pi).x;
            const float l2 = nph_scaled_gaussian(mv, rd, rk[to], a.log_inv_sqrt_2pi).x;
            if (!isfinite(l1) || !isfinite(l2)) { bad |= kNonFinite; continue; }
            // get_skip_bin: (size_t)(fabs(l1 - l2) / 0.5) in double, clamped to the last bin
            const double q = __ddiv_rn(fabs(__dsub_rn((double)l1, (double)l2)), 0.5);
            const int b = q >= (double)(NPH_TT_BINS - 1) ? NPH_TT_BINS - 1 : (int)q;
            atomicAdd(&c[kTotal + b], 1ull);
            if (s == 2) atomicAdd(&c[kCount + b], 1ull);
        }
    }
    if (bad) atomicOr(a.flags, bad);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < a.n_groups * kWords; i += kThreads)
        if (s_cnt[i]) atomicAdd(&a.counts[i], s_cnt[i]);
}

} // namespace

extern "C" int nph_train_transitions_batch(nph_ctx* ctx,
                                           const nph_read* reads, size_t n_reads,
                                           const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                           const uint8_t* seq_codes, size_t n_codes_total,
                                           const nph_hmm_job* jobs, size_t n_jobs, const uint8_t* groups,
                                           nph_tt_params* params, double indel_bias,
                                           float* scores_out, nph_transition_counts* counts_out)
{
    if (!ctx || !params || !counts_out || (n_jobs && (!jobs || !scores_out || !seq_codes))) return NPH_ERR_INVALID;
    const uint32_t n_groups = params->n_groups;
    if (n_groups < 1 || n_groups > NPH_TT_MAX_GROUPS) { ctx->last_error = "n_groups outside 1..256"; return NPH_ERR_INVALID; }
    for (uint32_t g = 0; g < n_groups; ++g) counts_out[g] = nph_transition_counts{};
    params->n_chunks_out = 0;
    params->viterbi_ms_out = params->observe_ms_out = 0.f;
    if (n_jobs == 0) { nph_timing_staged(ctx, 0.f, 0); return NPH_OK; }
    uint32_t max_K = 1, max_E = 1;
    for (size_t j = 0; j < n_jobs; ++j) {
        if (groups && groups[j] >= n_groups) {
            ctx->last_error = "job " + std::to_string(j) + ": group " + std::to_string(groups[j]) + " >= n_groups";
            return NPH_ERR_INVALID;
        }
        max_K = std::max(max_K, jobs[j].n_kmers);
        const uint32_t e = jobs[j].event_start > jobs[j].event_stop ? jobs[j].event_start - jobs[j].event_stop : jobs[j].event_stop - jobs[j].event_start;
        max_E = std::max(max_E, e + 1);
    }
    // K1: the batch as nph_hmm_score_batch_seq scores it (also its validation of every job)
    NPH_TRY(nph_hmm_score_batch_seq(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, seq_codes, n_codes_total, jobs, n_jobs,
                                    indel_bias, scores_out));
    float kernel_ms = 0.f;
    int launches = 0;
    NPH_TRY(nph_last_kernel_ms(ctx, &kernel_ms, &launches));
    cudaStream_t st = ctx->stream;
    unsigned long long* d_counts; unsigned int* d_flags; uint8_t* d_groups;
    NPH_TRY(nph_carve(ctx, ctx->tt.d_work, [&](NphArena& c) {
        d_counts = c.take<unsigned long long>((size_t)n_groups * kWords);
        d_flags = c.take<unsigned int>(1);
        d_groups = c.take<uint8_t>(groups ? n_jobs : 0);
    }));
    NPH_CUDA(ctx, cudaMemsetAsync(d_counts, 0, sizeof(unsigned long long) * n_groups * kWords, st));
    NPH_CUDA(ctx, cudaMemsetAsync(d_flags, 0, sizeof(unsigned int), st));
    if (groups) NPH_CUDA(ctx, cudaMemcpyAsync(d_groups, groups, n_jobs, cudaMemcpyHostToDevice, st));
    const size_t smem = sizeof(unsigned long long) * n_groups * kWords;
    if (smem > 48 * 1024) NPH_CUDA(ctx, cudaFuncSetAttribute(tt_observe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const TtArgs a{ctx->d_jobs.p, ctx->d_ranks.p, ctx->d_reads.p, ctx->d_models.p, groups ? d_groups : nullptr, n_groups,
                   params->ignore_edge_length, ctx->consts.log_inv_sqrt_2pi, d_counts, d_flags};
    float vit_ms = 0.f, observe_ms = 0.f;
    int vit_launches = 0;
    // the jobs stay where K1 left them: chunk [j0, j0 + nj) is ctx->d_jobs[j0 ..)
    NPH_TRY(nph_viterbi_chunks(ctx, ctx->tt.d_states, n_jobs, params->max_chunk_jobs, 1, max_K, max_E,
        [&](uint64_t j0, uint64_t, uint64_t& first) -> int { first = j0; return NPH_OK; },
        [&](const NphVitChunk& c) -> int {
            const unsigned grid = (unsigned)std::min<uint64_t>((c.n + kWarps - 1) / kWarps, (uint64_t)ctx->sm_count * 4);
            tt_observe_kernel<<<grid, kThreads, smem, st>>>(a, c.j0, c.n, c.states, c.states_off, c.n_states);
            NPH_CUDA(ctx, cudaGetLastError());
            return NPH_OK;
        },
        &vit_ms, &vit_launches, &params->n_chunks_out, &observe_ms));
    params->viterbi_ms_out = vit_ms - observe_ms;
    params->observe_ms_out = observe_ms;
    unsigned int bad = 0;
    NPH_CUDA(ctx, cudaMemcpyAsync(counts_out, d_counts, sizeof(nph_transition_counts) * n_groups, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(&bad, d_flags, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    nph_timing_staged(ctx, kernel_ms + vit_ms, launches + vit_launches);
    if (bad) {
        for (uint32_t g = 0; g < n_groups; ++g) counts_out[g] = nph_transition_counts{};
        ctx->last_error = (bad & kNoPath) ? "profile_hmm_align found no path for a job (the reference asserts)"
                        : (bad & kBadState) ? "a path state other than M, B or K (the reference asserts)"
                        : (bad & kKmerRange) ? "a skip observation past the sequence's k-mers (the reference asserts)"
                        : "a scaled k-mer mean is not finite (the reference's skip bin is undefined)";
        return NPH_ERR_INVALID;
    }
    return NPH_OK;
}
