// hmm_viterbi.cu — K3: Viterbi alignment of events to the k-mers of a sequence (SURVEY.md section 8f, row N1).
//
// Replaces, for a batch of (sequence, HMMInputData, flags) jobs:
//   profile_hmm_align_r9          ref: src/hmm/nanopolish_profile_hmm_r9.cpp:73-204
//   ProfileHMMViterbiOutputR9     ref: src/hmm/nanopolish_profile_hmm_r9.inl:130-197
//   (the fill itself is profile_hmm_fill_generic_r9, .inl:265-433, shared with the forward score)
//
// The systolic wavefront of hmm_wavefront.cuh, which the forward kernel also walks: a warp per job, lane j owns C
// k-mer columns, strips of 32*C columns chained.  What differs from the forward score is the cell:
//   * (+) is max with the reference's argmax rule — a compare chain over the six movement types in
//     index order where a LATER index wins ties (`from = max == x[i] ? i : from`), so an all -inf cell
//     records FROM_SOFT like the reference does;
//   * each block-cell stores its three 3-bit movement codes (9 bits in a uint16) to a per-warp trace
//     laid out by systolic step, so the 32 lanes of a step write one contiguous line;
//   * the reference keeps the whole float matrix only to report l_fm along the path; we keep no
//     values: after the backtrack the path is replayed forwards, and l_fm of each state is recomputed
//     from its predecessor with the very float operations the fill used (transition + value, + emission),
//     which reproduces the stored matrix entries bit for bit;
//   * the backtrack starts at (last event, MATCH of the last k-mer) and stops at FROM_SOFT, as the
//     reference does; where the reference would trip an assert (fewer than 2 events, path entering a
//     -inf cell) the job returns zero states.
#include "hmm_viterbi_kernel.cuh"
#include <algorithm>
#include <string>
#include <vector>

namespace {

constexpr int kWarps = 16;
constexpr int kThreads = kWarps * 32;
using namespace nph_vit;

struct VitParams {
    const float* level;
    const DevRead* reads;
    const float2* trans;
    const DevModelView* models;
    const uint32_t* ranks;
    const nph_hmm_job* jobs;
    const uint64_t* states_off;      // n_jobs + 1
    const uint32_t* order;           // nullptr: jobs in index order
    uint32_t n_jobs;
    unsigned int* counter;
    const float* flank;
    nph_align_state* states;
    uint32_t* n_states;
    float* scores;
    float4* scratch_params;
    float* scratch_edge;
    uint16_t* scratch_trace;
    uint32_t kpad_stride, edge_stride;
    uint64_t trace_stride;           // uint16 elements per warp
    HmmConsts c;
};

template <int C>
__global__ void __launch_bounds__(kThreads, 1) hmm_viterbi_kernel(const VitParams p)
{
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * kWarps + (threadIdx.x >> 5);
    __shared__ uint16_t s_tile[kWarps][32 * 32];
    VitScratch sc;
    sc.tile = s_tile[threadIdx.x >> 5];
    sc.params = warp_params(p.scratch_params, p.kpad_stride, warp_global);
    sc.edge = warp_edge_rows(p.scratch_edge, p.edge_stride, warp_global);
    sc.trace = p.scratch_trace + (size_t)warp_global * p.trace_stride;
    const float NEG = -CUDART_INF_F;

    for (;;) {
        const uint32_t slot = nph_warp_pop(p.counter, 1u, lane);
        if (slot >= p.n_jobs) break;
        const uint32_t job_idx = p.order ? p.order[slot] : slot;
        const nph_hmm_job job = p.jobs[job_idx];
        VitJob j;
        j.rd = p.reads[job.read];
        j.tr = p.trans[job.read];
        j.mv = p.models[job.model_id];
        j.lv = p.level + j.rd.event_off;
        j.rk = p.ranks + job.rank_off;
        j.K = (int)job.n_kmers;
        j.E = nph_job_events(job);
        j.stride = job.stride;
        j.e_first = (long long)job.event_start;
        j.pre_clip = (job.flags & NPH_HAF_ALLOW_PRE_CLIP) != 0;
        nph_align_state* const out = p.states + p.states_off[job_idx];
        const int cap = (int)(p.states_off[job_idx + 1] - p.states_off[job_idx]);

        if (j.E < 2) {                   // the reference asserts n_events >= 2 (profile_hmm_r9.cpp:88)
            if (lane == 0) { p.n_states[job_idx] = 0; if (p.scores) p.scores[job_idx] = NEG; }
            continue;
        }
        float last_v = NEG;
        const int n = viterbi_align<C>(p.c, p.flank, j, sc, out, cap, &last_v, lane);
        if (lane == 0) {
            p.n_states[job_idx] = (uint32_t)n;
            if (p.scores) p.scores[job_idx] = n ? last_v : NEG;
        }
        __syncwarp();
    }
}

template <int C>
int launch_vit(nph_ctx* ctx, const VitParams& base, const uint32_t* order, size_t count, unsigned int* counter, int max_ctas)
{
    VitParams p = base;
    p.order = order; p.n_jobs = (uint32_t)count; p.counter = counter;
    int grid = std::min(ctx->sm_count, max_ctas);
    if ((size_t)grid * kWarps > count) grid = (int)((count + kWarps - 1) / kWarps);
    if (grid < 1) grid = 1;
    hmm_viterbi_kernel<C><<<grid, kThreads, 0, ctx->stream>>>(p);
    NPH_CUDA(ctx, cudaGetLastError());
    return NPH_OK;
}

const int kVitCols[] = {1, 2, 3, 4, 6, 8};
const int kNumVit = 6;
const uint64_t kTraceBudget = 16ull << 30;

int launch_vit_class(nph_ctx* ctx, int cols, const VitParams& p, const uint32_t* order, size_t count, unsigned int* counter, int max_ctas)
{
    switch (cols) {
        case 1: return launch_vit<1>(ctx, p, order, count, counter, max_ctas);
        case 2: return launch_vit<2>(ctx, p, order, count, counter, max_ctas);
        case 3: return launch_vit<3>(ctx, p, order, count, counter, max_ctas);
        case 4: return launch_vit<4>(ctx, p, order, count, counter, max_ctas);
        case 6: return launch_vit<6>(ctx, p, order, count, counter, max_ctas);
        case 8: return launch_vit<8>(ctx, p, order, count, counter, max_ctas);
    }
    return NPH_ERR_STATE;
}

// the cheapest class for a K x E job and its geometry
int vit_class(uint32_t K, uint32_t E, nph_wave_geom& geo, uint32_t& steps)
{
    double best = 1e300; int bi = 0;
    for (int i = 0; i < kNumVit; ++i) {
        const nph_wave_geom g = nph_wave_geometry((int)K, (int)E, kVitCols[i], 32, true);
        const double cost = (double)g.total_steps() * (120.0 + 70.0 * kVitCols[i]);
        if (cost < best) { best = cost; bi = i; steps = (uint32_t)g.total_steps(); geo = g; }
    }
    return bi;
}

// CTAs whose movement traces fit kTraceBudget, or NPH_ERR_UNSUPPORTED when not even one CTA's do
int vit_max_ctas(nph_ctx* ctx, size_t trace_stride, int& max_ctas)
{
    const uint64_t per_cta = (uint64_t)sizeof(uint16_t) * trace_stride * kWarps;
    if (per_cta > kTraceBudget) {
        ctx->last_error = "profile_hmm_align window too large: its movement trace needs " + std::to_string(per_cta >> 20) + " MiB per CTA (limit 16 GiB)";
        return NPH_ERR_UNSUPPORTED;
    }
    max_ctas = (int)std::min<uint64_t>((uint64_t)ctx->sm_count, std::max<uint64_t>(1, kTraceBudget / per_cta));
    return NPH_OK;
}

// off[i] = i * stride, i = 0 .. n
__global__ void states_off_kernel(uint64_t* __restrict__ off, uint64_t n, uint64_t stride)
{
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i <= n) off[i] = i * stride;
}

// device memory for the Viterbi states of one chunk of nph_viterbi_chunks (16 B per state, max_K + max_E states per job)
constexpr uint64_t kStatesBudget = 1ull << 30;

} // namespace

int nph_viterbi_chunks(nph_ctx* ctx, DevBuf<uint8_t>& buf, uint64_t n_jobs, uint64_t max_chunk, uint64_t unit, uint32_t max_K, uint32_t max_E,
                       const std::function<int(uint64_t j0, uint64_t nj, uint64_t& first)>& prepare,
                       const std::function<int(const NphVitChunk&)>& fold, float* ms, int* launches, uint32_t* n_chunks,
                       float* fold_ms)
{
    const uint64_t stride = (uint64_t)max_K + max_E;
    uint64_t chunk = std::min<uint64_t>(max_chunk ? max_chunk : UINT64_MAX, kStatesBudget / (sizeof(nph_align_state) * stride));
    chunk = std::max<uint64_t>(unit, chunk / unit * unit);
    cudaStream_t st = ctx->stream;
    *ms = 0.f; *launches = 0; *n_chunks = 0;
    if (fold_ms) *fold_ms = 0.f;
    for (uint64_t j0 = 0; j0 < n_jobs; j0 += chunk) {
        const uint64_t nj = std::min(chunk, n_jobs - j0);
        uint64_t* d_off; uint32_t* d_n; nph_align_state* d_states;
        NPH_TRY(nph_carve(ctx, buf, [&](NphArena& c) {
            d_off = c.take<uint64_t>(nj + 1);
            d_n = c.take<uint32_t>(nj);
            d_states = c.take<nph_align_state>(nj * stride);
        }));
        uint64_t first = 0;
        NPH_TRY(prepare(j0, nj, first));
        NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
        states_off_kernel<<<(unsigned)((nj + 1 + 255) / 256), 256, 0, st>>>(d_off, nj, stride);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_viterbi_device_jobs(ctx, (size_t)nj, max_K, max_E, d_off, d_states, d_n, (size_t)first));
        NPH_CUDA(ctx, cudaEventRecord(ctx->ev_mid, st));
        NPH_TRY(fold(NphVitChunk{j0, nj, d_states, d_off, d_n}));
        NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
        NPH_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
        float t = 0.f, f = 0.f;
        NPH_CUDA(ctx, cudaEventElapsedTime(&t, ctx->ev0, ctx->ev1));
        NPH_CUDA(ctx, cudaEventElapsedTime(&f, ctx->ev_mid, ctx->ev1));
        *ms += t; *launches += 3; *n_chunks += 1;
        if (fold_ms) *fold_ms += f;
    }
    return NPH_OK;
}

int nph_viterbi_device_jobs(nph_ctx* ctx, size_t n_jobs, uint32_t max_K, uint32_t max_E, const uint64_t* d_states_off,
                            nph_align_state* d_states, uint32_t* d_n_states, size_t first_job)
{
    if (n_jobs == 0) return NPH_OK;
    // one class for the whole batch, chosen for its largest job, and no host pass over the jobs.  Homopolymer calling windows all
    // have one shape, so a per-job choice would differ little there; scorereads segments of 500 events vary in K (a long deletion
    // makes one segment's sequence longer), and one outlier then sets the class, the trace size and, in nph_viterbi_chunks, the
    // state stride of every job of the chunk (a cost not measured: the benchmark's segments are uniform)
    nph_wave_geom geo{};
    uint32_t steps = 0;
    const int ci = vit_class(max_K, max_E, geo, steps);
    const size_t trace_stride = (((uint64_t)(steps + 1) * geo.strip + 63) / 64) * 64;
    int max_ctas = 0;
    NPH_TRY(vit_max_ctas(ctx, trace_stride, max_ctas));
    const int warps = max_ctas * kWarps;
    const uint32_t kpad = std::max<uint32_t>(32, (uint32_t)geo.kpad), period = std::max<uint32_t>(NPH_MIN_PERIOD, (uint32_t)geo.P);
    VitParams p{};
    NPH_TRY(nph_carve_align_scratch(ctx, [&](NphArena& a) {
        nph_wave_scratch(a, kpad, period, warps, &p.scratch_params, &p.scratch_edge);
        p.scratch_trace = a.take<uint16_t>(trace_stride * warps);
    }));
    p.states_off = d_states_off; p.states = d_states; p.n_states = d_n_states; p.scores = nullptr;
    p.level = ctx->d_level.p; p.reads = ctx->d_reads.p; p.trans = ctx->d_trans.p; p.models = ctx->d_models.p;
    p.ranks = ctx->d_ranks.p; p.jobs = ctx->d_jobs.p + first_job; p.flank = ctx->d_flank.p;
    p.kpad_stride = kpad; p.edge_stride = nph_edge_stride(period); p.trace_stride = trace_stride; p.c = ctx->consts;
    NPH_CUDA(ctx, cudaMemsetAsync(ctx->d_counters.p, 0, sizeof(unsigned int), ctx->stream));
    return launch_vit_class(ctx, kVitCols[ci], p, nullptr, n_jobs, ctx->d_counters.p, max_ctas);
}

extern "C" int nph_hmm_align_batch(nph_ctx* ctx,
                                   const nph_read* reads, size_t n_reads,
                                   const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                   const uint32_t* kmer_ranks, size_t n_ranks_total,
                                   const nph_hmm_job* jobs, size_t n_jobs, double indel_bias,
                                   nph_align_state* states_out, const uint64_t* states_off,
                                   uint32_t* n_states_out, float* scores_out)
{
    if (!ctx || !jobs || !states_out || !states_off || !n_states_out || n_jobs == 0) return NPH_ERR_INVALID;
    NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
    return nph_hmm_align(ctx, kmer_ranks, n_ranks_total, jobs, n_jobs, indel_bias, states_out, states_off, n_states_out, scores_out);
}

extern "C" int nph_hmm_align(nph_ctx* ctx,
                             const uint32_t* kmer_ranks, size_t n_ranks_total,
                             const nph_hmm_job* jobs, size_t n_jobs, double indel_bias,
                             nph_align_state* states_out, const uint64_t* states_off,
                             uint32_t* n_states_out, float* scores_out)
{
    if (!ctx || !jobs || !states_out || !states_off || !n_states_out || n_jobs == 0) return NPH_ERR_INVALID;
    if (!ctx->reads_loaded) return NPH_ERR_STATE;
    // jobs, ranks, transitions and validation go through the forward path's loader (same job semantics)
    NPH_TRY(nph_hmm_jobs_load(ctx, kmer_ranks, n_ranks_total, jobs, n_jobs, indel_bias));

    // class per job (columns per lane) and schedule: class by class, longest first inside each
    std::vector<uint64_t> key(n_jobs);
    size_t first[kNumVit + 1] = {};
    uint32_t max_kpad = 32, max_period = NPH_MIN_PERIOD;
    uint64_t max_trace = 1;
    for (size_t j = 0; j < n_jobs; ++j) {
        const nph_hmm_job& jb = jobs[j];
        if (states_off[j + 1] < states_off[j]) return NPH_ERR_INVALID;
        uint32_t bsteps = 0;
        nph_wave_geom geo{};
        const int bi = vit_class(jb.n_kmers, (uint32_t)nph_job_events(jb), geo, bsteps);
        key[j] = (uint64_t)(kNumVit - 1 - bi) << 32 | bsteps;
        ++first[bi + 1];
        max_kpad = std::max(max_kpad, (uint32_t)geo.kpad);
        max_period = std::max(max_period, (uint32_t)geo.P);
        max_trace = std::max<uint64_t>(max_trace, (uint64_t)(bsteps + 1) * geo.strip);
    }
    const std::vector<uint32_t> order = nph_longest_first(key);
    for (int i = 0; i < kNumVit; ++i) first[i + 1] += first[i];

    // The movement trace is per resident warp and sized by the batch's largest job ((steps + 1) x strip uint16 entries),
    // so one long window must not multiply by every warp of the chip: the number of resident CTAs is capped so that
    // the trace arena stays within kTraceBudget, and a job whose trace does not fit a single CTA's 16 warps within
    // that budget is refused with NPH_ERR_UNSUPPORTED (documented in include/nph.h) instead of a NOMEM surprise.
    const size_t trace_stride = ((max_trace + 63) / 64) * 64;
    int max_ctas = 0;
    NPH_TRY(vit_max_ctas(ctx, trace_stride, max_ctas));
    const int warps = max_ctas * kWarps;
    const size_t total_states = (size_t)states_off[n_jobs];
    VitParams p{};
    uint64_t* d_off = nullptr;
    uint32_t* d_order = nullptr;
    NPH_TRY(nph_carve_align_scratch(ctx, [&](NphArena& a) {
        nph_wave_scratch(a, max_kpad, max_period, warps, &p.scratch_params, &p.scratch_edge);
        p.scratch_trace = a.take<uint16_t>(trace_stride * warps);
        p.states = a.take<nph_align_state>(total_states);
        d_off = a.take<uint64_t>(n_jobs + 1);
        p.n_states = a.take<uint32_t>(n_jobs);
        d_order = a.take<uint32_t>(n_jobs);
    }));
    p.states_off = d_off;
    p.level = ctx->d_level.p; p.reads = ctx->d_reads.p; p.trans = ctx->d_trans.p; p.models = ctx->d_models.p;
    p.ranks = ctx->d_ranks.p; p.jobs = ctx->d_jobs.p; p.flank = ctx->d_flank.p; p.scores = ctx->d_scores.p;
    p.kpad_stride = max_kpad; p.edge_stride = nph_edge_stride(max_period); p.trace_stride = trace_stride; p.c = ctx->consts;
    NPH_CUDA(ctx, cudaMemcpyAsync(d_off, states_off, sizeof(uint64_t) * (n_jobs + 1), cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_order, order.data(), sizeof(uint32_t) * n_jobs, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemsetAsync(ctx->d_counters.p, 0, sizeof(unsigned int) * NPH_NUM_COUNTERS, ctx->stream));
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    int launches = 0;
    for (int i = 0; i < kNumVit; ++i) {
        const size_t count = first[i + 1] - first[i];
        if (!count) continue;
        NPH_TRY(launch_vit_class(ctx, kVitCols[i], p, d_order + first[i], count, ctx->d_counters.p + i, max_ctas));
        ++launches;
    }
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    nph_timing_events(ctx, launches);
    // only the jobs' slices go back: states_out[0 .. states_off[0]) belongs to the caller
    NPH_CUDA(ctx, cudaMemcpyAsync(states_out + states_off[0], p.states + states_off[0], sizeof(nph_align_state) * (total_states - states_off[0]),
                                  cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(n_states_out, p.n_states, sizeof(uint32_t) * n_jobs, cudaMemcpyDeviceToHost, ctx->stream));
    if (scores_out) NPH_CUDA(ctx, cudaMemcpyAsync(scores_out, ctx->d_scores.p, sizeof(float) * n_jobs, cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return NPH_OK;
}
