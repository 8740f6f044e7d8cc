// hmm_schedule.cu — device-side validation, classification and scheduling of forward-HMM jobs.
//
// call-methylation batches hold ~10^6 tiny jobs; doing the per-job bookkeeping on the host cost more
// than scoring them.  Three small kernels replace it: (1) validate each job against its read exactly
// where the reference would assert or read out of bounds (profile_hmm_r9.inl:275, :305), choose its
// kernel class (hmm_classes.h) and histogram (class, step-count) keys; (2) exclusive scan of the histogram,
// a block per class, longest jobs first inside each class; (3) scatter job indices into the schedule.  The host reads
// back one small summary (error flag, per-class counts and costs, scratch sizes).
#include "nph_internal.cuh"
#include "hmm_classes.h"

namespace {

struct SchedSummary {
    int error;                 // 0, or 1 + index of the first offending job (any one of them)
    uint32_t max_kpad, max_period, max_E;
    unsigned long long class_count[NPH_NUM_CLASSES];
    float class_cost[NPH_NUM_CLASSES];
    unsigned long long rank_cursor;   // base-code jobs: k-mer ranks handed out so far (codes_to_ranks_kernel fills them)
};

__global__ void classify_kernel(const nph_hmm_job* __restrict__ jobs, uint32_t n_jobs, const DevRead* __restrict__ reads,
                                uint32_t n_reads, const DevModelView* __restrict__ models, const uint32_t* __restrict__ ranks, const uint8_t* __restrict__ codes,
                                uint32_t n_models, uint64_t n_ranks, uint32_t chunk_events, uint8_t* __restrict__ cls,
                                uint16_t* __restrict__ bkt, unsigned int* __restrict__ hist, SchedSummary* __restrict__ sum,
                                uint64_t* __restrict__ rank_base, int trusted_ranks)
{
    __shared__ unsigned int s_count[NPH_NUM_CLASSES];
    __shared__ float s_cost[NPH_NUM_CLASSES];
    __shared__ unsigned int s_kpad, s_period, s_E;
    for (int i = threadIdx.x; i < NPH_NUM_CLASSES; i += blockDim.x) { s_count[i] = 0; s_cost[i] = 0.f; }
    if (threadIdx.x == 0) { s_kpad = 0; s_period = 0; s_E = 0; }
    __syncthreads();
    // every warp walks whole rounds of 32 jobs (lanes past the end idle) so that the warp-wide votes below see all lanes
    const uint32_t n_round = (n_jobs + 31u) & ~31u;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_round; j += gridDim.x * blockDim.x) {
        const bool have = j < n_jobs;
        const nph_hmm_job jb = have ? jobs[j] : nph_hmm_job{};
        uint32_t chunk = 0;
        bool ok = have && jb.read < n_reads && jb.model_id < n_models && jb.n_kmers != 0 && jb.n_kmers <= n_ranks && jb.rank_off <= n_ranks - jb.n_kmers;   // overflow-safe
        // base-code jobs (nph_hmm_*_seq) read n_kmers + k - 1 codes at rank_off
        const uint32_t seq_len = (ok && codes) ? jb.n_kmers + models[jb.model_id].k - 1u : 0u;
        if (ok && codes) ok = seq_len <= n_ranks && jb.rank_off <= n_ranks - seq_len;
        ok = ok && (jb.stride == 1 || jb.stride == -1);
        if (ok) {
            const DevRead rd = reads[jb.read];
            const uint32_t ne = rd.n_events;
            if (chunk_events) chunk = (uint32_t)((rd.event_off + ne - 1) / chunk_events);
            ok = jb.event_start < ne && jb.event_stop < ne;
            ok = ok && !(jb.event_stop > jb.event_start && jb.stride != 1) && !(jb.event_stop < jb.event_start && jb.stride != -1);
        }
        if (ok && !(trusted_ranks && !codes)) {
            // every k-mer rank must index the job's model table (the reference would read past PoreModel::states); jobs whose ranks
            // a kernel of ours just wrote (call-methylation, variant screening) skip the walk over their ranks
            uint32_t worst = 0;
            if (codes) {                       // every code must be a symbol of the model's alphabet
                const uint8_t* cd = codes + jb.rank_off;
                for (uint32_t i = 0; i < seq_len; ++i) worst = max(worst, (uint32_t)cd[i]);
                ok = worst < models[jb.model_id].alphabet_size;
            } else {
                const uint32_t ns = models[jb.model_id].n_states;
                const uint32_t* rk = ranks + jb.rank_off;
                for (uint32_t i = 0; i < jb.n_kmers; ++i) worst = max(worst, rk[i]);
                ok = worst < ns;
            }
        }
        if (have && !ok) { atomicCAS(&sum->error, 0, (int)(j + 1)); cls[j] = 0; bkt[j] = 0; }
        uint32_t key = 0xffffffffu, steps = 0, K = jb.n_kmers, E = 0;
        int c = 0;
        if (ok) {
            E = (uint32_t)nph_job_events(jb);
            if (codes) rank_base[j] = atomicAdd(&sum->rank_cursor, (unsigned long long)K);     // where this job's ranks will live
            c = nph_choose_class(K, E, &steps);
            const uint32_t b = nph_key_bucket(steps, chunk);
            cls[j] = (uint8_t)c;
            bkt[j] = (uint16_t)b;
            key = (uint32_t)c * NPH_KEY_BUCKETS + b;
        }
        // one atomic per (class, bucket) present in the warp instead of one per job: batches of equal windows (call-methylation,
        // variant screening: millions of jobs on a handful of keys) serialised on those few addresses otherwise
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        const int lane = threadIdx.x & 31;
        const bool leader = lane == __ffs(peers) - 1;
        const int C = c % NPH_MAX_COLS + 1;
        const uint32_t W = nph_class_width(c / NPH_MAX_COLS);
        float cost = ok ? nph_class_cost(steps, C, W) : 0.0f;
        // the class totals: sum the costs of the peers (same key => same class) through the leader
        for (unsigned rest = peers & ~(1u << (__ffs(peers) - 1)); rest; rest &= rest - 1) {
            const float v = __shfl_sync(peers, cost, __ffs(rest) - 1);
            if (leader) cost += v;
        }
        if (ok && leader) {
            atomicAdd(&hist[key], (unsigned int)__popc(peers));
            atomicAdd(&s_count[c], (unsigned int)__popc(peers));
            atomicAdd(&s_cost[c], cost);
        }
        if (ok) {
            const nph_wave_geom geo = nph_wave_geometry((int)K, (int)E, C, (int)W, true);
            atomicMax(&s_kpad, (unsigned int)geo.kpad);
            atomicMax(&s_period, (unsigned int)geo.P);
            atomicMax(&s_E, E);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NPH_NUM_CLASSES; i += blockDim.x) {
        if (s_count[i]) { atomicAdd(&sum->class_count[i], (unsigned long long)s_count[i]); atomicAdd(&sum->class_cost[i], s_cost[i]); }
    }
    if (threadIdx.x == 0) { atomicMax(&sum->max_kpad, s_kpad); atomicMax(&sum->max_period, s_period); atomicMax(&sum->max_E, s_E); }
}

// exclusive scan of the histogram, class-major: one block per class scans its NPH_KEY_BUCKETS buckets and adds the
// class's base (the number of jobs in all earlier classes, from the summary the classify kernel accumulated)
__global__ void __launch_bounds__(1024) scan_kernel(const unsigned int* __restrict__ hist, unsigned int* __restrict__ offs,
                                                    const SchedSummary* __restrict__ sum)
{
    constexpr int T = 1024;
    constexpr int PER = (NPH_KEY_BUCKETS + T - 1) / T;
    __shared__ unsigned int s_warp[32];
    const int c = blockIdx.x, t = threadIdx.x;
    unsigned int base = 0;
    for (int k = 0; k < c; ++k) base += (unsigned int)sum->class_count[k];
    if (sum->class_count[c] == 0) return;                      // nothing to place
    const unsigned int* h = hist + (size_t)c * NPH_KEY_BUCKETS;
    unsigned int* o = offs + (size_t)c * NPH_KEY_BUCKETS;
    const int lo = t * PER, hi = min((int)NPH_KEY_BUCKETS, lo + PER);
    unsigned int s = 0;
    for (int i = lo; i < hi; ++i) s += h[i];
    unsigned int run = base + nph_block_scan_incl(s, s_warp, t) - s;      // exclusive over the 1024 partials
    for (int i = lo; i < hi; ++i) { o[i] = run; run += h[i]; }
}

// Base-code jobs (nph_hmm_*_seq): one warp per job turns the job's codes into its k-mer ranks — k-mer i of the strand's
// string sits at i, or (rc) at length - i - k, HMMInputSequence::get_kmer_rank (nanopolish_hmm_input_sequence.h:60-66) —
// at the slot classify_kernel reserved, then points the device copy of the job at them.  Every kernel after this one
// (forward, Viterbi) reads ranks only.
__global__ void __launch_bounds__(256) codes_to_ranks_kernel(nph_hmm_job* __restrict__ jobs, uint32_t n_jobs, const DevModelView* __restrict__ models,
                                                             const uint8_t* __restrict__ codes, const uint64_t* __restrict__ rank_base,
                                                             uint32_t* __restrict__ ranks)
{
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_jobs; j += warps) {
        const nph_hmm_job jb = jobs[j];
        const uint8_t* __restrict__ cd = codes + jb.rank_off;
        const uint32_t K = jb.n_kmers, mk = models[jb.model_id].k, A = models[jb.model_id].alphabet_size;
        uint32_t* out = ranks + rank_base[j];
        for (uint32_t i = lane; i < K; i += 32) {
            const uint8_t* km = cd + (jb.rc ? K - 1 - i : i);
            uint32_t r = 0;
            for (uint32_t t = 0; t < mk; ++t) r = r * A + km[t];
            out[i] = r;
        }
        __syncwarp();
        if (lane == 0) jobs[j].rank_off = rank_base[j];
    }
}

__global__ void scatter_kernel(uint32_t n_jobs, const uint8_t* __restrict__ cls, const uint16_t* __restrict__ bkt,
                               unsigned int* __restrict__ offs, uint32_t* __restrict__ order)
{
    const uint32_t n_round = (n_jobs + 31u) & ~31u;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_round; j += gridDim.x * blockDim.x) {
        const bool have = j < n_jobs;
        const uint32_t key = have ? (uint32_t)cls[j] * NPH_KEY_BUCKETS + bkt[j] : 0xffffffffu;
        // a slot range per key and warp (one atomic), handed out to the peers in lane order
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        const int lane = threadIdx.x & 31, lead = __ffs(peers) - 1;
        unsigned int base = 0;
        if (have && lane == lead) base = atomicAdd(&offs[key], (unsigned int)__popc(peers));
        base = __shfl_sync(peers, base, lead);
        if (have) order[base + __popc(peers & ((1u << lane) - 1u))] = j;
    }
}

} // namespace

// Runs on ctx->stream after the jobs are on the device.  Fills ctx->classes, max_kpad/max_period, returns
// NPH_ERR_INVALID if any job failed validation.  One stream synchronisation (the summary read-back).
int nph_schedule_hmm_jobs(nph_ctx* ctx, size_t n_jobs, size_t n_ranks_total, NphJobSource src, uint32_t* max_E_out)
{
    const bool codes = src == NphJobSource::HostCodes;
    const size_t hist_n = (size_t)NPH_NUM_CLASSES * NPH_KEY_BUCKETS;
    NPH_TRY(nph_reserve(ctx, ctx->d_sched_cls, n_jobs));
    NPH_TRY(nph_reserve(ctx, ctx->d_sched_bkt, n_jobs));
    if (codes) NPH_TRY(nph_reserve(ctx, ctx->d_rank_base, n_jobs));
    unsigned int* hist; unsigned int* offs; SchedSummary* d_sum;
    auto layout = [&](NphArena& a) {
        hist = a.take<unsigned int>(hist_n);
        offs = a.take<unsigned int>(hist_n);
        d_sum = a.take<SchedSummary>(1);
    };
    const size_t bytes = nph_layout_bytes(layout);           // (before the carve: sizing leaves the pointers null)
    NPH_TRY(nph_carve(ctx, ctx->d_sched_hist, layout));
    NPH_CUDA(ctx, cudaMemsetAsync(hist, 0, bytes, ctx->stream));
    const int threads = 256;
    int blocks = (int)std::min<size_t>((n_jobs + threads - 1) / threads, (size_t)ctx->sm_count * 8);
    if (blocks < 1) blocks = 1;
    classify_kernel<<<blocks, threads, 0, ctx->stream>>>(ctx->d_jobs.p, (uint32_t)n_jobs, ctx->d_reads.p, (uint32_t)ctx->n_reads,
                                                        ctx->d_models.p, ctx->d_ranks.p, codes ? ctx->d_codes.p : nullptr, (uint32_t)ctx->models.size(), (uint64_t)n_ranks_total,
                                                        (uint32_t)(ctx->levels_inflight ? ctx->level_chunk_events : 0), ctx->d_sched_cls.p,
                                                        ctx->d_sched_bkt.p, hist, d_sum, codes ? ctx->d_rank_base.p : nullptr,
                                                        src == NphJobSource::DeviceRanks ? 1 : 0);
    NPH_CUDA(ctx, cudaGetLastError());
    scan_kernel<<<NPH_NUM_CLASSES, 1024, 0, ctx->stream>>>(hist, offs, d_sum);
    NPH_CUDA(ctx, cudaGetLastError());
    SchedSummary h{};
    NPH_CUDA(ctx, cudaMemcpyAsync(&h, d_sum, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    scatter_kernel<<<blocks, threads, 0, ctx->stream>>>((uint32_t)n_jobs, ctx->d_sched_cls.p, ctx->d_sched_bkt.p, offs, ctx->d_order.p);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h.error != 0) {
        ctx->last_error = "job " + std::to_string(h.error - 1) + " fails validation (read/model index, event range, stride, rank range or a k-mer rank outside the model)";
        return NPH_ERR_INVALID;
    }
    if (codes) {
        // the ranks the kernels read: formed here, once, from the codes (the jobs' device copies now index d_ranks)
        NPH_TRY(nph_reserve(ctx, ctx->d_ranks, (size_t)h.rank_cursor));
        const int wblocks = (int)std::min<size_t>((n_jobs + 7) / 8, (size_t)ctx->sm_count * 8);
        codes_to_ranks_kernel<<<wblocks, 256, 0, ctx->stream>>>(ctx->d_jobs.p, (uint32_t)n_jobs, ctx->d_models.p, ctx->d_codes.p, ctx->d_rank_base.p, ctx->d_ranks.p);
        NPH_CUDA(ctx, cudaGetLastError());
    }
    ctx->classes.clear();
    size_t first = 0;
    for (int c = 0; c < NPH_NUM_CLASSES; ++c) {
        ctx->classes.push_back(nph_ctx::ClassLaunch{c % NPH_MAX_COLS + 1, (int)nph_class_width(c / NPH_MAX_COLS), nph_class_chained(c / NPH_MAX_COLS), first,
                                                    (size_t)h.class_count[c], (double)h.class_cost[c]});
        first += (size_t)h.class_count[c];
    }
    ctx->max_kpad = std::max<uint32_t>(h.max_kpad, 32 * NPH_MAX_COLS);
    ctx->max_period = std::max<uint32_t>(h.max_period, NPH_MIN_PERIOD);
    *max_E_out = std::max<uint32_t>(h.max_E, 1);
    return NPH_OK;
}
