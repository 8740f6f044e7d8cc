// nph_internal.cuh — shared declarations of libnph.so (not installed; the public surface is include/nph.h)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string>
#include <vector>
#include <algorithm>
#include <functional>
#include <utility>
#include "../../include/nph.h"

#define NPH_LOGSUM_TBL 16000        // ref: p7_LOGSUM_TBL, src/common/logsum.h:20
#define NPH_TBL_SMEM   16385        // = NPH_LOGSUM_TBL_LEN: the saturated index of lsum_sat (exact_math.cuh) reaches 2^14
#define NPH_NUM_COUNTERS 64          // work-queue counters: one per forward class (<= 40), nph_check_ranks' flag, ABEA (last)

// Per-read record on the device (what the kernels need of nph_read after the prologue).
struct DevRead {
    uint64_t event_off;
    uint32_t n_events;
    uint32_t pad;
    double scale, shift, var, log_var;
};

// The eight read-independent transition log-probabilities + Gaussian constant, computed on the host
// with libm exactly as the reference does (logf of float probabilities).
struct HmmConsts {
    float lp_mk, lp_mb, lp_bb, lp_bk, lp_bm_next, lp_bm_self, lp_kk, lp_km;
    float log_inv_sqrt_2pi;
};

// Device-side view of the models for kernels (array of pointers)
struct DevModelView { const double* mean; const double* stdv; const double* log_stdv; uint32_t n_states; uint16_t k; uint16_t alphabet_size; };

// Device memory that frees itself: move-only, released when the owner (the context, a model) goes away.
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;   // elements
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
};

// Page-locked host memory that frees itself.
template <typename T>
struct PinnedBuf {
    T* p = nullptr;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
};

struct DevModel {
    DevBuf<double> mean, stdv, log_stdv;
    uint32_t n_states = 0, k = 0, alphabet_size = 0;
};

// The event-aligned records of a call-methylation or screening batch: reference bytes, each record's event alignment as a pair
// list or in compact form, the records.  Each record's [ref_off, ref_off + ref_len) indexes the n_map bases of the event map.
struct NphEventRecords {
    size_t n_records = 0, n_ref = 0, n_map = 0;
    bool compact = false;                  // int16 deltas per base + first_event per record, expanded by nph_event_records_expand
    DevBuf<uint8_t> d_ref;
    DevBuf<nph_aligned_pair> d_pairs;      // pair form
    DevBuf<uint16_t> d_deltas;             // compact form: n_map int16 deltas
    DevBuf<uint8_t> d_dense;               // compact form: event index per base, first_event and first valid base per record
    DevBuf<nph_meth_record> d_records;
};

struct nph_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 0;
    std::string last_error;

    // constant tables
    DevBuf<float> d_logsum;          // NPH_TBL_SMEM floats
    DevBuf<float> d_flank;           // clip-penalty table, grown on demand
    std::vector<float> h_flank;
    HmmConsts consts;

    // models
    std::vector<DevModel> models;
    DevBuf<DevModelView> d_models;

    // resident reads
    size_t n_reads = 0, n_events_total = 0;
    DevBuf<DevRead> d_reads;
    DevBuf<float> d_ev_mean;
    DevBuf<double> d_ev_time;
    DevBuf<float> d_level;           // drift-scaled levels
    DevBuf<double> d_drift;          // per read SquiggleScalings::drift (consumed by the read prologue)
    std::vector<double> h_events_per_base;
    std::vector<uint32_t> h_read_n_events;
    bool reads_loaded = false;

    // resident HMM jobs
    size_t n_jobs = 0, n_ranks = 0;
    DevBuf<uint32_t> d_ranks;
    DevBuf<uint8_t> d_codes;         // jobs loaded through the *_seq calls: base codes instead of k-mer ranks (jobs' rank_off index this)
    DevBuf<uint64_t> d_rank_base;    // base-code jobs: where each job's ranks start in d_ranks (hmm_schedule.cu)
    DevBuf<nph_hmm_job> d_jobs;
    DevBuf<float2> d_trans;          // per read: (lp_mm_self, lp_mm_next)
    DevBuf<uint32_t> d_order;        // job indices grouped by kernel class, heavy first
    DevBuf<float> d_scores;
    DevBuf<unsigned int> d_counters;
    DevBuf<uint8_t> d_sched_cls;     // per job: kernel class
    DevBuf<uint16_t> d_sched_bkt;    // per job: schedule key bucket
    DevBuf<uint8_t> d_sched_hist;    // histogram, offsets, summary (hmm_schedule.cu)
    DevBuf<uint8_t> d_scratch;
    struct ClassLaunch { int cols_per_lane; int group_width; bool chained; size_t first; size_t count; double cost; };
    std::vector<ClassLaunch> classes;
    uint32_t max_kpad = 0, max_period = 0;
    bool jobs_loaded = false;

    // resident ABEA jobs
    size_t n_abea_jobs = 0, abea_pairs_total = 0;
    uint32_t abea_model = 0;
    DevBuf<nph_abea_job> d_abea_jobs;
    DevBuf<uint32_t> d_abea_ranks;
    DevBuf<nph_aligned_pair> d_pairs;
    DevBuf<nph_abea_result> d_abea_res;
    DevBuf<uint8_t> d_align_scratch; // ABEA's band trace, and the scratch of every other alignment-prologue call (nph_carve_align_scratch)
    DevBuf<uint32_t> d_abea_order;
    DevBuf<double> d_abea_consts;    // per job (lp_stay, lp_step); also the MoM output buffer
    DevBuf<uint8_t> d_prep;          // load_from_raw: event SoA staging, MoM output, calibration buffers
    uint32_t abea_kmax = 0;
    uint64_t abea_trace_stride = 0;
    bool abea_loaded = false;

    // the records of the last nph_eventalign_chain_run, where the kernel wrote them in d_align_scratch (eventalign_chain.cu), and
    // the buffers of nph_eventalign_tsv (eventalign_tsv.cu)
    struct EaState {
        bool resident = false;             // dropped by nph_carve_align_scratch, nph_abea_stage and nph_reads_resident
        size_t records_total = 0, n_ranks = 0;
        const nph_ea_chain* d_chains = nullptr;
        const nph_ea_record* d_records = nullptr;
        const nph_ea_result* d_results = nullptr;
        const uint32_t* d_ranks_fwd = nullptr;
        const uint32_t* d_ranks_rc = nullptr;
        std::vector<nph_ea_chain> h_chains;
        std::vector<nph_ea_result> h_results;
        DevBuf<uint8_t> d_tsv_in;          // names, reference characters, event and sample arrays, per-read and per-chain tables
        DevBuf<uint8_t> d_tsv_off;         // bytes of each row, their exclusive prefix, the refusal flags
        DevBuf<uint8_t> d_tsv;             // the rows
    } ea;

    // resident call-methylation batch (methylation.cu)
    struct MethState {
        bool loaded = false, ran = false;
        size_t prov_total = 0;
        nph_meth_params params{};
        double indel_bias = 1.0;
        uint64_t n_sites = 0, n_ranks = 0, n_scored_events = 0;
        NphEventRecords ev;                // pair lists (nph_methylation_load) or compact form (nph_methylation_load_compact)
        DevBuf<uint64_t> d_prov_off;       // n_records + 1: where each record's provisional group rows start
        DevBuf<uint8_t> d_prov;            // provisional group rows (MethGroup)
        DevBuf<uint8_t> d_counts;          // meth_counts_layout: per-record groups and ranks, their offsets, the summary
        DevBuf<nph_meth_site> d_sites;
        DevBuf<uint8_t> d_tsv_in;          // nph_methylation_tsv: contig, read names, name offsets, strand flags
        DevBuf<uint8_t> d_tsv_off;         // bytes of each record's rows, their exclusive prefix, the refusal flag
        DevBuf<uint8_t> d_tsv;             // the rows
        std::vector<uint64_t> h_prov_off;
    } meth;

    // per-site methylation frequency accumulated over call-methylation batches (meth_frequency.cu)
    struct FreqState {
        nph_methfreq_params params{2.0, 0, 0};
        size_t slots = 0;                  // hash table slots, a power of two (0: no accumulator yet)
        uint32_t n_batches = 0;            // folds so far: the batch part of the first-row ordinals
        uint64_t n_calls = 0, n_ambiguous = 0;
        DevBuf<uint8_t> d_summary;         // the accumulator's key and pool counters, the fold's batch counts
        DevBuf<uint8_t> d_table;           // keys, first-row ordinals, called, methylated, sequence offsets, group info per slot
        DevBuf<uint8_t> d_pool;            // sequence bytes of the keys' first rows
        DevBuf<uint8_t> d_work;            // nph_methfreq_tsv: names, ranks, compaction, sort and row offsets
        DevBuf<uint8_t> d_out;             // nph_methfreq_tsv: the rows
    } freq;

    // resident variant-screening batch (variants.cu)
    struct ScreenState {
        bool loaded = false, ran = false;
        nph_screen_params params{};
        double indel_bias = 1.0;
        size_t n_pos = 0;
        uint32_t n_rounds = 0;
        uint64_t n_jobs = 0, n_scored_events = 0, n_jobs_no_exit = 0, n_reference_events = 0;
        NphEventRecords ev;                // region reference, compact event alignments over n_map bases
        DevBuf<uint64_t> d_pos_off;        // n_pos + 1: where each position's bounded reads start
        DevBuf<uint8_t> d_pos_reads;       // {record, e1, e2} per bounded read
        DevBuf<uint8_t> d_state;           // screen_state_layout: per-position state, counters, methylated-alternatives masks
        DevBuf<uint8_t> d_job_off;         // per position: job count and first job of the round, scan scratch
        uint32_t n_types = 0;              // methylation types (nph_screen_load_methylation)
        std::vector<uint8_t> h_meth;       // their MethDev tables (meth_dev.cuh), the source of d_meth's upload
        DevBuf<uint8_t> d_meth;
        DevBuf<uint32_t> d_alt_models;     // n_records x n_types model ids
    } screen;

    // the last nph_phase_reads_batch (phase_reads.cu)
    struct PhaseState {
        NphEventRecords ev;                // fetched references, compact event alignments, records
        DevBuf<uint8_t> d_in;              // variants and per-record variant ranges
        DevBuf<uint8_t> d_counts;          // per-record sites, their offsets, the scan's scratch, the scored-event count
        DevBuf<nph_phase_call> d_calls;
    } phase;

    // the batch of the last one-shot region call (nph_homopolymer_likelihoods_batch, nph_all_support_batch,
    // nph_screen_variants_batch, nph_call_variant_groups_batch; window_reads.cu).  None of them is staged, so each may take over
    // what the one before it left.
    struct RegionState {
        NphEventRecords ev;                // region reference, compact event alignments, records
        DevBuf<uint8_t> d_counts;          // the windows' bounds, per-window counts, pair offsets, the scan's scratch, the largest rows
        DevBuf<uint8_t> d_pairs;           // the windows' pairs and the window of each
    } region;

    // the last nph_homopolymer_likelihoods_batch (homopolymer.cu)
    struct HpState {
        DevBuf<uint8_t> d_in;              // windows, calling sequences, event durations
        DevBuf<uint8_t> d_jobs;            // per job the forward score and sum_duration, the no-path flag
        DevBuf<uint8_t> d_states;          // one chunk's state offsets, state counts and Viterbi states
    } hp;

    // the last nph_all_support_batch (all_support.cu)
    struct SupportState {
        DevBuf<uint8_t> d_jobs;            // per variant its window, per job the difference score - log-sum
    } sup;

    // the last nph_screen_variants_batch (screen_variants.cu)
    struct ScreenListState {
        DevBuf<uint8_t> d_in;              // windows, sequences, the window's candidates, alleles, methylation tables and model ids
        DevBuf<uint8_t> d_state;           // per-window round state, job counts and offsets, scan scratch, per-candidate state,
                                           // methylated-alternative masks, counters
    } sl;

    // the last nph_call_variant_groups_batch (call_variants.cu)
    struct CallState {
        DevBuf<uint8_t> d_in;              // groups, haplotypes, their bases and variant ids, key ranks, methylation tables and model ids
        DevBuf<uint8_t> d_work;            // per-group offsets, masks, pair scores, key tables, partial maxima, group results
    } call;

    // the last nph_train_transitions_batch (transitions.cu)
    struct TtState {
        DevBuf<uint8_t> d_work;            // the group records, the refusal flags, the jobs' groups
        DevBuf<uint8_t> d_states;          // one chunk's state offsets, state counts and Viterbi states
    } tt;

    // measurement
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_mid = nullptr;    // nph_viterbi_chunks: between K3 and the fold of a chunk
    // side streams so that the tail of one forward class overlaps the head of the next (fork/join by events)
    static const int kSideStreams = 4;
    cudaStream_t side[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[4] = {nullptr, nullptr, nullptr, nullptr};
    int last_launches = 0;
    enum class Timing { None, Events, Staged } timing = Timing::None;   // set by nph_timing_events / nph_timing_staged
    float staged_ms = 0.0f;

    // pipelined level upload of the one-shot call: copy stream, progress word polled by the forward kernel
    static const int kLevelChunks = 8;
    cudaStream_t cstream = nullptr;
    cudaEvent_t ev_reset = nullptr;
    DevBuf<uint32_t> d_progress;             // number of level chunks that have landed
    PinnedBuf<uint32_t> h_progress_vals;     // {1, 2, ...}: sources of the progress writes
    size_t level_chunk_events = 0;           // 0 = levels fully resident, kernels do not poll
    bool levels_inflight = false;
    std::vector<DevRead> h_stage_reads;      // host staging that must outlive async copies
    std::vector<double> h_stage_drift;
    std::vector<float2> h_stage_trans;
    std::vector<nph_raw_range> h_last_trim;  // surviving sample range per job of the last nph_load_from_raw_batch

    DevBuf<uint8_t> d_polya;                 // nph_polya_batch / nph_detect_polyi_batch: raw samples, durations, event map, jobs, order, results
};

int nph_set_cuda_error(nph_ctx* ctx, cudaError_t e, const char* what);
#define NPH_CUDA(ctx, call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return nph_set_cuda_error((ctx), e__, #call); } while (0)
#define NPH_TRY(expr) do { int rc__ = (expr); if (rc__ != NPH_OK) return rc__; } while (0)

// Grows b to hold at least n elements (with room for n / 8 + 16 more); the old contents are not kept, and the old
// allocation is freed before the new one is made.
template <typename T>
int nph_reserve(nph_ctx* ctx, DevBuf<T>& b, size_t n)
{
    if (n <= b.cap && b.p) return NPH_OK;
    if (b.p) { NPH_CUDA(ctx, cudaFree(b.p)); b.p = nullptr; b.cap = 0; }
    const size_t want = n + n / 8 + 16;
    NPH_CUDA(ctx, cudaMalloc((void**)&b.p, want * sizeof(T)));
    b.cap = want;
    return NPH_OK;
}

// One scratch layout.  A layout function lists every slice once, in order, through take(); run over an arena without a
// base it only adds up the bytes, run over a reserved buffer it hands out the pointers.  Every slice starts on 256 bytes.
struct NphArena {
    uint8_t* base = nullptr;
    size_t used = 0;
    template <typename T> T* take(size_t n)
    {
        T* q = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += (sizeof(T) * n + 255) / 256 * 256;
        return q;
    }
};
template <typename Layout>
size_t nph_layout_bytes(Layout&& layout) { NphArena a; layout(a); return a.used; }
// reserve buf for the layout, then carve it
template <typename Layout>
int nph_carve(nph_ctx* ctx, DevBuf<uint8_t>& buf, Layout&& layout)
{
    NPH_TRY(nph_reserve(ctx, buf, nph_layout_bytes(layout)));
    NphArena a{buf.p};
    layout(a);
    return NPH_OK;
}
// Carve the alignment scratch for a call other than ABEA: the staged ABEA batch keeps its band trace there and an eventalign
// chain run its records, so both are dropped.
template <typename Layout>
int nph_carve_align_scratch(nph_ctx* ctx, Layout&& layout)
{
    ctx->abea_loaded = false;
    ctx->ea.resident = false;
    return nph_carve(ctx, ctx->d_align_scratch, layout);
}

// off + len <= total, in a form that cannot wrap
inline bool nph_slice_ok(uint64_t off, uint64_t len, uint64_t total) { return len <= total && off <= total - len; }
// A job's k-mers: at least one, with ranks [rank_off, rank_off + n_kmers) inside the call's n_ranks
inline bool nph_kmers_ok(uint64_t rank_off, uint32_t n_kmers, uint64_t n_ranks) { return n_kmers > 0 && nph_slice_ok(rank_off, n_kmers, n_ranks); }
// An ABEA-shaped job (ABEA, MoM, calibration): its read is one of the call's n_reads, its k-mers are nph_kmers_ok and its
// n_pairs pairs from pairs_off lie inside pairs_total (the defaults: a call without pairs).  The ranks themselves are checked
// on the device by nph_check_ranks.
inline bool nph_abea_job_ok(const nph_abea_job& jb, size_t n_reads, uint64_t n_ranks, uint64_t n_pairs = 0, uint64_t pairs_total = UINT64_MAX)
{ return jb.read < n_reads && nph_kmers_ok(jb.rank_off, jb.n_kmers, n_ranks) && nph_slice_ok(jb.pairs_off, n_pairs, pairs_total); }
// No two jobs share a k-mer rank: [rank_off, rank_off + n_kmers) of the jobs are pairwise disjoint.  The calibration builds each
// job's base_to_event map in place at its rank_off (a warp per job, with atomics over its own pair indices), so jobs that share
// ranks would mix two jobs' pair lists; nph_recalibrate_batch and nph_load_from_raw_batch refuse them.  ABEA and MoM only read
// the ranks and take shared ranges.
template <typename Job>
bool nph_rank_ranges_disjoint(const Job* jobs, size_t n_jobs)
{
    size_t j = 1;                       // jobs laid out in rank order (the usual batch) need one pass and no copy
    while (j < n_jobs && jobs[j].rank_off >= jobs[j - 1].rank_off + jobs[j - 1].n_kmers) ++j;
    if (j >= n_jobs) return true;
    std::vector<std::pair<uint64_t, uint64_t>> r(n_jobs);
    for (size_t i = 0; i < n_jobs; ++i) r[i] = {jobs[i].rank_off, jobs[i].rank_off + jobs[i].n_kmers};
    std::sort(r.begin(), r.end());
    for (size_t i = 1; i < n_jobs; ++i)
        if (r[i].first < r[i - 1].second) return false;
    return true;
}

// Indices 0 .. n-1 by key, largest first; equal keys keep index order.
template <typename K>
std::vector<uint32_t> nph_longest_first(const std::vector<K>& key)
{
    std::vector<uint32_t> order(key.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = (uint32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] > key[b]; });
    return order;
}

// What nph_last_kernel_ms reports: the time between ctx->ev0 and ctx->ev1, or the summed device time of a call with host
// round trips between its kernels.
inline void nph_timing_events(nph_ctx* ctx, int launches) { ctx->last_launches = launches; ctx->timing = nph_ctx::Timing::Events; }
inline void nph_timing_staged(nph_ctx* ctx, float ms, int launches)
{
    ctx->staged_ms = ms; ctx->last_launches = launches; ctx->timing = nph_ctx::Timing::Staged;
}

// A new read batch is resident: the HMM and ABEA jobs and the eventalign records of the previous one no longer apply.
inline void nph_reads_resident(nph_ctx* ctx) { ctx->reads_loaded = true; ctx->jobs_loaded = false; ctx->abea_loaded = false; ctx->ea.resident = false; }

#ifdef __CUDACC__
// get_scaled_gaussian_from_pore_model_state (ref: src/nanopolish_squiggle_read.h:217-226) of k-mer rank r, formed in FP64 and
// narrowed: {mu', sigma', log(1/sqrt(2pi)) - log sigma', RN(1/sigma')}
__device__ __forceinline__ float4 nph_scaled_gaussian(const DevModelView& mv, const DevRead& rd, uint32_t r, float log_inv_sqrt_2pi)
{
    const float mu = (float)__dadd_rn(__dmul_rn(rd.scale, mv.mean[r]), rd.shift);
    const float sd = (float)__dmul_rn(mv.stdv[r], rd.var);
    const float lsd = (float)__dadd_rn(mv.log_stdv[r], rd.log_var);
    return make_float4(mu, sd, __fsub_rn(log_inv_sqrt_2pi, lsd), __frcp_rn(sd));
}

// the Gaussian of a padding column (no k-mer): z-score and log-density stay finite, and the column's cells are never live
__device__ __forceinline__ float4 nph_pad_gaussian() { return make_float4(0.f, 1.f, 0.f, 1.f); }

// Persistent warps: the warp's next n slots of a work queue (lane 0 pops, every lane gets the first slot's index)
__device__ __forceinline__ uint32_t nph_warp_pop(unsigned int* counter, unsigned int n, int lane)
{
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(counter, n);
    return __shfl_sync(0xffffffffu, base, 0);
}

// Inclusive sum of v over the block (blockDim.x a multiple of 32; every thread calls it), s: 32 values of shared memory.
// Each warp scans by shuffles, then warp 0 scans the warp totals.
template <typename T>
__device__ __forceinline__ T nph_block_scan_incl(T v, T* s, int t)
{
    const int lane = t & 31, w = t >> 5;
    for (int o = 1; o < 32; o <<= 1) { const T x = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += x; }
    if (lane == 31) s[w] = v;
    __syncthreads();
    if (w == 0) {
        T x = s[lane];
        for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        s[lane] = x;
    }
    __syncthreads();
    if (w > 0) v += s[w - 1];
    __syncthreads();
    return v;
}

#endif

// where the HMM jobs in ctx->d_jobs and their ranks come from
enum class NphJobSource {
    HostRanks,      // k-mer ranks from the caller: every rank is checked against the model
    HostCodes,      // base codes from the caller (the *_seq calls): every code is checked, then turned into ranks
    DeviceRanks,    // ranks a kernel of ours wrote (call-methylation, variant screening): job ranges are checked, ranks are not walked
};

// kernels (defined in hmm_forward.cu / abea.cu)
int nph_launch_read_prologue(nph_ctx* ctx);
int nph_launch_hmm_forward(nph_ctx* ctx, float* scores_dev);
size_t nph_hmm_scratch_bytes(const nph_ctx* ctx);
int nph_launch_abea(nph_ctx* ctx);
int nph_schedule_hmm_jobs(nph_ctx* ctx, size_t n_jobs, size_t n_ranks_total, NphJobSource src, uint32_t* max_E_out);
// per-read (lp_mm_self, lp_mm_next) of the resident reads into ctx->d_trans (host libm, like calculate_transitions)
int nph_upload_read_transitions(nph_ctx* ctx, double indel_bias);
// Checks every record (read and model index, its slice of the n_map bases, its pair-list slice, ref_len <= max_len, then
// check(r, R)) and uploads the batch into ev (methylation.cu).  compact: deltas (n_map) and first_event; else pairs.
int nph_event_records_load(nph_ctx* ctx, NphEventRecords& ev, const char* ref, size_t n_ref, size_t n_map, bool compact,
                           const int16_t* deltas, const int32_t* first_event, const nph_aligned_pair* pairs, size_t n_pairs,
                           const nph_meth_record* records, size_t n_records, uint32_t max_len,
                           const std::function<int(size_t, const nph_meth_record&)>& check);
// Compact form: the event index of every base (NPH_NO_EVENT: no entry) at dense[ref_off + o] and each record's first base with
// an entry (ref_len: none) at first_valid[record].  Pair form: both nullptr, nothing launched.
int nph_event_records_expand(nph_ctx* ctx, NphEventRecords& ev, const int32_t** dense, const int32_t** first_valid);
constexpr int32_t NPH_NO_EVENT = INT32_MIN;
// Exclusive prefix sum over n values on ctx->stream (scan.cu): out[0..n) the prefix, out[n] the total.  scratch holds
// nph_scan_scratch(n) values from the caller's arena.
size_t nph_scan_scratch(size_t n);
int nph_scan_exclusive(nph_ctx* ctx, const uint64_t* in, uint32_t n, uint64_t* out, uint64_t* scratch);

// One event sequence of a calling window: the record and its events e1 (window start) and e2 (window end).
struct NphWinPair { uint32_t record; int32_t e1, e2; };
// The profile HMM's DP rows of a pair's job: one per event of [e1, e2] or [e2, e1].
__host__ __device__ inline uint32_t nph_pair_rows(int32_t e1, int32_t e2) { return (uint32_t)(e1 > e2 ? e1 - e2 : e2 - e1) + 1u; }

// The region calls (window_reads.cu).  nph_region_load: nph_reads_load, then the records into ctx->region.ev in compact form
// (records index the event deltas), each record also passing check(r, R).
int nph_region_load(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, const double* ev_start_time,
                    size_t n_events_total, const char* ref, size_t n_ref, const int16_t* deltas, size_t n_deltas, const int32_t* first_event,
                    const nph_meth_record* records, size_t n_records, const std::function<int(size_t, const nph_meth_record&)>& check);
// What nph_window_reads found for n windows: AlignmentDB::get_event_subsequences of each, keeping the pairs with |e1 - e2| >= min_span.
struct NphWindowReads {
    std::vector<uint64_t> off;             // n + 1: each window's first kept pair, then their total
    std::vector<uint32_t> met;             // per window: every event sequence found, kept or not
    std::vector<uint64_t> rows;            // per window: nph_pair_rows summed over its kept pairs
    uint32_t max_rows = 0;                 // the largest nph_pair_rows of a kept pair (0: none)
    const uint64_t* d_off = nullptr;       // device copies of off, and the kept pairs window by window, each window's in record
    const NphWinPair* d_pairs = nullptr;   // order, with the window of each pair
    const uint32_t* d_pair_win = nullptr;
    uint64_t n_pairs() const { return off.back(); }
};
// The reads of n >= 1 windows [bounds[w].x, bounds[w].y] over the records in ctx->region.ev: count, scan, one read-back, fill.
int nph_window_reads(nph_ctx* ctx, const std::vector<int2>& bounds, int min_span, NphWindowReads& wr);
// validate + classify + schedule the n_jobs jobs already sitting in ctx->d_jobs / d_ranks (one stream sync), size the scratch
int nph_jobs_schedule(nph_ctx* ctx, size_t n_jobs, size_t n_ranks_total, NphJobSource src);
// Scores n_jobs jobs that emit() writes into ctx->d_jobs (ranks already in ctx->d_ranks, written by a kernel of ours): reserves
// the job, order and score arrays, uploads the read transitions, runs emit(), schedules and launches the forward kernels.
int nph_score_device_jobs(nph_ctx* ctx, size_t n_jobs, size_t n_ranks_total, double indel_bias, const std::function<int()>& emit);
// K3 on the n_jobs jobs a kernel of ours wrote into ctx->d_jobs / d_ranks, read transitions and flank table already in place (as
// nph_score_device_jobs leaves them; hmm_viterbi.cu): one class and trace size for the bounds max_K x max_E, jobs in index order.
// Job j = ctx->d_jobs[first_job + j]: its path goes to d_states[d_states_off[j] ..) (room d_states_off[j + 1] - d_states_off[j]),
// its length to d_n_states[j] (0 where the reference would assert).  Device pointers; nothing is read back.
int nph_viterbi_device_jobs(nph_ctx* ctx, size_t n_jobs, uint32_t max_K, uint32_t max_E, const uint64_t* d_states_off,
                            nph_align_state* d_states, uint32_t* d_n_states, size_t first_job);
// One chunk of nph_viterbi_chunks: jobs [j0, j0 + n) of the caller's numbering, job j0 + i's path at states + states_off[i]
// (n_states[i] states, 0 where the reference asserts).  Device pointers.
struct NphVitChunk {
    uint64_t j0, n;
    const nph_align_state* states;
    const uint64_t* states_off;
    const uint32_t* n_states;
};
// K3 over n_jobs jobs in consecutive chunks whose Viterbi states, max_K + max_E per job, fit 1 GiB of buf, at most max_chunk jobs
// each (0: no cap), rounded down to a multiple of unit (at least unit).  Per chunk: prepare(j0, nj, first) puts the chunk's jobs in
// ctx->d_jobs from index `first` on (with their ranks, transitions and flank table, as nph_score_device_jobs leaves them), then K3
// runs on them and fold(chunk) launches the kernels that consume the paths.  *ms: the device time of the offset kernel, K3 and fold
// over all chunks, *fold_ms (optional) the fold's share of it; *launches: their launches; *n_chunks: the chunks.
int nph_viterbi_chunks(nph_ctx* ctx, DevBuf<uint8_t>& buf, uint64_t n_jobs, uint64_t max_chunk, uint64_t unit, uint32_t max_K, uint32_t max_E,
                       const std::function<int(uint64_t j0, uint64_t nj, uint64_t& first)>& prepare,
                       const std::function<int(const NphVitChunk&)>& fold, float* ms, int* launches, uint32_t* n_chunks,
                       float* fold_ms = nullptr);
// One-shot calls (read batch, work and results in one call).  Begin: read records on the main stream, then upload() (the
// jobs or records), then the event levels in chunks on the copy stream behind progress words the forward kernel polls —
// enumeration and scheduling run while the levels still cross PCIe.  Finish, on every path: wait for the copy stream.
int nph_oneshot_begin(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, const double* ev_start_time,
                      size_t n_events_total, const std::function<int()>& upload);
void nph_oneshot_finish(nph_ctx* ctx);

// ---- device-level pieces of the raw-read prologue (event_detect.cu, squiggle_prep.cu, abea.cu), chained by
// load_from_raw.cu without leaving the device.  Inputs named d_* are device pointers; everything runs on ctx->stream.
size_t nph_ed_scratch_bytes(size_t n_reads, size_t events_total);
int nph_detect_events_device(nph_ctx* ctx, const float* d_raw, size_t n_samples_total, const nph_raw_read* reads, size_t n_reads,
                             const nph_event_params* params, uint8_t* scratch, size_t events_total,
                             nph_event** d_events_out, uint32_t** d_n_events_out, std::vector<uint32_t>& h_n_events, int* launches_out);
size_t nph_trim_scratch_bytes(const nph_raw_read* reads, size_t n_reads, int32_t varseg_chunk);
int nph_trim_device(nph_ctx* ctx, const float* d_raw, size_t n_samples_total, const nph_raw_read* reads, size_t n_reads,
                    int32_t trim_start, int32_t trim_end, int32_t varseg_chunk, float varseg_thresh, uint8_t* scratch,
                    nph_raw_range* ranges_out /* host */);
struct NphCalArgs {
    const float* ev_mean;
    const nph_read* reads;
    const uint32_t* ranks;
    const nph_abea_job* jobs;
    const nph_abea_result* results;
    const nph_aligned_pair* pairs;
    uint32_t n_jobs, model_id;
    nph_event_range* b2e;        // n_kmers entries per job at rank_off
    nph_calibration* out;
    int* bad_input;
};
int nph_launch_recalibrate(nph_ctx* ctx, const NphCalArgs& args);
// estimate_scalings_using_mom of n_jobs jobs over the resident reads' event means: 2 doubles (shift, scale) per job
int nph_launch_mom(nph_ctx* ctx, const nph_abea_job* d_jobs, const uint32_t* d_ranks, size_t n_jobs, uint32_t model_id, double* d_out, bool reversed);
// Stages n_jobs checked ABEA jobs over reads on the device with n_events[read] events: transition terms, longest-first order,
// band trace room, every ABEA buffer reserved (the caller fills ctx->d_abea_ranks), uploads.  Sets no residency flag and does
// not synchronise.
int nph_abea_stage(nph_ctx* ctx, const uint32_t* n_events, const nph_abea_job* jobs, size_t n_jobs, size_t n_ranks_total, uint32_t model_id,
                   size_t pairs_total);
// NPH_ERR_INVALID unless every rank of d_ranks[0, n) is below n_states and every level of d_levels[0, n_levels) is within
// +-NPH_ABEA_MAX_LEVEL:
// one kernel, one flag copied back (a stream sync).
int nph_check_ranks(nph_ctx* ctx, const uint32_t* d_ranks, size_t n, uint32_t n_states, const float* d_levels = nullptr, size_t n_levels = 0);

#ifdef __CUDACC__
// AlignmentDB::_find_by_ref_bounds (ref: src/alignment/nanopolish_alignment_db.cpp:688-731) on one record's dense event map
// (event index per reference offset, NPH_NO_EVENT where aligned_events has no entry; fv its first offset with an entry) for the
// window [cs, ce] in reference coordinates: the event indices at the two lower_bounds.  nph_event_subsequence and phase-reads call it.
__device__ __forceinline__ int nph_first_valid_from(const int32_t* __restrict__ dense, int n, int from)
{
    for (int o = from < 0 ? 0 : from; o < n; ++o) if (dense[o] != NPH_NO_EVENT) return o;
    return n;
}
__device__ __forceinline__ bool nph_find_by_ref_bounds(const nph_meth_record& R, const int32_t* __restrict__ dense, int fv, int cs, int ce,
                                                       int& e1, int& e2)
{
    const int n = (int)R.ref_len;
    if (fv >= n) return false;                                   // aligned_events.empty()
    const int os = cs - R.ref_start_pos, oe = ce - R.ref_start_pos;
    if (oe >= n || os >= n) return false;                        // lower_bound(ref_stop) == end()
    const int is = nph_first_valid_from(dense, n, os);
    if (is >= n) return false;
    const int ie = nph_first_valid_from(dense, n, oe);
    if (ie >= n) return false;
    if (!(is <= os || is != fv)) return false;                   // left_bounded; right_bounded always holds for a lower_bound
    e1 = dense[is]; e2 = dense[ie];
    return true;
}
// AlignmentDB::get_event_subsequences (ref: src/alignment/nanopolish_alignment_db.cpp:172-221) for one record and the window
// [cs, ce]: nph_find_by_ref_bounds plus the event/bp ratio test.  The edit screen's var_bounds_kernel and the window-read walk of the
// region calls (window_reads.cu) call it.
__device__ __forceinline__ bool nph_event_subsequence(const nph_meth_record& R, const int32_t* __restrict__ dense, int fv, int cs, int ce,
                                                      int& e1, int& e2)
{
    if (!nph_find_by_ref_bounds(R, dense, fv, cs, ce, e1, e2)) return false;
    const double ratio = fabs((double)(e1 - e2)) / fabs((double)(ce - cs));
    return ratio < 20.0;                                         // MAX_EVENT_TO_BP_RATIO
}

// Alphabet::rank of the DNA alphabet: unknown symbols rank 0
__device__ __forceinline__ uint8_t nph_dna_code(uint8_t c) { return c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : 0; }
// HMMInputSequence::get_kmer_rank(q, k, false) and (q, k, true) of a DNA sequence held as nph_dna_code ranks: the k-mer at q and the
// rank of its reverse complement (the complement of rank c is 3 - c, so an unknown symbol complements like 'A')
__device__ __forceinline__ void nph_dna_kmer_ranks(const uint8_t* codes, int q, int k, uint32_t& fw, uint32_t& rc)
{
    uint32_t f = 0, r = 0;
    for (int t = 0; t < k; ++t) {
        f = f * 4u + codes[q + t];
        r = r * 4u + (3u - codes[q + k - 1 - t]);
    }
    fw = f; rc = r;
}
// The job header of pair P of record R; the caller fills in rank_off, model_id and n_kmers.
__device__ __forceinline__ nph_hmm_job nph_window_job(const nph_meth_record& R, const NphWinPair& P, uint8_t flags)
{
    nph_hmm_job jb;
    jb.read = R.read;
    jb.event_start = (uint32_t)P.e1; jb.event_stop = (uint32_t)P.e2;
    jb.stride = R.rc ? -1 : 1;          // EventAlignmentRecord::stride agrees with rc for every read the HMM accepts (profile_hmm_r9.inl:275)
    jb.rc = R.rc; jb.flags = flags; jb.reserved = 0;
    return jb;
}
// HMMInputSequence::get_kmer_rank(q, k, rc) of the DNA alphabet, one k-mer at a time, for the nk k-mers of an edited window whose
// base v has the nph_dna_code code(v): the ranks of strand rc into rk
template <typename Code>
__device__ __forceinline__ void nph_window_ranks(Code code, int nk, int k, bool rc, uint32_t* rk)
{
    for (int q = 0; q < nk; ++q) {
        uint8_t c[8];
        for (int i = 0; i < k; ++i) c[i] = code(q + i);
        uint32_t f, r;
        nph_dna_kmer_ranks(c, 0, k, f, r);
        rk[q] = rc ? r : f;
    }
}
#endif
