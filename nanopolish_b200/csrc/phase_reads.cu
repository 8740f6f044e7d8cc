// phase_reads.cu — phase-reads' per-read SNP loop on the device, for a whole batch of BAM records in one call.
//
// Replaces, for every record at once, the variant loop of
//   phase_single_read                    ref: src/nanopolish_phase_reads.cpp:178-347 (the loop :246-318)
//   AlignmentDB::_find_by_ref_bounds     ref: src/alignment/nanopolish_alignment_db.cpp:688-731 (nph_find_by_ref_bounds, shared
//                                        with variant screening)
//   Haplotype::apply_variant on the 61-base calling window   ref: src/nanopolish_haplotype.cpp:30-85
//   HMMInputSequence::get_kmer_rank      ref: src/hmm/nanopolish_hmm_input_sequence.h:76-91 (nph_dna_kmer_ranks, shared with screening)
// and the call / quality arithmetic after the two profile_hmm_score calls (nph_phase_quality, exact_math.cuh).
//
// Kernels around K1, in the load -> count -> scan -> emit -> score -> fill shape of call-methylation:
//   phase_count_kernel  a warp per record, a lane per variant of its range: the scored sites (SNPs whose window is bounded and
//                       whose centre base matches) and their scored events
//   (nph_scan_exclusive, scan.cu: each record's first site; one read-back sizes the job arrays and returns the offsets)
//   phase_emit_kernel   a warp per record, a lane per site: the k-mer ranks of the reference and alternative windows, two
//                       nph_hmm_job records and the site's call record, straight into the arrays K1's device-side scheduler reads
// then hmm_schedule.cu + the forward kernels run unchanged, and phase_fill_kernel turns each site's two scores into its call.
#include "nph_internal.cuh"
#include "exact_math.cuh"
#include <algorithm>
#include <string>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kWin = 2 * NPH_PHASE_FLANK + 1;            // the calling window: [p - 30, p + 30]
constexpr uint64_t kSiteRanks = 2 * (uint64_t)kWin;       // rank slots per site: reference window, then alternative window

struct PhaseArgs {
    const uint8_t* ref;
    const int32_t* dense;              // event index per reference base (nph_event_records_expand)
    const int32_t* first_valid;
    const nph_meth_record* records;
    const nph_phase_variant* variants;
    const uint32_t* range;             // [lo, hi) per record
    const DevModelView* models;
    uint32_t n_records;
};

// d_counts: per record its sites, their exclusive prefix (n + 1), the scan's scratch, the scored-event count
struct PhaseCounts { uint64_t* sites; uint64_t* off; uint64_t* scratch; unsigned long long* n_events; };
PhaseCounts phase_counts_layout(NphArena& a, size_t n)
{
    PhaseCounts c;
    c.sites = a.take<uint64_t>(n);
    c.off = a.take<uint64_t>(n + 1);
    c.scratch = a.take<uint64_t>(nph_scan_scratch(n));
    c.n_events = a.take<unsigned long long>(1);
    return c;
}

// variant v of record R is scored: a SNP, its window bounded by the record's event alignment, its centre base equal to ref_base
__device__ __forceinline__ bool phase_site(const PhaseArgs& a, const nph_meth_record& R, const int32_t* dense, int fv,
                                           const nph_phase_variant& v, int& e1, int& e2)
{
    if (!v.is_snp) return false;
    const int p = v.ref_position;
    if (!nph_find_by_ref_bounds(R, dense, fv, p - NPH_PHASE_FLANK, p + NPH_PHASE_FLANK, e1, e2)) return false;
    return a.ref[R.ref_off + (uint64_t)(p - R.ref_start_pos)] == (uint8_t)v.ref_base;      // a bounded window lies inside ref_seq
}

// EventAlignmentRecord::stride: front().read_pos < back().read_pos ? 1 : -1 over the record's aligned_events (whole warp)
__device__ __forceinline__ int record_stride(const int32_t* __restrict__ dense, int n, int fv, int lane)
{
    if (fv >= n) return 1;
    for (int base = n - 1; base >= fv; base -= 32) {
        const int o = base - lane;
        const unsigned m = __ballot_sync(kFull, o >= fv && dense[o] != NPH_NO_EVENT);
        if (m) return dense[fv] < dense[base - (__ffs(m) - 1)] ? 1 : -1;
    }
    return -1;
}

__global__ void __launch_bounds__(kThreads) phase_count_kernel(const PhaseArgs a, uint64_t* __restrict__ sites, unsigned long long* __restrict__ n_events)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t rec = warp; rec < a.n_records; rec += n_warps) {
        const nph_meth_record R = a.records[rec];
        const int32_t* dense = a.dense + R.ref_off;
        const int fv = a.first_valid[rec];
        const uint32_t lo = a.range[2 * rec], hi = a.range[2 * rec + 1];
        unsigned long long count = 0, ev = 0;
        for (uint32_t base = lo; base < hi; base += 32) {
            const uint32_t v = base + lane;
            int e1 = 0, e2 = 0;
            const bool s = v < hi && phase_site(a, R, dense, fv, a.variants[v], e1, e2);
            count += __popc(__ballot_sync(kFull, s));
            if (s) ev += 2ull * (unsigned long long)((e2 > e1 ? e2 - e1 : e1 - e2) + 1);
        }
        for (int o = 16; o; o >>= 1) ev += __shfl_xor_sync(kFull, ev, o);
        if (lane == 0) {
            sites[rec] = count;
            if (ev) atomicAdd(n_events, ev);
        }
    }
}

__global__ void __launch_bounds__(kThreads) phase_emit_kernel(const PhaseArgs a, const uint64_t* __restrict__ site_off, nph_hmm_job* __restrict__ jobs,
                                                              uint32_t* __restrict__ ranks, nph_phase_call* __restrict__ calls)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t rec = warp; rec < a.n_records; rec += n_warps) {
        const nph_meth_record R = a.records[rec];
        const int32_t* dense = a.dense + R.ref_off;
        const int fv = a.first_valid[rec];
        const int stride = record_stride(dense, (int)R.ref_len, fv, lane);
        const int k = a.models[R.model_id].k;
        const int nk = kWin - k + 1;
        const uint32_t lo = a.range[2 * rec], hi = a.range[2 * rec + 1];
        uint64_t site0 = site_off[rec];
        for (uint32_t base = lo; base < hi; base += 32) {
            const uint32_t v = base + lane;
            int e1 = 0, e2 = 0;
            nph_phase_variant V{};
            if (v < hi) V = a.variants[v];
            const bool s = v < hi && phase_site(a, R, dense, fv, V, e1, e2);
            const unsigned m = __ballot_sync(kFull, s);
            if (s) {
                const uint64_t site = site0 + (uint64_t)__popc(m & ((1u << lane) - 1u));
                // the window as DNA ranks; job k-mer q is get_kmer_rank(q, k, rc) of the reference window, then of the alternative one
                uint8_t w[kWin];
                const uint8_t* win = a.ref + R.ref_off + (uint64_t)(V.ref_position - NPH_PHASE_FLANK - R.ref_start_pos);
                for (int t = 0; t < kWin; ++t) w[t] = nph_dna_code(win[t]);
                uint32_t* out = ranks + site * kSiteRanks;
                for (int alt = 0; alt < 2; ++alt) {
                    if (alt) w[NPH_PHASE_FLANK] = nph_dna_code((uint8_t)V.alt_base);
                    for (int q = 0; q < nk; ++q) {
                        uint32_t fw, rc;
                        nph_dna_kmer_ranks(w, q, k, fw, rc);
                        out[alt * kWin + q] = R.rc ? rc : fw;
                    }
                }
                nph_hmm_job jb;
                jb.rank_off = site * kSiteRanks; jb.read = R.read; jb.model_id = R.model_id;
                jb.event_start = (uint32_t)e1; jb.event_stop = (uint32_t)e2; jb.n_kmers = (uint32_t)nk;
                jb.stride = (int8_t)stride; jb.rc = R.rc; jb.flags = NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP; jb.reserved = 0;
                jobs[2 * site] = jb;
                jb.rank_off += kWin;
                jobs[2 * site + 1] = jb;
                calls[site] = nph_phase_call{rec, v, 0.f, 0.f, 0, 0, {0, 0}};
            }
            site0 += (uint64_t)__popc(m);
        }
    }
}

__global__ void phase_fill_kernel(nph_phase_call* __restrict__ calls, const float* __restrict__ scores, const nph_phase_variant* __restrict__ variants,
                                  const float* __restrict__ tbl, uint64_t n_sites)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_sites; i += (uint64_t)gridDim.x * blockDim.x) {
        nph_phase_call c = calls[i];
        const nph_phase_variant V = variants[c.variant];
        c.ref_score = scores[2 * i];
        c.alt_score = scores[2 * i + 1];
        const NphPhaseCall q = nph_phase_quality(c.ref_score, c.alt_score, V.ref_base, V.alt_base, tbl);
        c.call = q.call; c.qual = q.q_char;
        calls[i] = c;
    }
}

// checks the batch and uploads it: records (nph_event_records_load), variants and ranges
int phase_load(nph_ctx* ctx, const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total, const int32_t* first_event,
               const nph_meth_record* records, size_t n_records, const nph_phase_variant* variants, size_t n_variants,
               const uint32_t* var_range, nph_phase_variant** d_variants, uint32_t** d_range)
{
    nph_ctx::PhaseState& ph = ctx->phase;
    for (size_t r = 0; r < n_records; ++r) {
        if (var_range[2 * r] > var_range[2 * r + 1] || var_range[2 * r + 1] > n_variants) {
            ctx->last_error = "record " + std::to_string(r) + ": variant range out of bounds";
            return NPH_ERR_INVALID;
        }
    }
    NPH_TRY(nph_event_records_load(ctx, ph.ev, ref_bases, n_ref_total, n_ref_total, true, event_deltas, first_event, nullptr, 0,
                                   records, n_records, 0x7fffffffu, [&](size_t r, const nph_meth_record& R) {
        const DevModel& mod = ctx->models[R.model_id];
        if (mod.alphabet_size == 4 && mod.k <= (uint32_t)kWin) return NPH_OK;
        ctx->last_error = "phase record " + std::to_string(r) + ": its model is not a nucleotide model";
        return NPH_ERR_INVALID;
    }));
    NPH_TRY(nph_carve(ctx, ph.d_in, [&](NphArena& a) {
        *d_variants = a.take<nph_phase_variant>(n_variants);
        *d_range = a.take<uint32_t>(2 * n_records);
    }));
    if (n_variants) NPH_CUDA(ctx, cudaMemcpyAsync(*d_variants, variants, sizeof(nph_phase_variant) * n_variants, cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(*d_range, var_range, sizeof(uint32_t) * 2 * n_records, cudaMemcpyHostToDevice, ctx->stream));
    NPH_TRY(nph_carve(ctx, ph.d_counts, [&](NphArena& a) { phase_counts_layout(a, n_records); }));
    return NPH_OK;
}

int phase_run(nph_ctx* ctx, const nph_phase_variant* d_variants, const uint32_t* d_range, double indel_bias, uint64_t* call_off_out,
              nph_phase_call* calls_out, size_t calls_cap, unsigned long long* n_events_out)
{
    nph_ctx::PhaseState& ph = ctx->phase;
    const uint32_t n = (uint32_t)ph.ev.n_records;
    NphArena ca{ph.d_counts.p};
    const PhaseCounts c = phase_counts_layout(ca, n);
    const int32_t* dense;
    const int32_t* first_valid;
    NPH_TRY(nph_event_records_expand(ctx, ph.ev, &dense, &first_valid));
    const PhaseArgs pa{ph.ev.d_ref.p, dense, first_valid, ph.ev.d_records.p, d_variants, d_range, ctx->d_models.p, n};
    const int grid = (int)std::min<size_t>((n + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 8);
    NPH_CUDA(ctx, cudaMemsetAsync(c.n_events, 0, sizeof(unsigned long long), ctx->stream));
    phase_count_kernel<<<grid, kThreads, 0, ctx->stream>>>(pa, c.sites, c.n_events);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_TRY(nph_scan_exclusive(ctx, c.sites, n, c.off, c.scratch));
    NPH_CUDA(ctx, cudaMemcpyAsync(call_off_out, c.off, sizeof(uint64_t) * (n + 1), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(n_events_out, c.n_events, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));          // read-back 1 of 2: the site count that sizes the job arrays
    const uint64_t n_sites = call_off_out[n];
    if (n_sites > calls_cap) {        // calls_out is non-null whenever calls_cap > 0
        ctx->last_error = "calls_cap too small: " + std::to_string(n_sites) + " calls";
        return NPH_ERR_INVALID;
    }
    ctx->n_jobs = 0; ctx->jobs_loaded = false;
    if (n_sites == 0) { ctx->classes.clear(); ctx->jobs_loaded = true; return NPH_OK; }
    const size_t n_ranks = (size_t)n_sites * kSiteRanks;
    NPH_TRY(nph_reserve(ctx, ctx->d_ranks, n_ranks));
    NPH_TRY(nph_reserve(ctx, ph.d_calls, (size_t)n_sites));
    // phase_emit_kernel writes the jobs and their k-mer ranks; the schedule is read-back 2 of 2
    NPH_TRY(nph_score_device_jobs(ctx, 2 * (size_t)n_sites, n_ranks, indel_bias, [&]() -> int {
        phase_emit_kernel<<<grid, kThreads, 0, ctx->stream>>>(pa, c.off, ctx->d_jobs.p, ctx->d_ranks.p, ph.d_calls.p);
        NPH_CUDA(ctx, cudaGetLastError());
        return NPH_OK;
    }));
    const int fgrid = (int)std::min<size_t>(((size_t)n_sites + 255) / 256, (size_t)ctx->sm_count * 8);
    phase_fill_kernel<<<fgrid, 256, 0, ctx->stream>>>(ph.d_calls.p, ctx->d_scores.p, d_variants, ctx->d_logsum.p, n_sites);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaMemcpyAsync(calls_out, ph.d_calls.p, sizeof(nph_phase_call) * (size_t)n_sites, cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->last_launches += 10;        // counted with the forward classes' launches: expand, count, a 3-launch scan, emit, classify/scan/scatter, fill
    return NPH_OK;
}

} // namespace

extern "C" int nph_phase_reads_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                     const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                     const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total, const int32_t* first_event,
                                     const nph_meth_record* records, size_t n_records,
                                     const nph_phase_variant* variants, size_t n_variants, const uint32_t* var_range,
                                     double indel_bias, uint64_t* call_off_out,
                                     nph_phase_call* calls_out, size_t calls_cap, uint64_t* n_scored_events_out)
{
    if (!ctx || !call_off_out) return NPH_ERR_INVALID;
    if (n_scored_events_out) *n_scored_events_out = 0;
    if (n_records == 0) { call_off_out[0] = 0; return NPH_OK; }
    if (!ref_bases || !event_deltas || !first_event || !records || !var_range || (n_variants && !variants)) return NPH_ERR_INVALID;
    if (!calls_out && calls_cap) { ctx->last_error = "calls_out is null but calls_cap is not 0"; return NPH_ERR_INVALID; }
    nph_phase_variant* d_variants = nullptr;
    uint32_t* d_range = nullptr;
    unsigned long long n_events = 0;
    int rc = nph_oneshot_begin(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, [&] {
        return phase_load(ctx, ref_bases, event_deltas, n_ref_total, first_event, records, n_records, variants, n_variants, var_range,
                          &d_variants, &d_range); });
    if (rc == NPH_OK) rc = phase_run(ctx, d_variants, d_range, indel_bias, call_off_out, calls_out, calls_cap, &n_events);
    nph_oneshot_finish(ctx);
    if (rc == NPH_OK && n_scored_events_out) *n_scored_events_out = n_events;
    return rc;
}
