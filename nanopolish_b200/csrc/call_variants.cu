// call_variants.cu — the central step of `nanopolish variants` on the device: the haplotype scores and genotype choice of every
// candidate group of a region in one call.
//
// Replaces, for every group of call_haplotype_from_candidates at once:
//   score_variant_group (its scoring loop)    ref: src/common/nanopolish_variant.cpp:234-258
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_window_reads)
//   VariantGroup's score and read-sum maps    ref: src/nanopolish_variant_db.cpp (set_combination_read_score, get_read_sum_scores)
//   simple_call's genotype search             ref: src/common/nanopolish_variant.cpp:279-367
//   simple_call's read support                ref: src/common/nanopolish_variant.cpp:369-414 (on the host, with its libm)
// The groups, their combinations and haplotypes come from the caller (the host Haplotype applies the variants).
//
// Kernels, after the window-read walk of window_reads.cu (count -> scan -> fill, a window per group) and the rank pool of
// score_sets.cu (nph_set_ranks: both strands of every haplotype and of each methylated copy, and which copies differ; one read-back
// of those masks sizes every group's jobs):
//   cv_emit_kernel       thread per (pair, haplotype): the jobs of its score set; then K1 (nph_score_device_jobs)
//   cv_combine_kernel    thread per (pair, haplotype): nph_score_set_fold of its jobs
//   cv_keys_kernel       warp per group: its pairs mapped to keys in key order, the last record's score per (combination, key),
//                        the read_sum chain over (record, combination) and the last record's strand
//   cv_genotype_kernel   thread per kSetsPerThread consecutive genotype sets of a group: unrank the first, then step through the
//                        rest in visit order; each set folds its keys in key order; block maximum (lowest index among equals)
//   cv_best_kernel       thread per group: its blocks' maxima in order
#include "nph_internal.cuh"
#include "exact_math.cuh"
#include "meth_dev.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kSetsPerThread = 32;
constexpr uint64_t kSetsPerBlock = (uint64_t)kThreads * kSetsPerThread;
constexpr uint64_t kNone = ~0ull;
constexpr uint64_t kMaxSets = 1ull << 60;
// simple_call's `double log_2 = log(2)`: the double nearest ln 2 (glibc's log is correctly rounded there)
constexpr double kLog2 = 0.69314718055994530942;

// per group, what the kernels need
struct CvGroup {
    uint64_t pair_first;                // its pairs [pair_first, pair_first + n_pairs) of the walk, in record order
    uint64_t item_base;                 // its (pair, haplotype) items and its key table: n_pairs x n_haps floats each
    uint64_t job_base;                  // its first job; each pair has jobs_per_pair consecutive jobs
    uint64_t n_sets;                    // genotype sets
    uint32_t n_pairs, n_haps, hap_first, jobs_per_pair;
};

__host__ __device__ inline uint64_t gt_binom(uint64_t n, uint32_t r)
{
    if (r > n) return 0;
    uint64_t v = 1;
    for (uint32_t i = 1; i <= r; ++i) v = v * (n - r + i) / i;     // exact at every step: C(n - r + i, i)
    return v;
}

// set idx of Combinations(n, p, CO_WITH_REPLACEMENT): the idx-th non-decreasing p-tuple over [0, n) in lexicographic order
__host__ __device__ inline void gt_unrank(uint64_t idx, uint32_t n, int p, uint32_t* c)
{
    uint32_t a = 0;
    for (int j = 0; j < p; ++j) {
        const uint32_t m = (uint32_t)(p - j - 1);
        for (uint32_t v = a;; ++v) {
            const uint64_t cnt = gt_binom((uint64_t)(n - v) + m - 1, m);    // tuples of the m ids after this one, over [v, n)
            if (idx < cnt || v == n - 1) { c[j] = v; a = v; break; }
            idx -= cnt;
        }
    }
}

__device__ __forceinline__ uint32_t cv_group_of(const uint64_t* __restrict__ off, uint32_t n, uint64_t x)
{
    uint32_t lo = 0, hi = n;                // the last g with off[g] <= x
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (off[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

struct CvArgs {
    const CvGroup* groups;
    const uint64_t* item_off;           // n_groups + 1: each group's item_base, then the total
    const NphSetSeq* haps;              // per haplotype: its bases and rank-pool offset
    const uint32_t* job_off;            // per haplotype: its first job in a pair's jobs
    const NphWinPair* pairs;
    const nph_meth_record* records;
    uint32_t n_groups, flags;
};

__global__ void cv_emit_kernel(const CvArgs a, uint64_t n_items, int k, nph_hmm_job* __restrict__ jobs, const NphSetTypes ty,
                               const uint32_t* __restrict__ alts)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_items) return;
    const uint32_t g = cv_group_of(a.item_off, a.n_groups, t);
    const CvGroup G = a.groups[g];
    const uint64_t local = t - G.item_base;
    const uint32_t pl = (uint32_t)(local / G.n_haps), h = G.hap_first + (uint32_t)(local % G.n_haps);
    const NphWinPair P = a.pairs[G.pair_first + pl];
    const nph_meth_record R = a.records[P.record];
    const NphSetSeq H = a.haps[h];
    nph_hmm_job jb = nph_window_job(R, P, (uint8_t)a.flags);
    jb.n_kmers = H.len - (uint32_t)k + 1u;
    set_jobs(ty, jb, R, P.record, ty.T ? alts[h] : 0u, H.rank_off, jb.n_kmers, jobs + G.job_base + (uint64_t)pl * G.jobs_per_pair + a.job_off[h]);
}

// s[item] = profile_hmm_score_set of the item's jobs (a float)
__global__ void cv_combine_kernel(const CvArgs a, uint64_t n_items, const float* __restrict__ scores, const NphSetTypes ty,
                                  const uint32_t* __restrict__ alts, float* __restrict__ s)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_items) return;
    const uint32_t g = cv_group_of(a.item_off, a.n_groups, t);
    const CvGroup G = a.groups[g];
    const uint64_t local = t - G.item_base;
    const uint32_t pl = (uint32_t)(local / G.n_haps), h = G.hap_first + (uint32_t)(local % G.n_haps);
    const uint32_t n = set_size(alts[h]);
    s[t] = nph_score_set_fold(scores + G.job_base + (uint64_t)pl * G.jobs_per_pair + a.job_off[h], n, ty.pen[n - 1], ty.tbl);
}

// warp per group.  Pair p of the group has key_rank kr(p); its key is the number of distinct ranks below kr(p).  A pair is its key's
// first (flag 1) or last (flag 2) record.  ks[item_base + c * n_pairs + key] = s of the key's last record and combination c (the
// std::map keeps the later score), read_sum[pair_first + key] = the add_logs chain over the key's records and combinations in loop
// order, key_rc[pair_first + key] = the last record's rc.
__global__ void __launch_bounds__(kThreads) cv_keys_kernel(const CvArgs a, const uint32_t* __restrict__ key_rank, const float* __restrict__ s,
                                                           const float* __restrict__ tbl, uint32_t* __restrict__ flag, uint32_t* __restrict__ key,
                                                           float* __restrict__ ks, float* __restrict__ read_sum, uint32_t* __restrict__ key_rc,
                                                           uint32_t* __restrict__ n_keys)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (warp >= a.n_groups) return;
    const CvGroup G = a.groups[warp];
    const NphWinPair* P = a.pairs + G.pair_first;
    const auto kr = [&](uint32_t p) { return key_rank[a.records[P[p].record].read]; };
    uint32_t* fl = flag + G.pair_first;
    uint32_t* ky = key + G.pair_first;
    uint32_t firsts = 0;
    for (uint32_t p = lane; p < G.n_pairs; p += 32) {
        const uint32_t r = kr(p);
        bool first = true, last = true;
        for (uint32_t i = 0; i < G.n_pairs; ++i) {
            if (i == p || kr(i) != r) continue;
            if (i < p) first = false; else last = false;
        }
        fl[p] = (first ? 1u : 0u) | (last ? 2u : 0u);
        firsts += first;
    }
    __syncwarp();
    for (uint32_t p = lane; p < G.n_pairs; p += 32) {
        const uint32_t r = kr(p);
        uint32_t below = 0;
        for (uint32_t i = 0; i < G.n_pairs; ++i) below += (fl[i] & 1u) && kr(i) < r;
        ky[p] = below;
    }
    for (int o = 16; o; o >>= 1) firsts += __shfl_xor_sync(kFull, firsts, o);
    __syncwarp();
    const float* sp = s + G.item_base;
    float* kt = ks + G.item_base;
    for (uint32_t q = lane; q < firsts; q += 32) {
        float sum = 0.f;
        bool any = false;
        for (uint32_t p = 0; p < G.n_pairs; ++p) {
            if (ky[p] != q) continue;
            const bool last = (fl[p] & 2u) != 0;
            for (uint32_t c = 0; c < G.n_haps; ++c) {
                const float v = sp[(uint64_t)p * G.n_haps + c];
                sum = any ? nph_flogsum(sum, v, tbl) : v;
                any = true;
                if (last) kt[(uint64_t)c * G.n_pairs + q] = v;
            }
            if (last) key_rc[G.pair_first + q] = a.records[P[p].record].rc;
        }
        read_sum[G.pair_first + q] = sum;
    }
    if (lane == 0) n_keys[warp] = firsts;
}

struct GtArgs {
    const CvGroup* groups;
    const uint64_t* blk_off;            // n_groups + 1: each group's first block, then the total
    const uint32_t* n_keys;
    const float* ks;
    const float* tbl;
    uint32_t n_groups;
    int ploidy;
};

struct GtBest { double score; uint64_t idx; };

// a beats b: a higher score, or the same score at a lower index (the first set to exceed the best so far)
__device__ __forceinline__ bool gt_better(double as, uint64_t ai, double bs, uint64_t bi) { return as > bs || (as == bs && ai < bi); }

template <int P>
__global__ void __launch_bounds__(kThreads, 2) cv_genotype_kernel(const GtArgs a, GtBest* __restrict__ partial, double* __restrict__ base_score)
{
    __shared__ GtBest sh[kWarps];
    const uint32_t g = cv_group_of(a.blk_off, a.n_groups, blockIdx.x);
    const CvGroup G = a.groups[g];
    const uint32_t nk = a.n_keys[g], n = G.n_haps, stride = G.n_pairs;
    const float* kt = a.ks + G.item_base;
    const uint64_t first = (blockIdx.x - a.blk_off[g]) * kSetsPerBlock + (uint64_t)threadIdx.x * kSetsPerThread;
    double best = -INFINITY;
    uint64_t best_i = kNone;
    if (first < G.n_sets) {
        uint32_t c[P];
        gt_unrank(first, n, P, c);
        const uint64_t end = min(first + (uint64_t)kSetsPerThread, G.n_sets);
        for (uint64_t i = first;;) {
            // set_score: per key in key order, set_sum = add_logs(set_sum, s - log_2) from -inf (p7_FLogsum narrows to float)
            double set_score = 0.0;
            for (uint32_t q = 0; q < nk; ++q) {
                float v = -INFINITY;
#pragma unroll
                for (int j = 0; j < P; ++j) v = nph_flogsum(v, __double2float_rn(__dsub_rn((double)kt[(uint64_t)c[j] * stride + q], kLog2)), a.tbl);
                set_score = __dadd_rn(set_score, (double)v);
            }
            if (i == 0) base_score[g] = set_score;
            if (set_score > best) { best = set_score; best_i = i; }
            if (++i == end) break;
            // the next non-decreasing tuple: the last id below n - 1 goes up by one, every id after it takes its value
            int last = 0;
#pragma unroll
            for (int j = 0; j < P; ++j) if (c[j] != n - 1) last = j;
            uint32_t v = 0;
#pragma unroll
            for (int j = 0; j < P; ++j) if (j == last) v = c[j] + 1;
#pragma unroll
            for (int j = 0; j < P; ++j) if (j >= last) c[j] = v;
        }
    }
    for (int o = 16; o; o >>= 1) {
        const double os = __shfl_xor_sync(kFull, best, o);
        const uint64_t oi = __shfl_xor_sync(kFull, best_i, o);
        if (gt_better(os, oi, best, best_i)) { best = os; best_i = oi; }
    }
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = GtBest{best, best_i};
    __syncthreads();
    if (threadIdx.x == 0) {
        GtBest b = sh[0];
        for (int w = 1; w < kWarps; ++w)
            if (gt_better(sh[w].score, sh[w].idx, b.score, b.idx)) b = sh[w];
        partial[blockIdx.x] = b;
    }
}

// one instantiation per ploidy, so that a set's ids stay in registers
template <int P>
void launch_genotype(const GtArgs& a, uint64_t blocks, cudaStream_t st, GtBest* partial, double* base)
{
    if (a.ploidy == P) cv_genotype_kernel<P><<<(unsigned)blocks, kThreads, 0, st>>>(a, partial, base);
    else if constexpr (P < NPH_CALL_MAX_PLOIDY) launch_genotype<P + 1>(a, blocks, st, partial, base);
}

// thread per group: its blocks' maxima in block (so set) order; kNone when no set exceeded -inf
__global__ void cv_best_kernel(const GtArgs a, const GtBest* __restrict__ partial, GtBest* __restrict__ out)
{
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.n_groups) return;
    GtBest b{-INFINITY, kNone};
    for (uint64_t x = a.blk_off[g]; x < a.blk_off[g + 1]; ++x)
        if (partial[x].idx != kNone && gt_better(partial[x].score, partial[x].idx, b.score, b.idx)) b = partial[x];
    out[g] = b;
}

// the checks on the caller's groups and haplotypes; n_sets per group
int check_groups(nph_ctx* ctx, const nph_call_params& p, size_t n_ref, const nph_call_group* groups, size_t n_groups,
                 const nph_call_haplotype* haps, size_t n_haps, size_t n_bases, const uint32_t* cvars, size_t n_cvars, size_t n_variants,
                 std::vector<uint64_t>& n_sets)
{
    const int64_t region_end = (int64_t)p.region_start + (int64_t)n_ref - 1;
    n_sets.resize(n_groups);
    for (size_t g = 0; g < n_groups; ++g) {
        const nph_call_group& G = groups[g];
        const std::string at = "group " + std::to_string(g) + ": ";
        if (G.n_haplotypes < 2) { ctx->last_error = at + "fewer than 2 haplotypes"; return NPH_ERR_INVALID; }
        if (G.n_haplotypes < p.ploidy) { ctx->last_error = at + "fewer haplotypes than the ploidy (Combinations asserts)"; return NPH_ERR_INVALID; }
        if (!nph_slice_ok(G.hap_first, G.n_haplotypes, n_haps)) { ctx->last_error = at + "haplotypes outside the haplotype array"; return NPH_ERR_INVALID; }
        if (!nph_slice_ok(G.var_first, G.n_variants, n_variants)) { ctx->last_error = at + "variants outside the variant results"; return NPH_ERR_INVALID; }
        if (G.calling_start > G.calling_end || G.calling_start < p.region_start || G.calling_end > region_end) {
            ctx->last_error = at + "window [" + std::to_string(G.calling_start) + ", " + std::to_string(G.calling_end) + "] outside the region (substr_by_reference asserts)";
            return NPH_ERR_INVALID;
        }
        for (uint32_t c = 0; c < G.n_haplotypes; ++c) {
            const nph_call_haplotype& H = haps[G.hap_first + c];
            const std::string ah = at + "haplotype " + std::to_string(c) + ": ";
            if (!nph_slice_ok(H.var_off, H.n_var, n_cvars)) { ctx->last_error = ah + "variant ids outside combination_variants"; return NPH_ERR_INVALID; }
            if ((c == 0) != (H.n_var == 0)) { ctx->last_error = ah + "combination 0 must be the only empty one"; return NPH_ERR_INVALID; }
            for (uint32_t i = 0; i < H.n_var; ++i)
                if (cvars[H.var_off + i] >= G.n_variants) { ctx->last_error = ah + "a variant id outside its group"; return NPH_ERR_INVALID; }
        }
        // C(n + ploidy - 1, ploidy) with the products of gt_binom kept below 2^64
        unsigned __int128 v = 1;
        const uint64_t N = (uint64_t)G.n_haplotypes + p.ploidy - 1;
        for (uint32_t i = 1; i <= p.ploidy; ++i) v = v * (N - p.ploidy + i) / i;
        if (v > kMaxSets) { ctx->last_error = at + "more than 2^60 genotype sets"; return NPH_ERR_INVALID; }
        n_sets[g] = (uint64_t)v;
    }
    return NPH_OK;
}

} // namespace

extern "C" int nph_call_variant_groups_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                             const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                             const char* ref_bases, size_t n_ref_bases,
                                             const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                             const nph_meth_record* records, size_t n_records, const uint32_t* key_rank,
                                             const nph_call_params* params,
                                             const nph_call_group* groups, size_t n_groups,
                                             const nph_call_haplotype* haplotypes, size_t n_haplotypes,
                                             const char* haplotype_bases, size_t n_bases,
                                             const uint32_t* combination_variants, size_t n_combination_variants,
                                             size_t n_variants, double indel_bias,
                                             const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                                             nph_call_group_result* groups_out, nph_call_variant_result* variants_out,
                                             nph_call_counts* counts_out)
{
    if (!ctx || !params || (n_groups && (!groups || !groups_out)) || (n_variants && !variants_out)) return NPH_ERR_INVALID;
    if ((n_haplotypes && !haplotypes) || (n_bases && !haplotype_bases) || (n_combination_variants && !combination_variants)) return NPH_ERR_INVALID;
    if (n_records && (!records || !first_event || (n_deltas_total && !event_deltas))) return NPH_ERR_INVALID;
    if (n_reads && !key_rank) return NPH_ERR_INVALID;
    if (!ref_bases || !ev_start_time) return NPH_ERR_INVALID;
    if (n_ref_bases < 1 || n_ref_bases > 0x7fffffffu || (int64_t)params->region_start + (int64_t)n_ref_bases - 1 > INT32_MAX) return NPH_ERR_INVALID;
    const nph_call_params p = *params;
    if (p.k < 1 || p.k > 8) { ctx->last_error = "k outside 1..8"; return NPH_ERR_INVALID; }
    if (p.ploidy < 1 || p.ploidy > NPH_CALL_MAX_PLOIDY) { ctx->last_error = "ploidy outside 1..NPH_CALL_MAX_PLOIDY"; return NPH_ERR_INVALID; }
    if (p.alignment_flags & ~(NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP)) { ctx->last_error = "unknown alignment_flags"; return NPH_ERR_INVALID; }
    if (n_haplotypes > 0xffffffffu || n_groups > 0xffffffffu) { ctx->last_error = "more than 2^32 - 1 groups or haplotypes"; return NPH_ERR_INVALID; }
    std::vector<MethDev> md;
    NPH_TRY(nph_region_types(ctx, p.k, meth, n_records, alt_model_ids, md));
    std::vector<uint64_t> n_sets;
    NPH_TRY(check_groups(ctx, p, n_ref_bases, groups, n_groups, haplotypes, n_haplotypes, n_bases, combination_variants, n_combination_variants,
                         n_variants, n_sets));
    nph_call_counts cnt{};
    cnt.n_groups = n_groups;
    for (size_t g = 0; g < n_groups; ++g) { cnt.n_haplotypes += groups[g].n_haplotypes; cnt.n_sets += n_sets[g]; }
    for (size_t v = 0; v < n_variants; ++v) variants_out[v] = nph_call_variant_result{0u, 0u, 0.0, {0.0, 0.0, 0.0, 0.0}};
    if (n_groups == 0) {
        if (counts_out) *counts_out = cnt;
        nph_timing_staged(ctx, 0.f, 0);
        return NPH_OK;
    }
    NphSetTypes ty;
    NPH_TRY(nph_region_load_types(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, ref_bases, n_ref_bases, event_deltas, n_deltas_total,
                                  first_event, records, n_records, p.k, md, alt_model_ids, ty));
    cudaStream_t st = ctx->stream;
    const size_t G = n_groups;
    std::vector<NphSetSeq> hv(n_haplotypes);
    for (size_t h = 0; h < n_haplotypes; ++h) {
        const nph_call_haplotype& H = haplotypes[h];
        if (H.seq_len < p.k || !nph_slice_ok(H.seq_off, H.seq_len, n_bases)) { ctx->last_error = "a haplotype outside haplotype_bases or with fewer than k bases"; return NPH_ERR_INVALID; }
        hv[h] = NphSetSeq{H.seq_off, 0, H.seq_len, 0u};
    }
    // the groups' reads
    std::vector<int2> bounds(G);
    for (size_t g = 0; g < G; ++g) bounds[g] = make_int2(groups[g].calling_start, groups[g].calling_end);
    NphWindowReads wr;
    NPH_TRY(nph_window_reads(ctx, bounds, 0, wr));
    const uint64_t n_pairs = wr.n_pairs();
    cnt.n_pairs = n_pairs;
    std::vector<CvGroup> gv(G);
    std::vector<uint64_t> item_off(G + 1), blk_off(G + 1);
    uint64_t items = 0, blocks = 0;
    for (size_t g = 0; g < G; ++g) {
        const uint32_t np = (uint32_t)(wr.off[g + 1] - wr.off[g]);
        gv[g] = CvGroup{wr.off[g], items, 0, n_sets[g], np, groups[g].n_haplotypes, groups[g].hap_first, 0u};
        item_off[g] = items;
        items += (uint64_t)np * groups[g].n_haplotypes;
        blk_off[g] = blocks;
        blocks += (n_sets[g] + kSetsPerBlock - 1) / kSetsPerBlock;
    }
    item_off[G] = items;
    blk_off[G] = blocks;
    if (blocks > (uint64_t)INT32_MAX) { ctx->last_error = "more genotype sets than one launch covers"; return NPH_ERR_INVALID; }
    nph_ctx::CallState& cs = ctx->call;
    CvGroup* d_groups; uint64_t* d_item_off; uint64_t* d_blk_off; NphSetSeq* d_haps; uint32_t* d_job_off; uint8_t* d_bases; uint32_t* d_key_rank;
    uint32_t* d_alts;
    NPH_TRY(nph_carve(ctx, cs.d_in, [&](NphArena& c) {
        d_groups = c.take<CvGroup>(G);
        d_item_off = c.take<uint64_t>(G + 1);
        d_blk_off = c.take<uint64_t>(G + 1);
        d_haps = c.take<NphSetSeq>(n_haplotypes);
        d_job_off = c.take<uint32_t>(n_haplotypes);
        d_bases = c.take<uint8_t>(n_bases + 1);
        d_key_rank = c.take<uint32_t>(n_reads + 1);
        d_alts = c.take<uint32_t>(n_haplotypes);
    }));
    float* d_s; float* d_ks; float* d_read_sum; uint32_t* d_key_rc; uint32_t* d_flag; uint32_t* d_key; uint32_t* d_n_keys;
    GtBest* d_partial; GtBest* d_best; double* d_base;
    NPH_TRY(nph_carve(ctx, cs.d_work, [&](NphArena& c) {
        d_s = c.take<float>(items + 1);
        d_ks = c.take<float>(items + 1);
        d_read_sum = c.take<float>(n_pairs + 1);
        d_key_rc = c.take<uint32_t>(n_pairs + 1);
        d_flag = c.take<uint32_t>(n_pairs + 1);
        d_key = c.take<uint32_t>(n_pairs + 1);
        d_n_keys = c.take<uint32_t>(G);
        d_partial = c.take<GtBest>(blocks);
        d_best = c.take<GtBest>(G);
        d_base = c.take<double>(G);
    }));
    if (n_bases) NPH_CUDA(ctx, cudaMemcpyAsync(d_bases, haplotype_bases, n_bases, cudaMemcpyHostToDevice, st));
    if (n_reads) NPH_CUDA(ctx, cudaMemcpyAsync(d_key_rank, key_rank, sizeof(uint32_t) * n_reads, cudaMemcpyHostToDevice, st));
    uint64_t pool = 0;
    NPH_TRY(nph_set_ranks(ctx, hv, d_haps, d_bases, p.k, ty, d_alts, &pool));
    std::vector<uint32_t> alts(n_haplotypes), job_off(n_haplotypes);
    NPH_CUDA(ctx, cudaMemcpyAsync(alts.data(), d_alts, sizeof(uint32_t) * n_haplotypes, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));                         // read-back: each haplotype's set size lays out the jobs
    uint64_t n_jobs = 0;
    for (size_t g = 0; g < G; ++g) {
        uint32_t J = 0;
        for (uint32_t c = 0; c < groups[g].n_haplotypes; ++c) {
            const uint32_t h = groups[g].hap_first + c;
            job_off[h] = J;
            J += 1u + (uint32_t)__builtin_popcount(alts[h]);
        }
        gv[g].jobs_per_pair = J;
        gv[g].job_base = n_jobs;
        n_jobs += (uint64_t)gv[g].n_pairs * J;
        cnt.n_dp_rows += wr.rows[g] * J;
    }
    cnt.n_jobs = n_jobs;
    NPH_CUDA(ctx, cudaMemcpyAsync(d_job_off, job_off.data(), sizeof(uint32_t) * n_haplotypes, cudaMemcpyHostToDevice, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_groups, gv.data(), sizeof(CvGroup) * G, cudaMemcpyHostToDevice, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_item_off, item_off.data(), sizeof(uint64_t) * (G + 1), cudaMemcpyHostToDevice, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_blk_off, blk_off.data(), sizeof(uint64_t) * (G + 1), cudaMemcpyHostToDevice, st));
    const CvArgs a{d_groups, d_item_off, d_haps, d_job_off, wr.d_pairs, ctx->region.ev.d_records.p, (uint32_t)G, p.alignment_flags};
    float forward_ms = 0.f;
    int launches = 5;
    if (n_jobs) {
        NPH_TRY(nph_score_device_jobs(ctx, (size_t)n_jobs, (size_t)pool, indel_bias, [&]() -> int {
            cv_emit_kernel<<<(unsigned)((items + 127) / 128), 128, 0, st>>>(a, items, (int)p.k, ctx->d_jobs.p, ty, d_alts);
            NPH_CUDA(ctx, cudaGetLastError());
            return NPH_OK;
        }));
        int nl = 0;
        if (nph_last_kernel_ms(ctx, &forward_ms, &nl) == NPH_OK) launches += nl + 1;
        cv_combine_kernel<<<(unsigned)((items + 255) / 256), 256, 0, st>>>(a, items, ctx->d_scores.p, ty, d_alts, d_s);
        NPH_CUDA(ctx, cudaGetLastError());
    }
    cv_keys_kernel<<<(unsigned)((G + kWarps - 1) / kWarps), kThreads, 0, st>>>(a, d_key_rank, d_s, ctx->d_logsum.p, d_flag, d_key, d_ks, d_read_sum,
                                                                              d_key_rc, d_n_keys);
    NPH_CUDA(ctx, cudaGetLastError());
    const GtArgs ga{d_groups, d_blk_off, d_n_keys, d_ks, ctx->d_logsum.p, (uint32_t)G, (int)p.ploidy};
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    launch_genotype<1>(ga, blocks, st, d_partial, d_base);
    NPH_CUDA(ctx, cudaGetLastError());
    cv_best_kernel<<<(unsigned)((G + 255) / 256), 256, 0, st>>>(ga, d_partial, d_best);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    std::vector<float> ks(items), read_sum(n_pairs);
    std::vector<uint32_t> key_rc(n_pairs), n_keys(G);
    std::vector<GtBest> best(G);
    std::vector<double> base(G);
    NPH_CUDA(ctx, cudaMemcpyAsync(ks.data(), d_ks, sizeof(float) * items, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(read_sum.data(), d_read_sum, sizeof(float) * n_pairs, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(key_rc.data(), d_key_rc, sizeof(uint32_t) * n_pairs, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(n_keys.data(), d_n_keys, sizeof(uint32_t) * G, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(best.data(), d_best, sizeof(GtBest) * G, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(base.data(), d_base, sizeof(double) * G, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    float genotype_ms = 0.f;
    NPH_CUDA(ctx, cudaEventElapsedTime(&genotype_ms, ctx->ev0, ctx->ev1));
    cnt.forward_ms = forward_ms;
    cnt.genotype_ms = genotype_ms;
    // simple_call on what the device found, in its loop orders, with the host's exp
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<double> rva;
    for (size_t g = 0; g < G; ++g) {
        const nph_call_group& Gr = groups[g];
        const CvGroup& D = gv[g];
        const uint32_t nk = n_keys[g], nc = Gr.n_haplotypes, nv = Gr.n_variants;
        cnt.n_set_terms += n_sets[g] * nk;
        nph_call_group_result& R = groups_out[g];
        R = nph_call_group_result{};
        R.n_keys = nk;
        R.n_combinations = nc;
        R.best_score = best[g].score;
        R.base_score = base[g];
        if (best[g].idx == kNone) {
            R.status = NPH_CALL_NO_BEST;
        } else if (best[g].score - base[g] < 20) {
            R.status = NPH_CALL_BASE_KEPT;
            R.ploidy = p.ploidy;
        } else {
            R.status = NPH_CALL_CALLED;
            R.ploidy = p.ploidy;
            gt_unrank(best[g].idx, nc, (int)p.ploidy, R.best_set);
        }
        nph_call_variant_result* V = variants_out + Gr.var_first;
        for (uint32_t j = 0; j < R.ploidy; ++j) {
            const nph_call_haplotype& H = haplotypes[Gr.hap_first + R.best_set[j]];
            for (uint32_t i = 0; i < H.n_var; ++i) V[combination_variants[H.var_off + i]].var_count += 1;
        }
        rva.assign((size_t)nk * nv, 0.0);
        const float* kt = ks.data() + D.item_base;
        const float* rs = read_sum.data() + D.pair_first;
        for (uint32_t c = 0; c < nc; ++c) {
            const nph_call_haplotype& H = haplotypes[Gr.hap_first + c];
            for (uint32_t ri = 0; ri < nk; ++ri) {
                const double post = exp((double)kt[(uint64_t)c * D.n_pairs + ri] - (double)rs[ri]);
                for (uint32_t i = 0; i < H.n_var; ++i) {
                    const uint32_t vi = combination_variants[H.var_off + i];
                    rva[(size_t)ri * nv + vi] += post;
                    V[vi].support_sum += post;
                }
            }
        }
        for (uint32_t vi = 0; vi < nv; ++vi) {
            for (uint32_t ri = 0; ri < nk; ++ri) {
                const uint32_t strand = key_rc[D.pair_first + ri] ? 1u : 0u;
                const double pp = rva[(size_t)ri * nv + vi];
                V[vi].strand[0 + strand] += (1 - pp);
                V[vi].strand[2 + strand] += pp;
            }
            V[vi].emit = (p.genotype_all || V[vi].var_count > 0) ? 1u : 0u;
        }
    }
    cnt.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    nph_timing_staged(ctx, forward_ms + genotype_ms, launches + 2);
    if (counts_out) *counts_out = cnt;
    return NPH_OK;
}
