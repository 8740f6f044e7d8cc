// variants.cu — candidate screening of `nanopolish variants` on the device (SURVEY.md section 8f row N2, BASELINE configs[4]).
//
// Replaces, for a whole reference region at once:
//   generate_candidate_single_base_edits      ref: src/nanopolish_call_variants.cpp:288-361
//   AlignmentDB::get_event_subsequences        ref: src/alignment/nanopolish_alignment_db.cpp:172-221
//   AlignmentDB::_find_by_ref_bounds           ref: src/alignment/nanopolish_alignment_db.cpp:688-731
//   score_variant_thresholded                  ref: src/common/nanopolish_variant.cpp:765-799
//   Haplotype::apply_variant on the 22-base test haplotype   ref: src/nanopolish_haplotype.cpp:30-85
// (profile_hmm_score_set with no methylation alternative is profile_hmm_score: K1, unchanged.)
//
// Kernels:
//   var_bounds_kernel   per position: the records whose event alignment bounds the window, in record order, with their
//                       event range (two passes: count, then fill behind a prefix sum)
//   var_ranks_kernel    per (position, sequence, alternative): the k-mer ranks of the base window and of its nine edited versions
//                       (substitution / insertion per base, deletion), both strands — a fixed pool K1's jobs point into; with
//                       methylation types, also of each sequence's methylated copy per type where methylate changes it
//   var_emit_kernel     per round: the jobs of the next reads_per_round reads of every position that still has a live
//                       candidate (base + live candidates per read)
//   var_accumulate_kernel  per position: the sequential `if (fabs(total) < threshold) total += variant - base` over the
//                       round's reads in order (each side profile_hmm_score_set's fold of its sequence and alternatives);
//                       candidates inside the threshold stay live
// The host drives the rounds; per round one read-back (job count) plus the scheduler's summary.  The -q sets (a sequence and its
// methylated copies) use the set description and helpers of meth_dev.cuh and score_sets.cu, shared with list screening and group
// calling; the pool, the masks and the -q tables stay this screen's own.
#include "nph_internal.cuh"
#include "exact_math.cuh"
#include "meth_dev.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace {

constexpr int kSeqs = NPH_SCREEN_SLOTS + 1;      // nine candidates + the base haplotype (slot 9)
constexpr int kBlock = 256;
constexpr int kListCap = 2048;                   // records overlapping one block of positions, kept in shared memory

struct PosState {
    double total[NPH_SCREEN_SLOTS];
    uint32_t valid;       // bit c: candidate c exists (bit 31: the position is screened at all)
    uint32_t alive;       // bit c: |total_c| < threshold so far
    uint32_t done;        // reads consumed
    uint32_t chunk;       // reads of the current round
    unsigned long long ref_rows;   // DP rows the reference's loop scores at this position (2 sequences per candidate and read until exit)
};

struct VarDev {
    int flank, region_start, n_pos, n_ref, k, rpr;
    uint32_t flags, threshold;
    int win;              // 2 * flank + 2
    int stride;           // rank slots per (position, sequence, alternative, strand): the insertion's win + 1 - k + 1 k-mers
    int T;                // methylation types; alternative a = 0 is the nucleotide sequence, a = 1 + t its methylated copy of type t
};

// the copies of sequence seq in a position's mask (bit seq * T + t: its methylated copy of type t differs from it)
__device__ __forceinline__ uint32_t seq_mask(unsigned long long alts, int seq, int T)
{
    return (uint32_t)((alts >> (seq * T)) & ((1ull << T) - 1ull));
}

// pool slot of (position, sequence, alternative): 2 * stride ranks (forward, reverse strand)
__device__ __forceinline__ uint64_t pool_slot(const VarDev& d, int pi, int seq, int a)
{
    return ((uint64_t)pi * kSeqs + (uint64_t)seq) * (uint64_t)(1 + d.T) + (uint64_t)a;
}

// pass 0: counts per position; pass 1: fills pos_reads behind pos_off
template <bool FILL>
__global__ void __launch_bounds__(kBlock) var_bounds_kernel(const VarDev d, const nph_meth_record* __restrict__ records, uint32_t n_records,
                                                            const int32_t* __restrict__ dense, const int32_t* __restrict__ first_valid,
                                                            uint64_t* __restrict__ counts, const uint64_t* __restrict__ pos_off,
                                                            NphWinPair* __restrict__ pos_reads)
{
    __shared__ uint32_t s_list[kListCap];
    __shared__ uint32_t s_n, s_warp[kBlock / 32];
    const int p0 = blockIdx.x * kBlock;
    const int pi = p0 + threadIdx.x;
    // records that can bound a window of this block of positions: their extent meets [first window start, last window end]
    const int lo = d.region_start + p0 - d.flank, hi = d.region_start + min(p0 + kBlock - 1, d.n_pos - 1) + 1 + d.flank;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    bool overflow = false;
    for (uint32_t base = 0; base < n_records; base += kBlock) {
        const uint32_t r = base + threadIdx.x;
        bool take = false;
        if (r < n_records) {
            const nph_meth_record R = records[r];
            take = R.ref_len > 0 && R.ref_start_pos <= hi && R.ref_start_pos + (int)R.ref_len - 1 >= lo;
        }
        // ordered append: record order is the order the reference walks its event records in
        const unsigned m = __ballot_sync(0xffffffffu, take);
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        if (lane == 0) s_warp[w] = __popc(m);
        __syncthreads();
        uint32_t before = 0;
        for (int i = 0; i < w; ++i) before += s_warp[i];
        uint32_t tot = 0;
        for (int i = 0; i < kBlock / 32; ++i) tot += s_warp[i];
        const uint32_t at = s_n + before + __popc(m & ((1u << lane) - 1u));
        if (take) { if (at < kListCap) s_list[at] = r; else overflow = true; }
        __syncthreads();
        if (threadIdx.x == 0) s_n = min(s_n + tot, (uint32_t)kListCap + 1u);
        __syncthreads();
    }
    const bool use_list = !__syncthreads_or(overflow) && s_n <= kListCap;
    if (pi >= d.n_pos) return;
    const int i = d.region_start + pi;
    const int cs = i - d.flank, ce = i + 1 + d.flank;
    const bool pos_ok = cs >= d.region_start && ce <= d.region_start + d.n_ref - 1;       // are_coordinates_valid
    uint64_t cnt = 0;
    NphWinPair* out = FILL ? pos_reads + pos_off[pi] : nullptr;
    if (pos_ok) {
        const uint32_t n_it = use_list ? s_n : n_records;
        for (uint32_t t = 0; t < n_it; ++t) {
            const uint32_t r = use_list ? s_list[t] : t;
            const nph_meth_record R = records[r];
            int e1, e2;
            if (nph_event_subsequence(R, dense + R.ref_off, first_valid[r], cs, ce, e1, e2)) {
                if (FILL) out[cnt] = NphWinPair{r, e1, e2};
                ++cnt;
            }
        }
    }
    if (!FILL) counts[pi] = cnt;
}

// the sequence of slot `seq` at a position: the window (characters) with the slot's edit applied, length returned.
// slots 2j / 2j+1: substitution to / insertion of base j at window offset `flank`; slot 8: deletion of that base; slot 9: base.
__device__ __forceinline__ int edited_window(const uint8_t* __restrict__ w, int win, int flank, int seq, uint8_t* out)
{
    if (seq == NPH_SCREEN_SLOTS) { for (int t = 0; t < win; ++t) out[t] = w[t]; return win; }
    if (seq == 8) {                                              // ref_seq = bases i-1, i; alt = base i-1
        for (int t = 0; t < flank; ++t) out[t] = w[t];
        for (int t = flank + 1; t < win; ++t) out[t - 1] = w[t];
        return win - 1;
    }
    const uint8_t j = (uint8_t)(0x54474341u >> (8 * (seq >> 1)));  // 'A', 'C', 'G', 'T'
    if ((seq & 1) == 0) { for (int t = 0; t < win; ++t) out[t] = w[t]; out[flank] = j; return win; }
    for (int t = 0; t <= flank; ++t) out[t] = w[t];              // alt = base i followed by j
    out[flank + 1] = j;
    for (int t = flank + 1; t < win; ++t) out[t + 1] = w[t];
    return win + 1;
}

// thread per (position, sequence, alternative): ranks of both strands into the pool; the base sequence's nucleotide thread also
// writes candidate validity into the position state, a methylated copy that differs from its sequence sets its bit in alts
__global__ void __launch_bounds__(kBlock) var_ranks_kernel(const VarDev d, const uint8_t* __restrict__ ref, uint32_t* __restrict__ pool,
                                                           PosState* __restrict__ state, const uint64_t* __restrict__ pos_off, const NphSetTypes st,
                                                           unsigned long long* __restrict__ alts)
{
    const long long gid = (long long)blockIdx.x * kBlock + threadIdx.x;
    const int na = 1 + d.T;
    if (gid >= (long long)d.n_pos * kSeqs * na) return;
    const int pi = (int)(gid / (kSeqs * na)), rem = (int)(gid % (kSeqs * na));
    const int seq = rem / na, a = rem % na;
    const int i = d.region_start + pi;
    const int cs = i - d.flank, ce = i + 1 + d.flank;
    const bool pos_ok = cs >= d.region_start && ce <= d.region_start + d.n_ref - 1;
    if (seq == NPH_SCREEN_SLOTS && a == 0) {
        // the base-haplotype thread also initialises the position's state
        PosState st;
        for (int c = 0; c < NPH_SCREEN_SLOTS; ++c) st.total[c] = 0.0;
        st.valid = 0; st.alive = 0; st.done = 0; st.chunk = 0; st.ref_rows = 0;
        if (pos_ok) {
            const uint8_t b = nph_dna_code(ref[cs - d.region_start + d.flank]), bp = nph_dna_code(ref[cs - d.region_start + d.flank - 1]);
            uint32_t v = 0x80000000u;
            for (int j = 0; j < 4; ++j) if (j != b) v |= (1u << (2 * j)) | (1u << (2 * j + 1));   // substitution != ref; insertion "A" -> "AA" is redundant
            if (bp != b) v |= 1u << 8;                                                           // deletion "AA" -> "A" is redundant
            st.valid = v;
            st.alive = (pos_off[pi + 1] > pos_off[pi]) ? (v & 0x1ffu) : 0u;                      // no event sequence: nothing to score, quality 0
        }
        state[pi] = st;
    }
    if (!pos_ok) return;
    // the edited window as characters: Alphabet::methylate matches sites on the string, so an N (code 0 below) never completes one
    uint8_t w[NPH_SCREEN_MAX_WINDOW], sq[NPH_SCREEN_MAX_WINDOW + 1];
    for (int t = 0; t < d.win; ++t) w[t] = ref[cs - d.region_start + t];
    const int L = edited_window(w, d.win, d.flank, seq, sq);
    const int nk = L - d.k + 1;
    uint32_t* fw = pool + pool_slot(d, pi, seq, a) * 2 * d.stride;
    uint32_t* rc = fw + d.stride;
    if (a == 0) {
        for (int t = 0; t < L; ++t) sq[t] = nph_dna_code(sq[t]);
        for (int q = 0; q < nk; ++q) nph_dna_kmer_ranks(sq, q, d.k, fw[q], rc[q]);
        return;
    }
    // methylated copy of type a - 1: fr = ranks of methylate(sq), rv = ranks of Alphabet::reverse_complement of it
    const MethDev& md = st.types[a - 1];
    bool changed = false;
    for (int q = 0; q < L && !changed; ++q) changed = site_at(md, sq, q, L) >= 0;
    if (!changed) return;                                        // generate_methylated_alternatives keeps only a copy that differs
    atomicOr(alts + pi, 1ull << (seq * d.T + a - 1));
    uint8_t* fr = w;
    uint8_t rv[NPH_SCREEN_MAX_WINDOW + 1];
    for (int t = 0; t < L; ++t) {
        uint32_t f, r;
        meth_copy_rank(md, sq, L, t, f, r);
        fr[t] = (uint8_t)f; rv[L - 1 - t] = (uint8_t)r;
    }
    for (int q = 0; q < nk; ++q) {
        uint32_t rf = 0, rr = 0;
        for (int t = 0; t < d.k; ++t) { rf = rf * md.asize + fr[q + t]; rr = rr * md.asize + rv[L - q - d.k + t]; }
        fw[q] = rf; rc[q] = rr;
    }
}

// round bookkeeping, thread per position: how many jobs the position contributes this round (per read: the base sequence's set and
// the set of every live candidate)
__global__ void var_round_count_kernel(const VarDev d, PosState* __restrict__ state, const uint64_t* __restrict__ pos_off, uint64_t* __restrict__ job_cnt,
                                       const unsigned long long* __restrict__ alts)
{
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= d.n_pos) return;
    PosState& st = state[pi];
    const uint32_t n_reads = (uint32_t)(pos_off[pi + 1] - pos_off[pi]);
    uint32_t chunk = 0;
    if (st.alive && st.done < n_reads) chunk = min((uint32_t)d.rpr, n_reads - st.done);
    st.chunk = chunk;
    uint32_t per_read = 1u + __popc(st.alive);
    if (d.T) {
        const unsigned long long am = alts[pi];
        per_read = set_size(seq_mask(am, NPH_SCREEN_SLOTS, d.T));
        for (int c = 0; c < NPH_SCREEN_SLOTS; ++c) if ((st.alive >> c) & 1u) per_read += set_size(seq_mask(am, c, d.T));
    }
    job_cnt[pi] = (uint64_t)chunk * per_read;
}

__global__ void var_emit_kernel(const VarDev d, const PosState* __restrict__ state, const uint64_t* __restrict__ pos_off,
                                const NphWinPair* __restrict__ pos_reads, const nph_meth_record* __restrict__ records,
                                const uint64_t* __restrict__ job_off, nph_hmm_job* __restrict__ jobs, unsigned long long* __restrict__ events,
                                const NphSetTypes ty, const unsigned long long* __restrict__ alts)
{
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long ev = 0;
    if (pi < d.n_pos) {
        const PosState st = state[pi];
        if (st.chunk) {
            const unsigned long long am = d.T ? alts[pi] : 0ull;
            const NphWinPair* rd = pos_reads + pos_off[pi] + st.done;
            nph_hmm_job* out = jobs + job_off[pi];
            for (uint32_t r = 0; r < st.chunk; ++r) {
                const NphWinPair pr = rd[r];
                const nph_meth_record R = records[pr.record];
                nph_hmm_job jb = nph_window_job(R, pr, (uint8_t)d.flags);
                nph_hmm_job* const first = out;
                // the base haplotype first, then the live candidates in slot order
                for (int seq = NPH_SCREEN_SLOTS; ; ) {
                    const int L = seq == NPH_SCREEN_SLOTS ? d.win : (seq == 8 ? d.win - 1 : ((seq & 1) ? d.win + 1 : d.win));
                    jb.n_kmers = (uint32_t)(L - d.k + 1);
                    out = set_jobs(ty, jb, R, pr.record, seq_mask(am, seq, d.T), pool_slot(d, pi, seq, 0) * 2 * d.stride, (uint32_t)d.stride, out);
                    if (seq == NPH_SCREEN_SLOTS) seq = -1;
                    do { ++seq; } while (seq < NPH_SCREEN_SLOTS && !((st.alive >> seq) & 1u));
                    if (seq >= NPH_SCREEN_SLOTS) break;
                }
                ev += (unsigned long long)(out - first) * nph_pair_rows(pr.e1, pr.e2);
            }
        }
    }
    // scored events of the round
    for (int o = 16; o; o >>= 1) ev += __shfl_xor_sync(0xffffffffu, ev, o);
    if ((threadIdx.x & 31) == 0 && ev) atomicAdd(events, ev);
}

__global__ void var_accumulate_kernel(const VarDev d, PosState* __restrict__ state, const uint64_t* __restrict__ job_off,
                                      const float* __restrict__ scores, unsigned int* __restrict__ any_left, const uint64_t* __restrict__ pos_off,
                                      const NphWinPair* __restrict__ pos_reads, unsigned long long* __restrict__ ref_events, const NphSetTypes ty,
                                      const unsigned long long* __restrict__ alts)
{
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= d.n_pos) return;
    PosState st = state[pi];
    if (!st.chunk) return;
    const unsigned long long am = d.T ? alts[pi] : 0ull;
    const float* s = scores + job_off[pi];
    const NphWinPair* rd = pos_reads + pos_off[pi] + st.done;
    const double thr = (double)d.threshold;
    const uint32_t nb = set_size(seq_mask(am, NPH_SCREEN_SLOTS, d.T));
    unsigned long long ref_ev = 0;
    for (uint32_t r = 0; r < st.chunk; ++r) {
        // double base_score = profile_hmm_score_set(...) (a float); a set of one is its score
        const double base_score = (double)nph_score_set_fold(s, nb, ty.pen[nb - 1], ty.tbl);
        s += nb;
        const unsigned long long E = nph_pair_rows(rd[r].e1, rd[r].e2);
        for (int c = 0; c < NPH_SCREEN_SLOTS; ++c) {
            if (!((st.alive >> c) & 1u)) continue;
            const uint32_t nc = set_size(seq_mask(am, c, d.T));
            const double variant_score = (double)nph_score_set_fold(s, nc, ty.pen[nc - 1], ty.tbl);
            s += nc;
            if (fabs(st.total[c]) < thr) {
                st.total[c] = __dadd_rn(st.total[c], __dsub_rn(variant_score, base_score));
                ref_ev += (unsigned long long)(nb + nc) * E;     // what the reference's loop scores here: the base AND the variant set
            }
        }
    }
    if (ref_ev) atomicAdd(ref_events, ref_ev);
    st.ref_rows += ref_ev;
    st.done += st.chunk;
    uint32_t alive = 0;
    for (int c = 0; c < NPH_SCREEN_SLOTS; ++c) if (((st.alive >> c) & 1u) && fabs(st.total[c]) < thr) alive |= 1u << c;
    st.alive = alive;
    st.chunk = 0;
    state[pi] = st;
    if (alive && st.done < (uint32_t)(pos_off[pi + 1] - pos_off[pi])) atomicOr(any_left, 1u);
}

// per position: qualities, read count, reference rows, and into *no_exit the jobs a screening without early exit would have run:
// reads x (n(base) + sum of n(c) over the candidates with a quality), nothing for a position without one
__global__ void var_output_kernel(const VarDev d, const PosState* __restrict__ state, const uint64_t* __restrict__ pos_off,
                                  double* __restrict__ qual, uint32_t* __restrict__ n_reads, unsigned long long* __restrict__ ref_rows,
                                  const unsigned long long* __restrict__ alts, unsigned long long* __restrict__ no_exit)
{
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long full = 0;
    if (pi < d.n_pos) {
        const PosState st = state[pi];
        const unsigned long long am = d.T ? alts[pi] : 0ull;
        const uint32_t nr = (uint32_t)(pos_off[pi + 1] - pos_off[pi]);
        ref_rows[pi] = st.ref_rows;
        uint32_t per_read = set_size(seq_mask(am, NPH_SCREEN_SLOTS, d.T));
        bool any = false;
        for (int c = 0; c < NPH_SCREEN_SLOTS; ++c) {
            const double q = ((st.valid >> c) & 1u) ? st.total[c] : __longlong_as_double(0x7ff8000000000000ll);
            qual[(size_t)pi * NPH_SCREEN_SLOTS + c] = q;
            if (!isnan(q)) { any = true; per_read += set_size(seq_mask(am, c, d.T)); }
        }
        n_reads[pi] = nr;
        if (any) full = (unsigned long long)nr * per_read;
    }
    for (int o = 16; o; o >>= 1) full += __shfl_xor_sync(0xffffffffu, full, o);
    if ((threadIdx.x & 31) == 0 && full) atomicAdd(no_exit, full);
}

int make_dev(nph_ctx* ctx, const nph_screen_params& p, size_t n_ref, uint32_t n_types, VarDev& d)
{
    if (p.flank < 1 || 2 * p.flank + 3 > NPH_SCREEN_MAX_WINDOW) { ctx->last_error = "nph_screen_params: flank outside 1..30"; return NPH_ERR_UNSUPPORTED; }
    if (p.k < 1 || (int)p.k > 2 * p.flank + 1 || p.reads_per_round == 0 || n_ref < 2 || n_ref > 0x7fffffffu) return NPH_ERR_INVALID;
    d.flank = p.flank; d.region_start = p.region_start; d.n_ref = (int)n_ref; d.n_pos = (int)n_ref - 1;
    d.k = (int)p.k; d.rpr = (int)p.reads_per_round; d.flags = p.alignment_flags; d.threshold = p.score_threshold;
    d.win = 2 * p.flank + 2;
    d.stride = d.win + 1 - d.k + 1;
    d.T = (int)n_types;
    return NPH_OK;
}

// the counters of a screening: scored events, the reference's scored events, whether any position has reads left
struct ScreenCounters { unsigned long long events, ref_events; unsigned int any_left; };

// d_state: per-position state | the counters | per position the methylated-alternatives mask
struct ScreenStateLayout { PosState* state; ScreenCounters* counters; unsigned long long* alts; };
ScreenStateLayout screen_state_layout(NphArena& a, size_t n_pos)
{
    ScreenStateLayout l;
    l.state = a.take<PosState>(n_pos);
    l.counters = a.take<ScreenCounters>(1);
    l.alts = a.take<unsigned long long>(n_pos);
    return l;
}

} // namespace

extern "C" int nph_screen_load_methylation(nph_ctx* ctx, const char* ref_bases, size_t n_ref_bases, const int16_t* event_deltas, size_t n_deltas_total,
                                           const int32_t* first_event, const nph_meth_record* records, size_t n_records,
                                           const nph_screen_params* params, double indel_bias,
                                           const nph_screen_methylation* meth, const uint32_t* alt_model_ids)
{
    if (!ctx || !params || !ref_bases || (n_records && (!records || !first_event || (n_deltas_total && !event_deltas)))) return NPH_ERR_INVALID;
    nph_ctx::ScreenState& m = ctx->screen;
    m.loaded = false; m.ran = false;
    if (!meth) return NPH_ERR_INVALID;
    if (!ctx->reads_loaded) return NPH_ERR_STATE;
    VarDev d;
    NPH_TRY(make_dev(ctx, *params, n_ref_bases, meth->n_types, d));
    const uint32_t T = meth->n_types;
    std::vector<MethDev> md;
    NPH_TRY(nph_screen_types(ctx, params->k, *meth, n_records, alt_model_ids, md));
    // records index the event deltas, not the region's reference
    NPH_TRY(nph_event_records_load(ctx, m.ev, ref_bases, n_ref_bases, n_deltas_total, true, event_deltas, first_event, nullptr, 0,
                                   records, n_records, 0x3fffffffu, [&](size_t r, const nph_meth_record& R) {
        return nph_screen_record_check(ctx, params->k, md, alt_model_ids, r, R);
    }));
    m.h_meth.resize(sizeof(MethDev) * T);
    if (T) {
        std::memcpy(m.h_meth.data(), md.data(), m.h_meth.size());
        NPH_TRY(nph_reserve(ctx, m.d_meth, m.h_meth.size()));
        NPH_TRY(nph_reserve(ctx, m.d_alt_models, n_records * T + 1));
        NPH_CUDA(ctx, cudaMemcpyAsync(m.d_meth.p, m.h_meth.data(), m.h_meth.size(), cudaMemcpyHostToDevice, ctx->stream));
        if (n_records) NPH_CUDA(ctx, cudaMemcpyAsync(m.d_alt_models.p, alt_model_ids, sizeof(uint32_t) * n_records * T, cudaMemcpyHostToDevice, ctx->stream));
    }
    m.n_types = T;
    m.params = *params; m.indel_bias = indel_bias;
    m.n_pos = (size_t)d.n_pos;
    m.loaded = true;
    return NPH_OK;
}

extern "C" int nph_screen_load(nph_ctx* ctx, const char* ref_bases, size_t n_ref_bases, const int16_t* event_deltas, size_t n_deltas_total,
                               const int32_t* first_event, const nph_meth_record* records, size_t n_records,
                               const nph_screen_params* params, double indel_bias)
{
    static const nph_screen_methylation none{};
    return nph_screen_load_methylation(ctx, ref_bases, n_ref_bases, event_deltas, n_deltas_total, first_event, records, n_records, params, indel_bias,
                                       &none, nullptr);
}

extern "C" int nph_screen_run(nph_ctx* ctx)
{
    if (!ctx) return NPH_ERR_INVALID;
    nph_ctx::ScreenState& m = ctx->screen;
    if (!m.loaded || !ctx->reads_loaded) return NPH_ERR_STATE;
    m.ran = false; m.n_rounds = 0; m.n_jobs = 0; m.n_scored_events = 0; m.n_jobs_no_exit = 0; m.n_reference_events = 0;
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));
    VarDev d;
    NPH_TRY(make_dev(ctx, m.params, m.ev.n_ref, m.n_types, d));
    const uint32_t n_pos = (uint32_t)m.n_pos, n_rec = (uint32_t)m.ev.n_records;
    const nph_meth_record* records = m.ev.d_records.p;
    cudaStream_t st = ctx->stream;
    const int32_t* dense;
    const int32_t* first_valid;
    NPH_TRY(nph_event_records_expand(ctx, m.ev, &dense, &first_valid));
    // per position: its event sequences
    NPH_TRY(nph_reserve(ctx, m.d_pos_off, (size_t)n_pos + 1));
    uint64_t* counts; uint64_t* job_off; uint64_t* scan_scratch;     // per-position counts (reads, then each round's jobs) and job offsets
    NPH_TRY(nph_carve(ctx, m.d_job_off, [&](NphArena& a) {
        counts = a.take<uint64_t>(n_pos);
        job_off = a.take<uint64_t>((size_t)n_pos + 1);
        scan_scratch = a.take<uint64_t>(nph_scan_scratch(n_pos));
    }));
    const int pgrid = (int)((n_pos + kBlock - 1) / kBlock);
    var_bounds_kernel<false><<<pgrid, kBlock, 0, st>>>(d, records, n_rec, dense, first_valid, counts, nullptr, nullptr);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_TRY(nph_scan_exclusive(ctx, counts, n_pos, m.d_pos_off.p, scan_scratch));
    uint64_t n_pos_reads = 0;
    NPH_CUDA(ctx, cudaMemcpyAsync(&n_pos_reads, m.d_pos_off.p + n_pos, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    NPH_TRY(nph_reserve(ctx, m.d_pos_reads, sizeof(NphWinPair) * ((size_t)n_pos_reads + 1)));
    NphWinPair* pos_reads = reinterpret_cast<NphWinPair*>(m.d_pos_reads.p);
    var_bounds_kernel<true><<<pgrid, kBlock, 0, st>>>(d, records, n_rec, dense, first_valid, nullptr, m.d_pos_off.p, pos_reads);
    NPH_CUDA(ctx, cudaGetLastError());
    // rank pool (K1's d_ranks for this batch: per position, sequence and alternative both strands) and position state
    const size_t pool = (size_t)n_pos * kSeqs * (size_t)(1 + d.T) * 2 * (size_t)d.stride;
    NPH_TRY(nph_reserve(ctx, ctx->d_ranks, pool));
    ScreenStateLayout sl;
    NPH_TRY(nph_carve(ctx, m.d_state, [&](NphArena& a) { sl = screen_state_layout(a, n_pos); }));
    PosState* state = sl.state;
    const NphSetTypes ty = nph_set_types(reinterpret_cast<const MethDev*>(m.d_meth.p), m.d_alt_models.p, ctx->d_logsum.p, d.T);
    NPH_CUDA(ctx, cudaMemsetAsync(ctx->d_ranks.p, 0, sizeof(uint32_t) * pool, st));
    if (d.T) NPH_CUDA(ctx, cudaMemsetAsync(sl.alts, 0, sizeof(unsigned long long) * (size_t)n_pos, st));
    const long long n_thr = (long long)n_pos * kSeqs * (1 + d.T);
    var_ranks_kernel<<<(unsigned)((n_thr + kBlock - 1) / kBlock), kBlock, 0, st>>>(d, m.ev.d_ref.p, ctx->d_ranks.p, state, m.d_pos_off.p, ty, sl.alts);
    NPH_CUDA(ctx, cudaGetLastError());
    ScreenCounters* ctr = sl.counters;
    NPH_CUDA(ctx, cudaMemsetAsync(ctr, 0, sizeof(ScreenCounters), st));
    float kernel_ms_total = 0.f;
    int launches_total = 0;
    for (;;) {
        var_round_count_kernel<<<pgrid, kBlock, 0, st>>>(d, state, m.d_pos_off.p, counts, sl.alts);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_scan_exclusive(ctx, counts, n_pos, job_off, scan_scratch));
        uint64_t n_jobs = 0;
        NPH_CUDA(ctx, cudaMemcpyAsync(&n_jobs, job_off + n_pos, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));                         // read-back: the round's job count
        if (n_jobs == 0) break;
        // var_emit_kernel writes the round's jobs over the pool var_ranks_kernel wrote; the schedule is one more read-back
        NPH_TRY(nph_score_device_jobs(ctx, (size_t)n_jobs, pool, m.indel_bias, [&]() -> int {
            var_emit_kernel<<<pgrid, kBlock, 0, st>>>(d, state, m.d_pos_off.p, pos_reads, records, job_off, ctx->d_jobs.p, &ctr->events, ty, sl.alts);
            NPH_CUDA(ctx, cudaGetLastError());
            return NPH_OK;
        }));
        NPH_CUDA(ctx, cudaMemsetAsync(&ctr->any_left, 0, sizeof(unsigned int), st));
        var_accumulate_kernel<<<pgrid, kBlock, 0, st>>>(d, state, job_off, ctx->d_scores.p, &ctr->any_left, m.d_pos_off.p, pos_reads, &ctr->ref_events, ty, sl.alts);
        NPH_CUDA(ctx, cudaGetLastError());
        float ms = 0.f; int nl = 0;
        if (nph_last_kernel_ms(ctx, &ms, &nl) == NPH_OK) { kernel_ms_total += ms; launches_total += nl + 6; }
        m.n_rounds += 1;
        m.n_jobs += n_jobs;
    }
    ScreenCounters h{};
    NPH_CUDA(ctx, cudaMemcpyAsync(&h, ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    m.n_scored_events = h.events;
    m.n_reference_events = h.ref_events;
    nph_timing_staged(ctx, kernel_ms_total, launches_total);
    m.ran = true;
    return NPH_OK;
}

extern "C" int nph_screen_counts(nph_ctx* ctx, uint32_t* n_rounds_out, uint64_t* n_jobs_out, uint64_t* n_scored_events_out, uint64_t* n_jobs_without_exit_out,
                                 uint64_t* n_reference_events_out)
{
    if (!ctx) return NPH_ERR_INVALID;
    nph_ctx::ScreenState& m = ctx->screen;
    if (!m.ran) return NPH_ERR_STATE;
    if (n_rounds_out) *n_rounds_out = m.n_rounds;
    if (n_jobs_out) *n_jobs_out = m.n_jobs;
    if (n_scored_events_out) *n_scored_events_out = m.n_scored_events;
    if (n_jobs_without_exit_out) *n_jobs_without_exit_out = m.n_jobs_no_exit;
    if (n_reference_events_out) *n_reference_events_out = m.n_reference_events;
    return NPH_OK;
}

extern "C" int nph_screen_fetch(nph_ctx* ctx, double* qualities_out, uint32_t* n_reads_out, uint64_t* reference_rows_out)
{
    if (!ctx || !qualities_out) return NPH_ERR_INVALID;
    nph_ctx::ScreenState& m = ctx->screen;
    if (!m.ran) return NPH_ERR_STATE;
    VarDev d;
    NPH_TRY(make_dev(ctx, m.params, m.ev.n_ref, m.n_types, d));
    const uint32_t n_pos = (uint32_t)m.n_pos;
    // outputs staged in the (now idle) prologue buffer: per position the slot qualities, reference rows and read count
    const size_t b_q = sizeof(double) * NPH_SCREEN_SLOTS * (size_t)n_pos, b_n = sizeof(uint32_t) * (size_t)n_pos;
    const size_t b_r = sizeof(unsigned long long) * (size_t)n_pos;
    double* d_q; unsigned long long* d_r; uint32_t* d_n; unsigned long long* d_full;
    NPH_TRY(nph_carve(ctx, ctx->d_prep, [&](NphArena& a) {
        d_q = a.take<double>(NPH_SCREEN_SLOTS * (size_t)n_pos);
        d_r = a.take<unsigned long long>(n_pos);
        d_n = a.take<uint32_t>(n_pos);
        d_full = a.take<unsigned long long>(1);
    }));
    NphArena sa{m.d_state.p};
    const ScreenStateLayout sl = screen_state_layout(sa, n_pos);
    NPH_CUDA(ctx, cudaMemsetAsync(d_full, 0, sizeof(unsigned long long), ctx->stream));
    var_output_kernel<<<(n_pos + kBlock - 1) / kBlock, kBlock, 0, ctx->stream>>>(d, sl.state, m.d_pos_off.p, d_q, d_n, d_r, sl.alts, d_full);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaMemcpyAsync(qualities_out, d_q, b_q, cudaMemcpyDeviceToHost, ctx->stream));
    if (n_reads_out) NPH_CUDA(ctx, cudaMemcpyAsync(n_reads_out, d_n, b_n, cudaMemcpyDeviceToHost, ctx->stream));
    if (reference_rows_out) NPH_CUDA(ctx, cudaMemcpyAsync(reference_rows_out, d_r, b_r, cudaMemcpyDeviceToHost, ctx->stream));
    unsigned long long full = 0;
    NPH_CUDA(ctx, cudaMemcpyAsync(&full, d_full, sizeof(full), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    m.n_jobs_no_exit = full;
    return NPH_OK;
}

extern "C" int nph_screen_edits_batch(nph_ctx* ctx,
                                      const nph_read* reads, size_t n_reads,
                                      const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                      const char* ref_bases, size_t n_ref_bases,
                                      const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                      const nph_meth_record* records, size_t n_records,
                                      const nph_screen_params* params, double indel_bias,
                                      double* qualities_out, uint32_t* n_reads_out, uint64_t* n_scored_events_out)
{
    if (!ctx) return NPH_ERR_INVALID;
    NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
    NPH_TRY(nph_screen_load(ctx, ref_bases, n_ref_bases, event_deltas, n_deltas_total, first_event, records, n_records, params, indel_bias));
    NPH_TRY(nph_screen_run(ctx));
    NPH_TRY(nph_screen_fetch(ctx, qualities_out, n_reads_out, nullptr));
    if (n_scored_events_out) *n_scored_events_out = ctx->screen.n_scored_events;
    return NPH_OK;
}

extern "C" int nph_screen_edits_batch_methylation(nph_ctx* ctx,
                                                  const nph_read* reads, size_t n_reads,
                                                  const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                                  const char* ref_bases, size_t n_ref_bases,
                                                  const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                                  const nph_meth_record* records, size_t n_records,
                                                  const nph_screen_params* params, double indel_bias,
                                                  const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                                                  double* qualities_out, uint32_t* n_reads_out, uint64_t* n_scored_events_out)
{
    if (!ctx) return NPH_ERR_INVALID;
    NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
    NPH_TRY(nph_screen_load_methylation(ctx, ref_bases, n_ref_bases, event_deltas, n_deltas_total, first_event, records, n_records, params, indel_bias,
                                        meth, alt_model_ids));
    NPH_TRY(nph_screen_run(ctx));
    NPH_TRY(nph_screen_fetch(ctx, qualities_out, n_reads_out, nullptr));
    if (n_scored_events_out) *n_scored_events_out = ctx->screen.n_scored_events;
    return NPH_OK;
}
