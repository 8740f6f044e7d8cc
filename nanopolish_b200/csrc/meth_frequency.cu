// meth_frequency.cu — the per-site methylation frequency table of call-methylation's output, accumulated on the device.
//
// What scripts/calculate_methylation_frequency.py of the reference computes from methylation_calls.tsv, without the TSV:
// every row of every folded batch (the rows nph_methylation_tsv would write, in its order) is
//   skipped when abs(llr) < call_threshold * num_motifs, llr = Python's float() of the row's "%.2lf" text,
//   else counted at the key (chromosome, start, end) — or, with split_groups and num_motifs > 1, once per "CG" of its
//   sequence column (overlapping matches count) at (chromosome, start + pos - first_pos, same), group size 1,
//   and a key keeps the group size and sequence of the first row that created it, in input order.
// The table is the script's output: a header, then one row per key in the order Python sorts (str, int, int) tuples.
//
// Exactness: the "%.2lf" text of a row is the integer D = fixed_of<2>(llr_m - llr_u) (tsv_format.cuh, the same arithmetic the
// row writer prints), so Python's float() of it is the correctly rounded D / 100, which (double)D / 100.0 is as long as D is
// a double (D < 2^53; larger values are refused).  is_methylated (llr > 0) is D > 0 with a '+' sign: "-0.00" is not.  Counts
// are 64-bit integer atomics and the first row of a key is an atomicMin over (batch, row) ordinals, so the table does not
// depend on thread order.  The frequency is the double m / n, printed by fixed_of<3> — Python's "%.3f" of that double.
//
// Per fold (nph_methfreq_add): validate (every row's numbers, the packing limits, the batch's call and byte counts; one
// read-back) -> grow the table / byte pool if needed -> insert (counts, first ordinal) -> claim (the first row's group size
// and sequence bytes).  A refused batch leaves the accumulator as it was.
// Per table (nph_methfreq_tsv): compact the occupied slots (nph_scan_exclusive), key = (rank of the contig's name, start,
// span), cub radix sort, row lengths -> scan -> rows (one read-back between), one D2H copy.
#include "nph_internal.cuh"
#include "meth_dev.cuh"
#include "tsv_format.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

namespace {

constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

// key = contig (20 bits) | start (31 bits) | end - start (13 bits); the sort key is the same with the contig's name rank in
// place of its id, so (rank, start, span) order is (name, start, end) order.
constexpr int kSpanBits = 13, kStartBits = 31, kContigShift = kSpanBits + kStartBits;
constexpr uint64_t kMaxContigs = 1ull << (64 - kContigShift);
constexpr uint64_t kLowMask = (1ull << kContigShift) - 1;
// an empty slot: no key has every bit set (start = 2^31 - 1 leaves no room for a span, end being an int32 too)
constexpr uint64_t kEmpty = ~0ull;
// ordinal = batch << 40 | site index within the batch
constexpr int kRowBits = 40;
constexpr uint32_t kSplitSeq = 0xffffffffu;     // info's sequence length of a split key: "split-group"
constexpr double kMaxLoad = 0.5;
constexpr size_t kMinSlots = 1024;

// refusal bits of a batch
constexpr int kRefuseNumber = 1;                // non-finite, |v| >= 2^52, or a printed llr of 2^53 / 100 or more
constexpr int kRefuseSeq = 2;                   // the sequence column would start before the record's reference
constexpr int kRefusePacking = 4;               // a start or span outside the key's fields

struct FreqSummary {
    // the accumulator (kept across folds)
    unsigned long long n_keys, pool_used;
    // the batch being folded (cleared by each fold)
    unsigned long long calls, ambiguous, seq_bytes;
    int refused;
};

struct FreqTable {
    uint64_t* key;
    unsigned long long* first;     // smallest ordinal that reached the key
    unsigned long long* called;
    unsigned long long* methylated;
    uint64_t* seq_off;             // into the byte pool
    uint64_t* info;                // group size << 32 | sequence length (kSplitSeq: split key)
    uint64_t mask;                 // slots - 1
};
FreqTable table_layout(NphArena& a, size_t slots)
{
    FreqTable t;
    t.key = a.take<uint64_t>(slots);
    t.first = a.take<unsigned long long>(slots);
    t.called = a.take<unsigned long long>(slots);
    t.methylated = a.take<unsigned long long>(slots);
    t.seq_off = a.take<uint64_t>(slots);
    t.info = a.take<uint64_t>(slots);
    t.mask = slots - 1;
    return t;
}
FreqTable table_of(const nph_ctx::FreqState& f) { NphArena a{f.d_table.p}; return table_layout(a, f.slots); }

__device__ __forceinline__ uint64_t slot_hash(uint64_t x)
{
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// the slot holding key, created if absent (*created: this thread created it)
__device__ __forceinline__ uint64_t slot_insert(const FreqTable& t, uint64_t key, bool* created)
{
    for (uint64_t s = slot_hash(key) & t.mask;; s = (s + 1) & t.mask) {
        const unsigned long long k = t.key[s];
        if (k == key) { *created = false; return s; }
        if (k == kEmpty) {
            const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(t.key + s), kEmpty, (unsigned long long)key);
            if (prev == kEmpty) { *created = true; return s; }
            if (prev == key) { *created = false; return s; }
        }
    }
}

__device__ __forceinline__ uint64_t slot_find(const FreqTable& t, uint64_t key)
{
    uint64_t s = slot_hash(key) & t.mask;
    while (t.key[s] != key) s = (s + 1) & t.mask;
    return s;
}

struct FoldArgs {
    const nph_meth_site* sites;
    const nph_meth_record* records;
    const uint8_t* ref;
    uint64_t n_sites;
    uint32_t k;
    double threshold;
    bool split;
    uint64_t contig;               // contig id << kContigShift
    unsigned long long ord0;       // batch << kRowBits
    FreqTable t;
    FreqSummary* sum;
    uint8_t* pool;
};

// one row as the script reads it
struct FreqRow {
    bool call, meth, split;
    int refused;
    uint32_t n_motif, seq_len;
    int32_t start, end;
    const uint8_t* seq;
};

__device__ __forceinline__ FreqRow freq_row(const FoldArgs& a, uint64_t i)
{
    const nph_meth_site ms = a.sites[i];
    const nph_meth_record R = a.records[ms.record];
    const nph_tsv::RowNums r = nph_tsv::row_numbers(ms, R, a.k);
    FreqRow f;
    f.refused = 0;
    if (!(r.diff.ok && r.m.ok && r.u.ok) || r.diff.q >= (1ull << 53)) f.refused |= kRefuseNumber;
    if (!r.seq_ok) f.refused |= kRefuseSeq;
    const double abs_llr = __ddiv_rn(__ull2double_rn(r.diff.q), 100.0);
    f.call = !(abs_llr < __dmul_rn(a.threshold, __uint2double_rn(ms.n_motif)));
    f.meth = !r.diff.neg && r.diff.q > 0;
    f.split = a.split && ms.n_motif > 1;
    f.n_motif = ms.n_motif;
    f.start = ms.start_position; f.end = ms.end_position;
    f.seq = a.ref + R.ref_off + r.seq_b;
    f.seq_len = r.seq_len;
    return f;
}

__device__ __forceinline__ bool key_fits(int64_t start, int64_t end)
{
    return start >= 0 && end >= start && end - start < (1 << kSpanBits) && end <= INT32_MAX;
}

__device__ __forceinline__ uint64_t pack(const FoldArgs& a, int64_t start, int64_t end)
{
    return a.contig | ((uint64_t)start << kSpanBits) | (uint64_t)(end - start);
}

__device__ __forceinline__ bool is_cg(const uint8_t* s, uint32_t i) { return s[i] == 'C' && s[i + 1] == 'G'; }

// every call of row r: f(start, end, n, with_seq) — the row's own key, or with split each "CG" of its sequence column
template <typename F>
__device__ __forceinline__ void for_each_call(const FreqRow& r, F&& f)
{
    if (!r.call) return;
    if (!r.split) { f((int64_t)r.start, (int64_t)r.end, r.n_motif, true); return; }
    int64_t first = -1;
    for (uint32_t p = 0; p + 1 < r.seq_len; ++p) {
        if (!is_cg(r.seq, p)) continue;
        if (first < 0) first = p;
        const int64_t s = (int64_t)r.start + ((int64_t)p - first);
        f(s, s, 1u, false);
    }
}

// pass 1: refusals, packing limits and the batch's counts (calls, skipped rows, sequence bytes a new key could need)
__global__ void __launch_bounds__(kThreads) freq_validate_kernel(const FoldArgs a)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t n_iter = (a.n_sites + stride - 1) / stride;          // uniform across the warp: the sums below are warp-wide
    int refused = 0;
    uint32_t calls = 0, ambiguous = 0;
    unsigned long long bytes = 0;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t i = it * stride + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
        if (i >= a.n_sites) continue;
        const FreqRow r = freq_row(a, i);
        refused |= r.refused;
        if (r.refused) continue;
        if (!r.call) { ++ambiguous; continue; }
        for_each_call(r, [&](int64_t start, int64_t end, uint32_t, bool with_seq) {
            if (!key_fits(start, end)) refused |= kRefusePacking;
            ++calls;
            if (with_seq) bytes += r.seq_len;
        });
    }
    refused = __reduce_or_sync(kFull, (unsigned)refused);
    calls = __reduce_add_sync(kFull, calls);
    ambiguous = __reduce_add_sync(kFull, ambiguous);
    for (int o = 16; o > 0; o >>= 1) bytes += __shfl_down_sync(kFull, bytes, o);
    if ((threadIdx.x & 31) == 0) {
        if (refused) atomicOr(&a.sum->refused, refused);
        if (calls) atomicAdd(&a.sum->calls, (unsigned long long)calls);
        if (ambiguous) atomicAdd(&a.sum->ambiguous, (unsigned long long)ambiguous);
        if (bytes) atomicAdd(&a.sum->seq_bytes, bytes);
    }
}

// pass 2: every call adds its counts and offers its ordinal
__global__ void __launch_bounds__(kThreads) freq_insert_kernel(const FoldArgs a)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < a.n_sites; i += (uint64_t)gridDim.x * blockDim.x) {
        const FreqRow r = freq_row(a, i);
        const unsigned long long ord = a.ord0 | i;
        for_each_call(r, [&](int64_t start, int64_t end, uint32_t n, bool) {
            bool created;
            const uint64_t s = slot_insert(a.t, pack(a, start, end), &created);
            if (created) atomicAdd(&a.sum->n_keys, 1ull);
            atomicAdd(a.t.called + s, (unsigned long long)n);
            if (r.meth) atomicAdd(a.t.methylated + s, (unsigned long long)n);
            atomicMin(a.t.first + s, ord);
        });
    }
}

// pass 3: the call that holds a key's smallest ordinal stores its group size and sequence (a key created by an earlier batch
// has a smaller ordinal than any call of this one)
__global__ void __launch_bounds__(kThreads) freq_claim_kernel(const FoldArgs a)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < a.n_sites; i += (uint64_t)gridDim.x * blockDim.x) {
        const FreqRow r = freq_row(a, i);
        const unsigned long long ord = a.ord0 | i;
        for_each_call(r, [&](int64_t start, int64_t end, uint32_t n, bool with_seq) {
            const uint64_t s = slot_find(a.t, pack(a, start, end));
            if (a.t.first[s] != ord) return;
            a.t.info[s] = (uint64_t)n << 32 | (with_seq ? r.seq_len : kSplitSeq);
            if (!with_seq) return;
            const unsigned long long off = atomicAdd(&a.sum->pool_used, (unsigned long long)r.seq_len);
            a.t.seq_off[s] = off;
            for (uint32_t b = 0; b < r.seq_len; ++b) a.pool[off + b] = r.seq[b];
        });
    }
}

__global__ void __launch_bounds__(kThreads) freq_rehash_kernel(const FreqTable from, const FreqTable to)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= from.mask; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t key = from.key[i];
        if (key == kEmpty) continue;
        bool created;
        const uint64_t s = slot_insert(to, key, &created);
        to.first[s] = from.first[i]; to.called[s] = from.called[i]; to.methylated[s] = from.methylated[i];
        to.seq_off[s] = from.seq_off[i]; to.info[s] = from.info[i];
    }
}

int grid_for(const nph_ctx* ctx, uint64_t n) { return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, (uint64_t)ctx->sm_count * 8)); }

// a fresh table of `slots` slots in buf: keys and ordinals all ones, counts zero
int table_alloc(nph_ctx* ctx, DevBuf<uint8_t>& buf, size_t slots, FreqTable* t)
{
    NPH_TRY(nph_carve(ctx, buf, [&](NphArena& a) { *t = table_layout(a, slots); }));
    const size_t ones = (size_t)(reinterpret_cast<uint8_t*>(t->called) - reinterpret_cast<uint8_t*>(t->key));
    const size_t zeros = nph_layout_bytes([&](NphArena& a) { table_layout(a, slots); }) - ones;
    NPH_CUDA(ctx, cudaMemsetAsync(t->key, 0xff, ones, ctx->stream));
    NPH_CUDA(ctx, cudaMemsetAsync(t->called, 0, zeros, ctx->stream));
    return NPH_OK;
}

FreqSummary* summary_of(nph_ctx::FreqState& f) { return reinterpret_cast<FreqSummary*>(f.d_summary.p); }

// the accumulator exists (empty table, zero counters)
int freq_init(nph_ctx* ctx, nph_ctx::FreqState& f)
{
    if (f.slots) return NPH_OK;
    NPH_TRY(nph_reserve(ctx, f.d_summary, sizeof(FreqSummary)));
    NPH_CUDA(ctx, cudaMemsetAsync(f.d_summary.p, 0, sizeof(FreqSummary), ctx->stream));
    FreqTable t;
    NPH_TRY(table_alloc(ctx, f.d_table, kMinSlots, &t));
    f.slots = kMinSlots;
    f.n_batches = 0; f.n_calls = 0; f.n_ambiguous = 0;
    return NPH_OK;
}

} // namespace

extern "C" int nph_methfreq_reset(nph_ctx* ctx, const nph_methfreq_params* params)
{
    if (!ctx) return NPH_ERR_INVALID;
    nph_ctx::FreqState& f = ctx->freq;
    f.params = params ? *params : nph_methfreq_params{2.0, 0, 0};
    f.slots = 0;                         // the next fold (or table) starts from an empty accumulator
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));
    return freq_init(ctx, f);
}

extern "C" int nph_methfreq_add(nph_ctx* ctx, uint32_t contig_id)
{
    if (!ctx) return NPH_ERR_INVALID;
    const nph_ctx::MethState& m = ctx->meth;
    nph_ctx::FreqState& f = ctx->freq;
    if (!m.ran) return NPH_ERR_STATE;
    if (contig_id >= kMaxContigs) { ctx->last_error = "contig_id must be below 2^20"; return NPH_ERR_INVALID; }
    if (f.n_batches + 1 >= (1u << (64 - kRowBits)) || m.n_sites >= (1ull << kRowBits)) {
        ctx->last_error = "more than 2^24 folded batches or 2^40 sites in one batch";
        return NPH_ERR_UNSUPPORTED;
    }
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));
    NPH_TRY(freq_init(ctx, f));
    FreqSummary* d_sum = summary_of(f);
    FoldArgs a{m.d_sites.p, m.ev.d_records.p, m.ev.d_ref.p, m.ev.n_records ? m.n_sites : 0, m.params.k, f.params.call_threshold,
               f.params.split_groups != 0, (uint64_t)contig_id << kContigShift, (unsigned long long)f.n_batches << kRowBits,
               table_of(f), d_sum, nullptr};
    if (a.n_sites == 0) { f.n_batches += 1; return NPH_OK; }
    const int grid = grid_for(ctx, a.n_sites);
    NPH_CUDA(ctx, cudaMemsetAsync(&d_sum->calls, 0, sizeof(FreqSummary) - offsetof(FreqSummary, calls), ctx->stream));
    freq_validate_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    NPH_CUDA(ctx, cudaGetLastError());
    FreqSummary h{};
    NPH_CUDA(ctx, cudaMemcpyAsync(&h, d_sum, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));            // the fold's one read-back
    if (h.refused & kRefuseSeq) {
        ctx->last_error = nph_tsv::kSeqRefused;
        return NPH_ERR_INVALID;
    }
    if (h.refused) {
        ctx->last_error = (h.refused & kRefuseNumber)
            ? "a log-likelihood is not finite, beyond 2^52, or its printed ratio is 2^53 / 100 or more: the batch was not folded"
            : "a site's start is negative or its span reaches 2^13: the batch was not folded";
        return NPH_ERR_UNSUPPORTED;
    }
    // room for every call of the batch as a new key at the table's load limit, and for every new key's sequence
    const uint64_t need = h.n_keys + h.calls;
    if ((double)need > kMaxLoad * (double)f.slots) {
        size_t slots = f.slots;
        while ((double)need > kMaxLoad * (double)slots) slots *= 2;
        if (slots > (1ull << 31)) { ctx->last_error = "the frequency table would exceed 2^31 slots"; return NPH_ERR_UNSUPPORTED; }
        DevBuf<uint8_t> grown;
        FreqTable t;
        NPH_TRY(table_alloc(ctx, grown, slots, &t));
        freq_rehash_kernel<<<grid_for(ctx, f.slots), kThreads, 0, ctx->stream>>>(a.t, t);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));        // the old table is freed below
        f.d_table = std::move(grown);
        f.slots = slots;
        a.t = t;
    }
    if (h.pool_used + h.seq_bytes > f.d_pool.cap) {
        DevBuf<uint8_t> grown;
        NPH_TRY(nph_reserve(ctx, grown, (size_t)(2 * (h.pool_used + h.seq_bytes))));
        if (h.pool_used) NPH_CUDA(ctx, cudaMemcpyAsync(grown.p, f.d_pool.p, (size_t)h.pool_used, cudaMemcpyDeviceToDevice, ctx->stream));
        NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        f.d_pool = std::move(grown);
    }
    a.pool = f.d_pool.p;
    freq_insert_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    NPH_CUDA(ctx, cudaGetLastError());
    freq_claim_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    NPH_CUDA(ctx, cudaGetLastError());
    f.n_batches += 1;
    f.n_calls += h.calls;
    f.n_ambiguous += h.ambiguous;
    return NPH_OK;
}

extern "C" int nph_methfreq_counts(nph_ctx* ctx, uint64_t* n_keys_out, uint64_t* n_calls_out, uint64_t* n_ambiguous_out)
{
    if (!ctx) return NPH_ERR_INVALID;
    nph_ctx::FreqState& f = ctx->freq;
    unsigned long long n_keys = 0;
    if (f.slots) {
        NPH_CUDA(ctx, cudaSetDevice(ctx->device));
        NPH_CUDA(ctx, cudaMemcpyAsync(&n_keys, &summary_of(f)->n_keys, sizeof(n_keys), cudaMemcpyDeviceToHost, ctx->stream));
        NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (n_keys_out) *n_keys_out = n_keys;
    if (n_calls_out) *n_calls_out = f.slots ? f.n_calls : 0;
    if (n_ambiguous_out) *n_ambiguous_out = f.slots ? f.n_ambiguous : 0;
    return NPH_OK;
}

// ---- the table -------------------------------------------------------------------------------------------------------
namespace {

const char kHeader[] = "chromosome\tstart\tend\tnum_motifs_in_group\tcalled_sites\tcalled_sites_methylated\tmethylated_frequency\tgroup_sequence\n";
#define NPH_SPLIT_GROUP "split-group"

__global__ void __launch_bounds__(kThreads) freq_occupied_kernel(const FreqTable t, uint64_t* occupied)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= t.mask; i += (uint64_t)gridDim.x * blockDim.x)
        occupied[i] = t.key[i] != kEmpty ? 1u : 0u;
}

// occupied slot i -> position off[i]: sort key (name rank, start, span) and the slot
__global__ void __launch_bounds__(kThreads) freq_scatter_kernel(const FreqTable t, const uint64_t* off, const uint32_t* rank, uint32_t n_contigs,
                                                                uint64_t* sort_key, uint32_t* sort_slot, int* missing)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= t.mask; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t key = t.key[i];
        if (key == kEmpty) continue;
        const uint64_t contig = key >> kContigShift;
        if (contig >= n_contigs) { *missing = 1; continue; }
        sort_key[off[i]] = (uint64_t)rank[contig] << kContigShift | (key & kLowMask);
        sort_slot[off[i]] = (uint32_t)i;
    }
}

struct RowArgs {
    FreqTable t;
    const uint64_t* sort_key;
    const uint32_t* sort_slot;
    const char* names; const uint32_t* name_off;        // in rank order
    const uint8_t* pool;
    uint64_t n_rows;
    uint64_t* row_bytes;
    const uint64_t* row_off;
    char* out;
};

// pass 1 (WRITE = false): bytes per row; pass 2: the row at row_off[j]
template <bool WRITE>
__global__ void __launch_bounds__(kThreads) freq_rows_kernel(const RowArgs a)
{
    for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < a.n_rows; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t sk = a.sort_key[j];
        const uint32_t s = a.sort_slot[j];
        const uint32_t rank = (uint32_t)(sk >> kContigShift);
        const int start = (int)((sk & kLowMask) >> kSpanBits);
        const int end = start + (int)(sk & ((1u << kSpanBits) - 1));
        const uint64_t n = a.t.called[s], m = a.t.methylated[s], info = a.t.info[s];
        const uint32_t group = (uint32_t)(info >> 32), seq_len = (uint32_t)info;
        // Python: float(m) / n, both converted to double first
        const nph_tsv::Fixed freq = nph_tsv::fixed_of<3>(__ddiv_rn(__ull2double_rn(m), __ull2double_rn(n)));
        const uint32_t nb = a.name_off[rank], name_len = a.name_off[rank + 1] - nb;
        const uint32_t shown = seq_len == kSplitSeq ? (uint32_t)(sizeof(NPH_SPLIT_GROUP) - 1) : seq_len;
        if (!WRITE) {
            a.row_bytes[j] = name_len + 1 + nph_tsv::int_len(start) + 1 + nph_tsv::int_len(end) + 1 + nph_tsv::ndigits(group) + 1 +
                             nph_tsv::ndigits(n) + 1 + nph_tsv::ndigits(m) + 1 + nph_tsv::fixed_len<3>(freq) + 1 + shown + 1;
            continue;
        }
        char* o = a.out + a.row_off[j];
        for (uint32_t i = 0; i < name_len; ++i) *o++ = a.names[nb + i];
        *o++ = '\t'; o = nph_tsv::put_int(o, start);
        *o++ = '\t'; o = nph_tsv::put_int(o, end);
        *o++ = '\t'; o = nph_tsv::put_u64(o, group);
        *o++ = '\t'; o = nph_tsv::put_u64(o, n);
        *o++ = '\t'; o = nph_tsv::put_u64(o, m);
        *o++ = '\t'; o = nph_tsv::put_fixed<3>(o, freq);
        *o++ = '\t';
        if (seq_len == kSplitSeq) { for (uint32_t i = 0; i < shown; ++i) *o++ = NPH_SPLIT_GROUP[i]; }
        else { const uint8_t* q = a.pool + a.t.seq_off[s]; for (uint32_t i = 0; i < seq_len; ++i) *o++ = (char)q[i]; }
        *o++ = '\n';
    }
}

} // namespace

extern "C" int nph_methfreq_tsv(nph_ctx* ctx, const char* names, const uint32_t* name_off, uint32_t n_contigs,
                                char* out, size_t cap, uint64_t* n_bytes_out)
{
    if (!ctx || !n_bytes_out) return NPH_ERR_INVALID;
    *n_bytes_out = 0;
    if (n_contigs && (!names || !name_off)) return NPH_ERR_INVALID;
    if (n_contigs > kMaxContigs) { ctx->last_error = "more than 2^20 contig names"; return NPH_ERR_INVALID; }
    nph_ctx::FreqState& f = ctx->freq;
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));
    NPH_TRY(freq_init(ctx, f));
    // the names in Python's string order (bytewise for UTF-8), each contig id's rank in it
    std::vector<uint32_t> order(n_contigs), rank(n_contigs + 1, 0);
    for (uint32_t c = 0; c < n_contigs; ++c) {
        if (name_off[c] > name_off[c + 1]) { ctx->last_error = "name_off must ascend"; return NPH_ERR_INVALID; }
        order[c] = c;
    }
    auto name = [&](uint32_t c) { return std::string(names + name_off[c], names + name_off[c + 1]); };
    std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return name(x) < name(y); });
    std::string blob;
    std::vector<uint32_t> sorted_off(n_contigs + 1, 0);
    for (uint32_t r = 0; r < n_contigs; ++r) {
        if (r && name(order[r]) == name(order[r - 1])) { ctx->last_error = "duplicate contig name " + name(order[r]); return NPH_ERR_INVALID; }
        rank[order[r]] = r;
        blob += name(order[r]);
        sorted_off[r + 1] = (uint32_t)blob.size();
    }
    const FreqTable t = table_of(f);
    const size_t slots = f.slots, header = sizeof(kHeader) - 1;
    // staging: names, offsets, ranks | occupied flags, offsets, scan scratch, sort keys and slots (both halves), row bytes and
    // offsets, cub's temporary storage, the missing-name flag
    size_t cub_bytes = 0;
    NPH_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                                  (uint32_t*)nullptr, (int)slots, 0, 64, ctx->stream));
    char* d_names; uint32_t* d_noff; uint32_t* d_rank; uint64_t* occupied; uint64_t* off; uint64_t* scratch;
    uint64_t* key_in; uint64_t* key_out; uint32_t* slot_in; uint32_t* slot_out; uint64_t* row_bytes; uint64_t* row_off; uint8_t* cub_tmp; int* missing;
    NPH_TRY(nph_carve(ctx, f.d_work, [&](NphArena& a) {
        d_names = a.take<char>(blob.size() + 1);
        d_noff = a.take<uint32_t>(n_contigs + 1);
        d_rank = a.take<uint32_t>(n_contigs + 1);
        occupied = a.take<uint64_t>(slots);
        off = a.take<uint64_t>(slots + 1);
        scratch = a.take<uint64_t>(nph_scan_scratch(slots));
        key_in = a.take<uint64_t>(slots); key_out = a.take<uint64_t>(slots);
        slot_in = a.take<uint32_t>(slots); slot_out = a.take<uint32_t>(slots);
        row_bytes = a.take<uint64_t>(slots);
        row_off = a.take<uint64_t>(slots + 1);
        cub_tmp = a.take<uint8_t>(cub_bytes);
        missing = a.take<int>(1);
    }));
    if (!blob.empty()) NPH_CUDA(ctx, cudaMemcpyAsync(d_names, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_noff, sorted_off.data(), sizeof(uint32_t) * (n_contigs + 1), cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_rank, rank.data(), sizeof(uint32_t) * (n_contigs + 1), cudaMemcpyHostToDevice, ctx->stream));
    NPH_CUDA(ctx, cudaMemsetAsync(missing, 0, sizeof(int), ctx->stream));
    const int grid = grid_for(ctx, slots);
    freq_occupied_kernel<<<grid, kThreads, 0, ctx->stream>>>(t, occupied);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_TRY(nph_scan_exclusive(ctx, occupied, (uint32_t)slots, off, scratch));
    freq_scatter_kernel<<<grid, kThreads, 0, ctx->stream>>>(t, off, d_rank, n_contigs, key_in, slot_in, missing);
    NPH_CUDA(ctx, cudaGetLastError());
    uint64_t n_rows = 0;
    int h_missing = 0;
    NPH_CUDA(ctx, cudaMemcpyAsync(&n_rows, off + slots, sizeof(n_rows), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(&h_missing, missing, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h_missing) { ctx->last_error = "a folded batch's contig_id has no name (n_contigs too small)"; return NPH_ERR_INVALID; }
    uint64_t rows_total = 0;
    RowArgs ra{t, key_out, slot_out, d_names, d_noff, f.d_pool.p, n_rows, row_bytes, row_off, nullptr};
    if (n_rows) {
        int end_bit = kContigShift;
        while (end_bit < 64 && (1ull << (end_bit - kContigShift)) < n_contigs) ++end_bit;
        NPH_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, key_in, key_out, slot_in, slot_out, (int)n_rows, 0, end_bit, ctx->stream));
        const int rgrid = grid_for(ctx, n_rows);
        freq_rows_kernel<false><<<rgrid, kThreads, 0, ctx->stream>>>(ra);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_scan_exclusive(ctx, row_bytes, (uint32_t)n_rows, row_off, scratch));
        NPH_CUDA(ctx, cudaMemcpyAsync(&rows_total, row_off + n_rows, sizeof(rows_total), cudaMemcpyDeviceToHost, ctx->stream));
        NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *n_bytes_out = header + rows_total;
    if (header + rows_total > cap || !out) {
        ctx->last_error = "out too small: " + std::to_string(header + rows_total) + " bytes";
        return NPH_ERR_INVALID;
    }
    std::memcpy(out, kHeader, header);
    if (!n_rows) return NPH_OK;
    NPH_TRY(nph_reserve(ctx, f.d_out, (size_t)rows_total));
    ra.out = reinterpret_cast<char*>(f.d_out.p);
    freq_rows_kernel<true><<<grid_for(ctx, n_rows), kThreads, 0, ctx->stream>>>(ra);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaMemcpyAsync(out + header, f.d_out.p, (size_t)rows_total, cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return NPH_OK;
}
