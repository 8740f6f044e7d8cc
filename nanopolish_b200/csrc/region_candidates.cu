// region_candidates.cu — AlignmentDB::get_variants_in_region (ref: src/alignment/nanopolish_alignment_db.cpp:259-368) on the device:
// the basecall candidates of a loaded region in one call (nph_region_candidates_batch, include/nph.h).
//
//   decode   meth_expand_kernel (methylation.cu, through nph_event_records_expand): the read position of every reference base
//   walk     cand_walk_kernel<false>, a warp per record: checks the record, adds its depth range to a difference array, counts
//            its instances; one exclusive scan for the depth, one for the instance offsets, one read-back of the total
//   fill     cand_walk_kernel<true>: the same walk writes each instance and its sort key (position, FNV-1a of the alleles)
//   merge    cub radix sort of the keys (stable), cand_rep_kernel: each instance's representative is the first instance of its
//            key's run with the same bytes, its count an integer atomic; a scan over the representatives; cand_emit_kernel
// The walk takes the pairs 32 reference positions at a time: valid, match and contiguous flags by ballot, and the next visited
// pair by __ffs on the valid (no gap) or match (after a gap) mask above the current one, carried across chunks.  The order of the
// output is the keys' (position, hash, first instance); the reference's std::map order and its filter are the host's.
#include "nph_internal.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;

struct CandInst { int32_t pos; uint32_t ref_len, alt_len, record; uint64_t alt_off; };

struct WalkArgs {
    const uint8_t* ref;                 // region reference
    const uint8_t* seq;                 // the records' bases
    const int16_t* deltas;
    const int32_t* dense;               // read position per reference base (NPH_NO_EVENT: no pair)
    const int32_t* first_valid;
    const nph_meth_record* recs;        // ref_off / ref_len / ref_start_pos: the record's compact alignment
    const nph_seq_record* srecs;
    uint32_t n_records;
    int32_t region_start, start, stop;
    unsigned long long* depth_diff;     // stop - start + 1 entries
    uint64_t* inst_count;               // per record
    const uint64_t* inst_off;           // per record (fill)
    CandInst* inst;                     // fill
    uint64_t* key;                      // fill
    uint32_t* order;                    // fill: instance index per key
    unsigned long long* n_pairs;
    int* bad;
};

__device__ __forceinline__ uint32_t fnv_step(uint32_t h, uint32_t b) { return (h ^ b) * 16777619u; }

template <bool FILL>
__global__ void __launch_bounds__(kThreads) cand_walk_kernel(WalkArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t rec = warp; rec < a.n_records; rec += n_warps) {
        const nph_meth_record R = a.recs[rec];
        const nph_seq_record S = a.srecs[rec];
        const int n = (int)R.ref_len;
        const int32_t* dense = a.dense + R.ref_off;
        const int fv = a.first_valid[rec];
        if (fv >= n) { if (!FILL && lane == 0) a.inst_count[rec] = 0; continue; }      // aligned_bases.empty()
        if (!FILL) {
            // the record's read positions: inside its bases and strictly increasing; the last pair for the depth
            bool bad = false;
            int last = -1;
            const int16_t* dl = a.deltas + R.ref_off;
            for (int base = 0; base < n; base += 32) {
                const int o = base + lane;
                const int d = o < n ? dense[o] : NPH_NO_EVENT;
                if (d != NPH_NO_EVENT) {
                    bad |= d < 0 || d >= (int)S.seq_len || (o != fv && dl[o] < 1);
                    last = o;
                }
            }
            for (int s = 16; s; s >>= 1) last = max(last, __shfl_xor_sync(kFull, last, s));
            if (__any_sync(kFull, bad)) { if (lane == 0) { atomicExch(a.bad, 1); a.inst_count[rec] = 0; } continue; }
            const int is = nph_first_valid_from(dense, n, a.start - R.ref_start_pos);
            if (is < n && lane == 0) {
                const int ie = nph_first_valid_from(dense, n, a.stop - R.ref_start_pos);
                const int ds = max(R.ref_start_pos + is, a.start);
                const int de = min(R.ref_start_pos + (ie < n ? ie : last), a.stop);
                if (ds < de) {
                    atomicAdd(a.depth_diff + (ds - a.start), 1ull);
                    atomicAdd(a.depth_diff + (de - a.start), ~0ull);               // -1, modulo 2^64: the scan sums to the depth
                }
            }
        }
        const int is = nph_first_valid_from(dense, n, a.start - R.ref_start_pos);
        const int ie = nph_first_valid_from(dense, n, a.stop - R.ref_start_pos);
        const uint8_t* seq = a.seq + S.seq_off;
        const uint8_t* ref = a.ref + (R.ref_start_pos - a.region_start);          // indexed by offsets in [is, ie): inside the region
        uint64_t n_inst = 0, at = FILL ? a.inst_off[rec] : 0;
        uint32_t walked = 0;
        int cur = -1;                    // the pair the walk stands on (-1: before the first)
        bool seek_match = false, emit = false;
        for (int base = is; base < ie; base += 32) {
            const int o = base + lane;
            const int d = o < ie ? dense[o] : NPH_NO_EVENT;
            const bool valid = d != NPH_NO_EVENT;
            const bool match = valid && ref[o] == seq[d];
            const bool contiguous = valid && o + 1 < n && dense[o + 1] == d + 1;
            const unsigned V = __ballot_sync(kFull, valid), M = __ballot_sync(kFull, match), C = __ballot_sync(kFull, contiguous);
            walked += __popc(V);
            unsigned above = cur < base ? kFull : 0u;
            for (;;) {
                const unsigned m = (seek_match ? M : V) & above;
                if (!m) break;
                const int b = __ffs(m) - 1, k = base + b;
                if (cur >= 0 && emit && R.ref_start_pos + k < a.stop - 1) {
                    if (FILL && lane == 0) {
                        const int r0 = dense[cur], r1 = dense[k];
                        CandInst I{R.ref_start_pos + cur, (uint32_t)(k - cur), (uint32_t)(r1 - r0), rec, S.seq_off + (uint64_t)r0};
                        uint32_t h = 2166136261u;
                        h = fnv_step(h, I.ref_len & 0xffffu); h = fnv_step(h, I.ref_len >> 16);
                        h = fnv_step(h, I.alt_len & 0xffffu); h = fnv_step(h, I.alt_len >> 16);
                        for (uint32_t q = 0; q < I.alt_len; ++q) h = fnv_step(h, seq[r0 + q]);
                        a.inst[at] = I;
                        a.key[at] = (uint64_t)(uint32_t)(I.pos - a.start) << 32 | h;
                        a.order[at] = (uint32_t)at;
                    }
                    ++at; ++n_inst;
                }
                cur = k;
                const bool c = (C >> b) & 1u, x = !((M >> b) & 1u);
                seek_match = !c;                 // a gap unless the next pair is (ref + 1, read + 1) or stop_iter
                emit = x || !c;
                above = b == 31 ? 0u : kFull << (b + 1);
            }
        }
        if (!FILL && lane == 0) {
            a.inst_count[rec] = n_inst;
            atomicAdd(a.n_pairs, (unsigned long long)walked);
        }
    }
}

struct MergeArgs {
    const uint8_t* seq;
    const uint8_t* ref;
    const CandInst* inst;
    const uint64_t* key;                // sorted
    const uint32_t* order;              // instance of each sorted key
    uint32_t* rep;                      // per sorted slot: the sorted slot of its representative
    uint64_t* is_rep;                   // per sorted slot
    unsigned int* count;                // per sorted slot (representatives)
    uint64_t n;
};

__device__ __forceinline__ bool same_alleles(const uint8_t* seq, const CandInst& x, const CandInst& y)
{
    if (x.pos != y.pos || x.ref_len != y.ref_len || x.alt_len != y.alt_len) return false;
    for (uint32_t q = 0; q < x.alt_len; ++q) if (seq[x.alt_off + q] != seq[y.alt_off + q]) return false;
    return true;
}

__global__ void __launch_bounds__(256) cand_rep_kernel(MergeArgs a)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < a.n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k = a.key[i];
        uint64_t lo = 0, hi = i;                                  // the first slot of i's key run
        while (lo < hi) { const uint64_t mid = (lo + hi) / 2; if (a.key[mid] < k) lo = mid + 1; else hi = mid; }
        const CandInst me = a.inst[a.order[i]];
        uint64_t j = lo;
        while (j < i && !same_alleles(a.seq, a.inst[a.order[j]], me)) ++j;
        a.rep[i] = (uint32_t)j;
        a.is_rep[i] = j == i;
        atomicAdd(a.count + j, 1u);
    }
}

__global__ void __launch_bounds__(256) cand_emit_kernel(MergeArgs a, const uint64_t* out_off, const unsigned long long* depth_excl, int32_t start,
                                                        nph_region_candidate* out)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < a.n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (!a.is_rep[i]) continue;
        const CandInst I = a.inst[a.order[i]];
        nph_region_candidate c;
        c.ref_position = I.pos; c.ref_len = I.ref_len; c.alt_len = I.alt_len;
        c.count = a.count[i];
        c.depth = (uint32_t)depth_excl[I.pos - start + 1];       // the inclusive sum of the differences at the position
        c.record = I.record; c.alt_off = I.alt_off;
        out[out_off[i]] = c;
    }
}

} // namespace

extern "C" int nph_region_candidates_batch(nph_ctx* ctx, const char* region_ref, size_t n_ref, int32_t region_start,
                                           const char* bases, size_t n_bases, const int16_t* base_deltas, size_t n_deltas,
                                           const nph_seq_record* records, size_t n_records, int32_t start, int32_t stop,
                                           nph_region_candidate* out, size_t out_cap, uint64_t* n_out, nph_candidate_counts* counts_out)
{
    if (!ctx || !n_out || (n_records && (!records || !base_deltas)) || (n_ref && !region_ref) || (n_bases && !bases) || (out_cap && !out))
        return NPH_ERR_INVALID;
    *n_out = 0;
    if (stop < start) { ctx->last_error = "stop < start"; return NPH_ERR_INVALID; }
    if (n_ref == 0 || start < region_start || (int64_t)stop > (int64_t)region_start + (int64_t)n_ref - 1) {
        ctx->last_error = "[start, stop] is not inside the loaded reference"; return NPH_ERR_INVALID;
    }
    if (n_records > UINT32_MAX) { ctx->last_error = "more than 2^32 - 1 records"; return NPH_ERR_INVALID; }
    std::vector<nph_meth_record> recs(n_records);
    std::vector<int32_t> first(std::max<size_t>(n_records, 1));
    for (size_t r = 0; r < n_records; ++r) {
        const nph_seq_record& S = records[r];
        if (!nph_slice_ok(S.seq_off, S.seq_len, n_bases) || !nph_slice_ok(S.map_off, S.map_len, n_deltas) ||
            (int64_t)S.ref_start_pos + (int64_t)S.map_len > (int64_t)INT32_MAX) {
            ctx->last_error = "record " + std::to_string(r) + ": its bases or alignment leave their arrays"; return NPH_ERR_INVALID;
        }
        std::memset(&recs[r], 0, sizeof(nph_meth_record));
        recs[r].ref_off = S.map_off; recs[r].ref_len = S.map_len; recs[r].ref_start_pos = S.ref_start_pos;
        first[r] = S.first_read_pos;
    }
    nph_candidate_counts cnt{};
    cnt.n_records = n_records;
    if (counts_out) *counts_out = cnt;
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));
    nph_ctx::CandState& cs = ctx->cand;
    cudaStream_t st = ctx->stream;
    NPH_TRY(nph_event_records_upload(ctx, cs.ev, region_ref, n_ref, n_deltas, true, base_deltas, first.data(), nullptr, 0, recs.data(), n_records));
    NPH_TRY(nph_reserve(ctx, cs.d_seq, n_bases + 16));
    if (n_bases) NPH_CUDA(ctx, cudaMemcpyAsync(cs.d_seq.p, bases, n_bases, cudaMemcpyHostToDevice, st));
    const size_t L = (size_t)(stop - start) + 1;
    const uint32_t nr = (uint32_t)n_records;
    unsigned long long *d_diff, *d_depth, *d_sum;
    uint64_t *d_cnt, *d_off, *d_scan;
    int* d_bad;
    NPH_TRY(nph_carve(ctx, cs.d_work, [&](NphArena& w) {
        d_diff = w.take<unsigned long long>(L + 1);
        d_depth = w.take<unsigned long long>(L + 2);
        d_cnt = w.take<uint64_t>(n_records + 1);
        d_off = w.take<uint64_t>(n_records + 1);
        d_scan = w.take<uint64_t>(nph_scan_scratch(std::max(L + 1, n_records + 1)) + 1);
        d_sum = w.take<unsigned long long>(1);
        d_bad = w.take<int>(1);
    }));
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, st));
    int launches = 0;
    const int32_t* dense;
    const int32_t* first_valid;
    NPH_TRY(nph_event_records_expand(ctx, cs.ev, &dense, &first_valid));
    launches += n_records ? 1 : 0;
    NPH_CUDA(ctx, cudaMemsetAsync(d_diff, 0, sizeof(unsigned long long) * (L + 1), st));
    NPH_CUDA(ctx, cudaMemsetAsync(d_sum, 0, sizeof(unsigned long long), st));
    NPH_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    WalkArgs wa{reinterpret_cast<const uint8_t*>(cs.ev.d_ref.p), cs.d_seq.p, reinterpret_cast<const int16_t*>(cs.ev.d_deltas.p), dense, first_valid,
                cs.ev.d_records.p, nullptr, nr, region_start, start, stop, d_diff, d_cnt, d_off, nullptr, nullptr, nullptr, d_sum, d_bad};
    // the records' nph_seq_record fields the walk reads (seq_off, seq_len) ride in a slice of the instance buffer's head
    nph_seq_record* d_srecs;
    NPH_TRY(nph_carve(ctx, cs.d_inst, [&](NphArena& w) { d_srecs = w.take<nph_seq_record>(n_records + 1); }));
    if (n_records) NPH_CUDA(ctx, cudaMemcpyAsync(d_srecs, records, sizeof(nph_seq_record) * n_records, cudaMemcpyHostToDevice, st));
    wa.srecs = d_srecs;
    const int grid = (int)std::min<size_t>((n_records + kWarps - 1) / kWarps + 1, (size_t)ctx->sm_count * 8);
    if (n_records) {
        cand_walk_kernel<false><<<grid, kThreads, 0, st>>>(wa);
        NPH_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    NPH_TRY(nph_scan_exclusive(ctx, reinterpret_cast<const uint64_t*>(d_diff), (uint32_t)L, reinterpret_cast<uint64_t*>(d_depth), d_scan));
    NPH_TRY(nph_scan_exclusive(ctx, d_cnt, nr, d_off, d_scan));
    launches += 6;
    uint64_t n_inst = 0;
    unsigned long long h_pairs = 0;
    int h_bad = 0;
    NPH_CUDA(ctx, cudaMemcpyAsync(&n_inst, d_off + nr, sizeof(n_inst), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(&h_pairs, d_sum, sizeof(h_pairs), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(&h_bad, d_bad, sizeof(h_bad), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    if (h_bad) { ctx->last_error = "a record's read positions leave its bases or do not strictly increase"; return NPH_ERR_INVALID; }
    cnt.n_pairs = h_pairs; cnt.n_instances = n_inst;
    uint64_t n_var = 0;
    if (n_inst) {
        if (n_inst > UINT32_MAX) { ctx->last_error = "more than 2^32 - 1 instances"; return NPH_ERR_UNSUPPORTED; }
        size_t cub_bytes = 0;
        NPH_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                                      (uint32_t*)nullptr, (int)n_inst, 0, 64, st));
        CandInst* d_inst;
        uint64_t *key_in, *key_out, *is_rep, *rep_off, *scan2;
        uint32_t *ord_in, *ord_out, *rep;
        unsigned int* count;
        nph_region_candidate* d_res;
        void* cub_tmp;
        // the records stay at the head (the same first slice as above), so the carve keeps d_srecs in place
        NPH_TRY(nph_carve(ctx, cs.d_inst, [&](NphArena& w) {
            d_srecs = w.take<nph_seq_record>(n_records + 1);
            d_inst = w.take<CandInst>(n_inst);
            key_in = w.take<uint64_t>(n_inst); key_out = w.take<uint64_t>(n_inst);
            ord_in = w.take<uint32_t>(n_inst); ord_out = w.take<uint32_t>(n_inst);
            rep = w.take<uint32_t>(n_inst);
            is_rep = w.take<uint64_t>(n_inst); rep_off = w.take<uint64_t>(n_inst + 1);
            count = w.take<unsigned int>(n_inst);
            d_res = w.take<nph_region_candidate>(n_inst);
            scan2 = w.take<uint64_t>(nph_scan_scratch(n_inst) + 1);
            cub_tmp = w.take<uint8_t>(cub_bytes);
        }));
        // nph_carve may have moved the buffer: the records go up again
        if (n_records) NPH_CUDA(ctx, cudaMemcpyAsync(d_srecs, records, sizeof(nph_seq_record) * n_records, cudaMemcpyHostToDevice, st));
        wa.srecs = d_srecs; wa.inst = d_inst; wa.key = key_in; wa.order = ord_in;
        cand_walk_kernel<true><<<grid, kThreads, 0, st>>>(wa);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, key_in, key_out, ord_in, ord_out, (int)n_inst, 0, 64, st));
        NPH_CUDA(ctx, cudaMemsetAsync(count, 0, sizeof(unsigned int) * n_inst, st));
        MergeArgs ma{cs.d_seq.p, reinterpret_cast<const uint8_t*>(cs.ev.d_ref.p), d_inst, key_out, ord_out, rep, is_rep, count, n_inst};
        const unsigned g2 = (unsigned)std::min<uint64_t>((n_inst + 255) / 256, (uint64_t)ctx->sm_count * 16);
        cand_rep_kernel<<<g2, 256, 0, st>>>(ma);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_scan_exclusive(ctx, is_rep, (uint32_t)n_inst, rep_off, scan2));
        NPH_CUDA(ctx, cudaMemcpyAsync(&n_var, rep_off + n_inst, sizeof(n_var), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));
        launches += 8;
        *n_out = n_var;
        if (n_var > out_cap) {
            ctx->last_error = "out_cap too small: " + std::to_string(n_var) + " variants";
            return NPH_ERR_INVALID;
        }
        cand_emit_kernel<<<g2, 256, 0, st>>>(ma, rep_off, d_depth, start, d_res);
        NPH_CUDA(ctx, cudaGetLastError());
        ++launches;
        NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(out, d_res, sizeof(nph_region_candidate) * n_var, cudaMemcpyDeviceToHost, st));
    } else {
        NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, st));
    }
    NPH_CUDA(ctx, cudaStreamSynchronize(st));
    float ms = 0.f;
    NPH_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    cnt.n_variants = n_var;
    cnt.kernel_ms = ms;
    nph_timing_staged(ctx, ms, launches);
    if (counts_out) *counts_out = cnt;
    return NPH_OK;
}
