// window_reads.cu — the reads of a list of calling windows, for the region calls of `nanopolish variants` on the device
// (fix-homopolymers, all-support and list screening).
//
// Replaces, for every window of a call at once:
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_event_subsequence)
//
// Kernels, count -> scan -> fill:
//   window_reads_kernel<false>  a warp per window, the records 32 at a time: the window's event sequences, the kept ones
//                               (|e1 - e2| >= min_span) and their DP rows, and the largest rows of a kept pair
//   (nph_scan_exclusive: each window's first kept pair; one read-back sizes the pairs)
//   window_reads_kernel<true>   the same walk, writing the kept pairs {record, e1, e2} in record order and the window of each
#include "nph_internal.cuh"
#include <algorithm>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;

struct WalkArgs {
    const nph_meth_record* records;
    const int32_t* dense;
    const int32_t* first_valid;
    const int2* bounds;                  // per window [cs, ce]
    uint32_t n_records, n_windows;
    uint32_t min_span;
};

// FILL = false: per window the event sequences, the kept ones and their rows, and the largest rows; FILL = true: the kept pairs
template <bool FILL>
__global__ void __launch_bounds__(kThreads) window_reads_kernel(const WalkArgs a, uint32_t* __restrict__ met, uint64_t* __restrict__ kept,
                                                                unsigned long long* __restrict__ rows, unsigned int* __restrict__ max_rows,
                                                                const uint64_t* __restrict__ off, NphWinPair* __restrict__ pairs,
                                                                uint32_t* __restrict__ pair_win)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t wi = warp; wi < a.n_windows; wi += n_warps) {
        const int2 b = a.bounds[wi];
        uint32_t n_met = 0;
        uint64_t n = 0;
        unsigned long long r_sum = 0;
        unsigned int r_max = 0;
        const uint64_t first = FILL ? off[wi] : 0;
        for (uint32_t base = 0; base < a.n_records; base += 32) {
            const uint32_t r = base + lane;
            int e1 = 0, e2 = 0;
            bool in = false;
            if (r < a.n_records) {
                const nph_meth_record R = a.records[r];
                in = nph_event_subsequence(R, a.dense + R.ref_off, a.first_valid[r], b.x, b.y, e1, e2);
            }
            const unsigned rw = in ? nph_pair_rows(e1, e2) : 0u;
            const bool keep = in && rw - 1u >= a.min_span;
            // ordered append: record order is the order the reference walks its event records in
            const unsigned m = __ballot_sync(kFull, keep);
            if (FILL && keep) {
                const uint64_t at = first + n + __popc(m & ((1u << lane) - 1u));
                pairs[at] = NphWinPair{r, e1, e2};
                pair_win[at] = wi;
            }
            n += __popc(m);
            if (!FILL) {
                n_met += __popc(__ballot_sync(kFull, in));
                if (keep) { r_sum += rw; r_max = max(r_max, rw); }
            }
        }
        if (!FILL) {
            for (int o = 16; o; o >>= 1) {
                r_sum += __shfl_xor_sync(kFull, r_sum, o);
                r_max = max(r_max, __shfl_xor_sync(kFull, r_max, o));
            }
            if (lane == 0) {
                met[wi] = n_met;
                kept[wi] = n;
                rows[wi] = r_sum;
                if (r_max) atomicMax(max_rows, r_max);
            }
        }
    }
}

} // namespace

int nph_region_load(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, const double* ev_start_time,
                    size_t n_events_total, const char* ref, size_t n_ref, const int16_t* deltas, size_t n_deltas, const int32_t* first_event,
                    const nph_meth_record* records, size_t n_records, const std::function<int(size_t, const nph_meth_record&)>& check)
{
    NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
    // records index the event deltas, as the edit screen's do
    return nph_event_records_load(ctx, ctx->region.ev, ref, n_ref, n_deltas, true, deltas, first_event, nullptr, 0, records, n_records,
                                  0x3fffffffu, check);
}

int nph_window_reads(nph_ctx* ctx, const std::vector<int2>& bounds, int min_span, NphWindowReads& wr)
{
    nph_ctx::RegionState& rs = ctx->region;
    cudaStream_t st = ctx->stream;
    const size_t n = bounds.size();
    int2* d_bounds; uint32_t* d_met; uint64_t* d_kept; unsigned long long* d_rows; uint64_t* d_off; uint64_t* d_scratch; unsigned int* d_max;
    NPH_TRY(nph_carve(ctx, rs.d_counts, [&](NphArena& c) {
        d_bounds = c.take<int2>(n);
        d_met = c.take<uint32_t>(n);
        d_kept = c.take<uint64_t>(n);
        d_rows = c.take<unsigned long long>(n);
        d_off = c.take<uint64_t>(n + 1);
        d_scratch = c.take<uint64_t>(nph_scan_scratch(n));
        d_max = c.take<unsigned int>(1);
    }));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_bounds, bounds.data(), sizeof(int2) * n, cudaMemcpyHostToDevice, st));
    NPH_CUDA(ctx, cudaMemsetAsync(d_max, 0, sizeof(unsigned int), st));
    const int32_t* dense;
    const int32_t* first_valid;
    NPH_TRY(nph_event_records_expand(ctx, rs.ev, &dense, &first_valid));
    const WalkArgs a{rs.ev.d_records.p, dense, first_valid, d_bounds, (uint32_t)rs.ev.n_records, (uint32_t)n, (uint32_t)min_span};
    const int grid = (int)std::min<size_t>((n + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 8);
    window_reads_kernel<false><<<grid, kThreads, 0, st>>>(a, d_met, d_kept, d_rows, d_max, nullptr, nullptr, nullptr);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_TRY(nph_scan_exclusive(ctx, d_kept, (uint32_t)n, d_off, d_scratch));
    wr.off.resize(n + 1);
    wr.met.resize(n);
    wr.rows.resize(n);
    NPH_CUDA(ctx, cudaMemcpyAsync(wr.off.data(), d_off, sizeof(uint64_t) * (n + 1), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(wr.met.data(), d_met, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(wr.rows.data(), d_rows, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaMemcpyAsync(&wr.max_rows, d_max, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    NPH_CUDA(ctx, cudaStreamSynchronize(st));                         // the one read-back that sizes the pairs and what follows them
    const uint64_t n_pairs = wr.n_pairs();
    NphWinPair* d_pairs; uint32_t* d_pair_win;
    NPH_TRY(nph_carve(ctx, rs.d_pairs, [&](NphArena& c) {
        d_pairs = c.take<NphWinPair>(n_pairs);
        d_pair_win = c.take<uint32_t>(n_pairs);
    }));
    wr.d_off = d_off; wr.d_pairs = d_pairs; wr.d_pair_win = d_pair_win;
    if (n_pairs == 0) return NPH_OK;
    window_reads_kernel<true><<<grid, kThreads, 0, st>>>(a, nullptr, nullptr, nullptr, nullptr, d_off, d_pairs, d_pair_win);
    NPH_CUDA(ctx, cudaGetLastError());
    return NPH_OK;
}
