// eventalign_tsv.cu — the rows of eventalign.tsv written on the device from the records an eventalign chain run left there.
//
// Replaces, for a batch of reads, the critical section of
//   emit_event_alignment_tsv                   ref: src/alignment/nanopolish_eventalign.cpp:398-484
// with what it calls per row
//   SquiggleRead::get_fully_scaled_level, get_scaled_gaussian_from_pore_model_state   ref: src/nanopolish_squiggle_read.h:149-171, 217-226
//   SquiggleRead::get_event_sample_idx, get_scaled_samples_for_event                  ref: src/nanopolish_squiggle_read.cpp:393-428
//
// A batch is tens of millions of rows of 80-130 bytes (a few hundred with --samples), each built from a 12-byte record, a k-mer
// rank, a model state and three event floats that are already in HBM.  Formatting them on the host means copying the records
// back and spending the host's threads on integer divisions; here the row rule of tsv_format.cuh (the one the host writer uses
// too) runs one thread per row: a length pass, the library's prefix sum over the lengths, a write pass in which every warp stages
// its 32 consecutive rows — consecutive bytes of the output — in shared memory and stores them as one span.  The sample column
// is a warp's work per row: lanes format samples, a warp prefix places them.  Reads with a value the exact formatters refuse
// get no bytes and a flag; their rows are the caller's to format with the C library.
#include "nph_internal.cuh"
#include "tsv_format.cuh"
#include <cstring>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kStage = 5120;          // shared bytes per warp in the write pass: 32 rows of up to ~150 bytes, plus 16 of alignment
constexpr unsigned kFull = 0xffffffffu;

struct EaTsvArgs {
    // resident since the chain run
    const nph_ea_chain* chains;
    const nph_ea_result* results;
    const nph_ea_record* records;
    const uint32_t* ranks_fwd;
    const uint32_t* ranks_rc;
    const DevRead* reads;
    const DevModelView* models;
    const float* level;
    // this call's inputs
    const uint64_t* chain_row;        // n_chains + 1: the first row of each chain
    const uint32_t* chain_read;       // n_chains: output read
    const nph_ea_tsv_read* treads;
    const char* text;
    const char* ref;
    const char* rc_ref;
    const float* ev_mean;
    const float* ev_stdv;
    const float* ev_duration;
    const double* ev_start_time;
    const float* samples;
    uint32_t n_chains;
    uint32_t n_rows;
    nph_ea_tsv_options opt;
    // working arrays
    uint64_t* row_len;                // n_rows
    const uint64_t* row_off;          // n_rows + 1
    unsigned int* refused;            // per output read
    char* out;
};

// everything one row is made of
struct RowState {
    nph_tsv::EaRow w;
    nph_tsv::EaRowNums r;
    nph_tsv::EaRead rd;
    uint32_t tread;                   // output read
    const float* samples;             // the read's raw samples
    uint64_t n_samples;               // how many the row's sample column has (0 without --samples)
    bool ok;
};

__device__ __forceinline__ uint32_t chain_of_row(const uint64_t* chain_row, uint32_t n_chains, uint32_t row)
{
    uint32_t lo = 0, hi = n_chains;                       // chain_row[lo] <= row < chain_row[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (chain_row[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ void load_row(const EaTsvArgs& a, uint32_t row, RowState& s)
{
    const uint32_t c = chain_of_row(a.chain_row, a.n_chains, row);
    const nph_ea_chain& ch = a.chains[c];
    const nph_ea_record rec = a.records[ch.out_off + (row - a.chain_row[c])];
    s.tread = a.chain_read[c];
    const nph_ea_tsv_read& tr = a.treads[s.tread];
    const DevRead rd = a.reads[ch.read];
    const uint32_t k = ch.k;
    const int64_t pos = (int64_t)rec.ref_position - ch.ref_offset;
    const char state = (char)rec.hmm_state;
    s.ok = pos >= 0 && (uint64_t)pos + k <= tr.ref_len && (uint32_t)rec.event_idx < tr.n_events;
    const uint32_t p = s.ok ? (uint32_t)pos : 0u, e = s.ok ? (uint32_t)rec.event_idx : 0u;

    s.rd.scale = rd.scale; s.rd.shift = rd.shift; s.rd.var = rd.var; s.rd.sqrt_var = nph_tsv::ea_sqrt(rd.var);
    s.rd.drift = tr.drift; s.rd.sample_rate = tr.sample_rate; s.rd.sample_start_time = tr.sample_start_time;
    double level_mean = 0.0, level_stdv = 0.0;
    if (state != 'B' && s.ok) {
        const uint32_t rank = (ch.rc ? a.ranks_rc : a.ranks_fwd)[ch.rank_off + p];
        const DevModelView mv = a.models[ch.model_id];
        level_mean = mv.mean[rank]; level_stdv = mv.stdv[rank];
    }
    const bool sample_idx = a.opt.write_signal_index || a.opt.write_samples;
    const uint64_t ev = tr.event_off + e;
    s.r = nph_tsv::ea_row_numbers(a.ev_mean[ev], a.opt.scale_events ? a.level[rd.event_off + e] : 0.0f, a.ev_stdv[ev], a.ev_duration[ev],
                                  sample_idx ? a.ev_start_time[ev] : 0.0, state, level_mean, level_stdv, s.rd, a.opt.scale_events != 0, sample_idx);
    s.ok = s.ok && s.r.ok;
    s.samples = nullptr; s.n_samples = 0;
    if (a.opt.write_samples && s.ok) {
        // an event without samples prints an empty column; a range that leaves the read's samples is the host's to report
        if (s.r.end_idx > s.r.start_idx) {
            if (s.r.end_idx > tr.n_samples) s.ok = false;
            else { s.samples = a.samples + tr.sample_off; s.n_samples = s.r.end_idx - s.r.start_idx; }
        }
    }
    s.w.contig = a.text + tr.contig_off; s.w.contig_len = tr.contig_len;
    s.w.ref_position = rec.ref_position;
    s.w.kmers = nph_tsv::ea_kmers_at(a.ref + tr.ref_off, a.rc_ref + tr.ref_off, tr.ref_len, p, k, ch.rc != 0, state);
    s.w.k = k;
    s.w.name = a.opt.print_read_names ? a.text + tr.name_off : nullptr; s.w.name_len = tr.name_len;
    s.w.read_idx = tr.read_idx;
    s.w.strand = tr.strand_idx ? 'c' : 't';
    s.w.event_idx = rec.event_idx;
    s.w.signal_index = a.opt.write_signal_index != 0;
}

// The sample column of the warp's rows, one row at a time: lanes take samples 32 at a time.  !WRITE: returns in lane `r` the
// bytes of row r's column and clears ok where a sample is outside the "%g" domain.  WRITE: the column at dst (lane r's, the byte
// after the row's tab).
template <bool WRITE>
__device__ __forceinline__ uint32_t sample_columns(const RowState& s, bool live, char* dst, bool& ok, int lane)
{
    uint32_t mine = 0;
    for (int r = 0; r < 32; ++r) {
        const unsigned long long n = __shfl_sync(kFull, live ? (unsigned long long)s.n_samples : 0ull, r);
        if (n == 0) continue;
        const float* smp = (const float*)__shfl_sync(kFull, (unsigned long long)s.samples, r);
        const unsigned long long first = __shfl_sync(kFull, (unsigned long long)s.r.start_idx, r);
        nph_tsv::EaRead rd;
        rd.scale = __shfl_sync(kFull, s.rd.scale, r); rd.shift = __shfl_sync(kFull, s.rd.shift, r); rd.drift = __shfl_sync(kFull, s.rd.drift, r);
        rd.sample_rate = __shfl_sync(kFull, s.rd.sample_rate, r);
        rd.sample_start_time = __shfl_sync(kFull, (unsigned long long)s.rd.sample_start_time, r);
        rd.var = 0.0; rd.sqrt_var = 0.0;
        char* o = WRITE ? (char*)__shfl_sync(kFull, (unsigned long long)dst, r) : nullptr;
        uint32_t total = 0;
        bool bad = false;
        for (unsigned long long base = 0; base < n; base += 32) {
            const unsigned long long i = base + lane;
            uint32_t len = 0;
            nph_tsv::G6 g{};
            if (i < n) {
                g = nph_tsv::g6_of(nph_tsv::ea_scaled_sample(smp[first + i], first + i, rd));
                bad |= !g.ok;
                len = (uint32_t)nph_tsv::g6_len(g) + (i ? 1u : 0u);          // ',' before every sample but the first
            }
            uint32_t incl = len;
            for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(kFull, incl, d); if (lane >= d) incl += v; }
            if (WRITE && i < n) {
                char* q = o + total + (incl - len);
                if (i) *q++ = ',';
                nph_tsv::put_g6(q, g);
            }
            total += __shfl_sync(kFull, incl, 31);
        }
        if (!WRITE && __any_sync(kFull, bad) && lane == r) ok = false;
        if (lane == r) mine = total;
    }
    return mine;
}

// pass 1: bytes of every row (0 and the read's flag where a value is refused)
__global__ void __launch_bounds__(kThreads) ea_tsv_len_kernel(const EaTsvArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint32_t n_tiles = (a.n_rows + 31) / 32;
    for (uint32_t tile = blockIdx.x * kWarps + (threadIdx.x >> 5); tile < n_tiles; tile += gridDim.x * kWarps) {
        const uint32_t row = tile * 32 + lane;
        const bool have = row < a.n_rows;
        RowState s;
        s.n_samples = 0; s.ok = false;
        if (have) load_row(a, row, s);
        bool ok = s.ok;
        uint32_t len = ok ? nph_tsv::ea_row_len(s.w, s.r) + 1u : 0u;            // + '\n'
        if (a.opt.write_samples) len += 1u + sample_columns<false>(s, have && ok, nullptr, ok, lane);     // + '\t'
        if (have) {
            if (!ok) a.refused[s.tread] = 1u;
            a.row_len[row] = ok ? len : 0u;
        }
    }
}

// between the passes: the rows of refused reads count zero
__global__ void __launch_bounds__(kThreads) ea_tsv_mask_kernel(const EaTsvArgs a)
{
    for (uint32_t row = blockIdx.x * kThreads + threadIdx.x; row < a.n_rows; row += gridDim.x * kThreads)
        if (a.refused[a.chain_read[chain_of_row(a.chain_row, a.n_chains, row)]]) a.row_len[row] = 0;
}

__global__ void ea_tsv_read_off_kernel(const uint64_t* row_off, const uint64_t* read_row, uint32_t n_reads, uint64_t* read_off)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= n_reads) read_off[r] = row_off[read_row[r]];
}

// pass 2: the rows at row_off
__global__ void __launch_bounds__(kThreads) ea_tsv_write_kernel(const EaTsvArgs a)
{
    __shared__ __align__(16) char s_stage[kWarps][kStage];
    const int lane = threadIdx.x & 31;
    char* const stage = s_stage[threadIdx.x >> 5];
    const uint32_t n_tiles = (a.n_rows + 31) / 32;
    for (uint32_t tile = blockIdx.x * kWarps + (threadIdx.x >> 5); tile < n_tiles; tile += gridDim.x * kWarps) {
        const uint32_t row = tile * 32 + lane, row_end = min(tile * 32 + 32, a.n_rows);
        const uint64_t g0 = a.row_off[tile * 32], span = a.row_off[row_end] - g0;
        if (span == 0) continue;
        const bool have = row < a.n_rows;
        const uint64_t off = have ? a.row_off[row] : 0;
        const bool live = have && a.row_off[row + 1] > off;
        RowState s;
        s.n_samples = 0;
        if (live) load_row(a, row, s);
        if (a.opt.write_samples) {
            // rows of a few hundred bytes: straight to the output, the sample column by the whole warp
            char* o = nullptr;
            if (live) { o = nph_tsv::put_ea_row(a.out + off, s.w, s.r); *o++ = '\t'; }
            bool ok = true;
            sample_columns<true>(s, live, o, ok, lane);
            if (live) a.out[a.row_off[row + 1] - 1] = '\n';
            continue;
        }
        const uint32_t skew = (uint32_t)(g0 & 15u);                              // shared and global bytes share their 16-byte phase
        const bool staged = span + skew <= (uint64_t)kStage;
        if (live) {
            char* o = nph_tsv::put_ea_row(staged ? stage + skew + (off - g0) : a.out + off, s.w, s.r);
            *o = '\n';
        }
        if (!staged) continue;
        __syncwarp();
        const uint32_t n = (uint32_t)span;
        const char* src = stage + skew;
        char* dst = a.out + g0;
        const uint32_t head = min(n, (16u - skew) & 15u);
        if ((uint32_t)lane < head) dst[lane] = src[lane];
        const uint32_t n_vec = (n - head) / 16u;
        const uint4* vs = reinterpret_cast<const uint4*>(src + head);
        uint4* vd = reinterpret_cast<uint4*>(dst + head);
        for (uint32_t i = lane; i < n_vec; i += 32) vd[i] = vs[i];
        const uint32_t done = head + 16u * n_vec;
        if (done + lane < n) dst[done + lane] = src[done + lane];
        __syncwarp();
    }
}

} // namespace

extern "C" int nph_eventalign_tsv(nph_ctx* ctx, const nph_ea_tsv_batch* in, const nph_ea_tsv_options* opt, char* tsv_out, size_t cap,
                                  uint64_t* row_off_out, uint64_t* read_off_out, uint8_t* read_refused_out, uint64_t* n_bytes_out)
{
    if (!ctx || !in || !opt || !read_off_out || !read_refused_out || !n_bytes_out) return NPH_ERR_INVALID;
    nph_ctx::EaState& ea = ctx->ea;
    if (!ea.resident || !ctx->reads_loaded) return NPH_ERR_STATE;
    *n_bytes_out = 0;
    const size_t n_chains = ea.h_chains.size(), n_reads = in->n_reads;
    const bool sample_idx = opt->write_signal_index || opt->write_samples;
    if (!in->reads || !in->chain_read || n_reads == 0 || !in->text || !in->ref || !in->rc_ref || !in->ev_mean || !in->ev_stdv || !in->ev_duration ||
        (sample_idx && !in->ev_start_time) || (opt->write_samples && in->n_samples && !in->samples))
        return NPH_ERR_INVALID;
    auto invalid = [&](const char* what) { ctx->last_error = what; return NPH_ERR_INVALID; };
    for (size_t r = 0; r < n_reads; ++r) {
        const nph_ea_tsv_read& t = in->reads[r];
        if (!nph_slice_ok(t.contig_off, t.contig_len, in->n_text) || !nph_slice_ok(t.name_off, t.name_len, in->n_text) ||
            !nph_slice_ok(t.ref_off, t.ref_len, in->n_ref) || !nph_slice_ok(t.event_off, t.n_events, in->n_events) ||
            (opt->write_samples && !nph_slice_ok(t.sample_off, t.n_samples, in->n_samples)))
            return invalid("nph_eventalign_tsv: a read's slice lies outside its array");
    }
    // rows: the records of every chain, in chain order; a chain the kernel did not finish refuses its read
    std::vector<uint64_t> chain_row(n_chains + 1, 0), read_row(n_reads + 1, 0);
    std::vector<unsigned int> refused(n_reads, 0u);
    uint32_t prev_read = 0;
    for (size_t c = 0; c < n_chains; ++c) {
        const uint32_t r = in->chain_read[c];
        if (r >= n_reads || r < prev_read) return invalid("nph_eventalign_tsv: chain_read must name the output reads in non-decreasing order");
        const nph_ea_chain& ch = ea.h_chains[c];
        if (in->reads[r].ref_len != ch.ref_len || in->reads[r].n_events != ctx->h_read_n_events[ch.read])
            return invalid("nph_eventalign_tsv: a read's reference or events are not those of its chain");
        for (uint32_t q = prev_read + 1; q <= r; ++q) read_row[q] = chain_row[c];
        prev_read = r;
        if (ea.h_results[c].status != NPH_EA_OK) refused[r] = 1u;
        chain_row[c + 1] = chain_row[c] + ea.h_results[c].n_records;
    }
    for (size_t q = prev_read + 1; q <= n_reads; ++q) read_row[q] = chain_row[n_chains];
    const uint64_t n_rows = chain_row[n_chains];
    if (n_rows >= UINT32_MAX) return invalid("nph_eventalign_tsv: more than 2^32 rows in one batch");
    NPH_CUDA(ctx, cudaSetDevice(ctx->device));

    const size_t n_smp = opt->write_samples ? in->n_samples : 0, n_time = sample_idx ? in->n_events : 0;
    EaTsvArgs a{};
    uint64_t* d_chain_row; uint32_t* d_chain_read; nph_ea_tsv_read* d_treads; char* d_text; char* d_ref; char* d_rc;
    float* d_mean; float* d_stdv; float* d_dur; double* d_time; float* d_smp; uint64_t* d_read_row;
    NPH_TRY(nph_carve(ctx, ea.d_tsv_in, [&](NphArena& ar) {
        d_chain_row = ar.take<uint64_t>(n_chains + 1);
        d_read_row = ar.take<uint64_t>(n_reads + 1);
        d_chain_read = ar.take<uint32_t>(n_chains);
        d_treads = ar.take<nph_ea_tsv_read>(n_reads);
        d_text = ar.take<char>(in->n_text + 1);
        d_ref = ar.take<char>(in->n_ref + 1);
        d_rc = ar.take<char>(in->n_ref + 1);
        d_mean = ar.take<float>(in->n_events + 1);
        d_stdv = ar.take<float>(in->n_events + 1);
        d_dur = ar.take<float>(in->n_events + 1);
        d_time = ar.take<double>(n_time + 1);
        d_smp = ar.take<float>(n_smp + 1);
    }));
    uint64_t* d_row_len; uint64_t* d_row_off; uint64_t* d_scan; uint64_t* d_read_off; unsigned int* d_refused;
    NPH_TRY(nph_carve(ctx, ea.d_tsv_off, [&](NphArena& ar) {
        d_row_len = ar.take<uint64_t>(n_rows + 1);
        d_row_off = ar.take<uint64_t>(n_rows + 1);
        d_scan = ar.take<uint64_t>(nph_scan_scratch(n_rows) + 1);
        d_read_off = ar.take<uint64_t>(n_reads + 1);
        d_refused = ar.take<unsigned int>(n_reads);
    }));
    auto up = [&](void* dst, const void* src, size_t bytes) {
        return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream) : cudaSuccess;
    };
    NPH_CUDA(ctx, up(d_chain_row, chain_row.data(), sizeof(uint64_t) * (n_chains + 1)));
    NPH_CUDA(ctx, up(d_read_row, read_row.data(), sizeof(uint64_t) * (n_reads + 1)));
    NPH_CUDA(ctx, up(d_chain_read, in->chain_read, sizeof(uint32_t) * n_chains));
    NPH_CUDA(ctx, up(d_treads, in->reads, sizeof(nph_ea_tsv_read) * n_reads));
    NPH_CUDA(ctx, up(d_text, in->text, in->n_text));
    NPH_CUDA(ctx, up(d_ref, in->ref, in->n_ref));
    NPH_CUDA(ctx, up(d_rc, in->rc_ref, in->n_ref));
    NPH_CUDA(ctx, up(d_mean, in->ev_mean, sizeof(float) * in->n_events));
    NPH_CUDA(ctx, up(d_stdv, in->ev_stdv, sizeof(float) * in->n_events));
    NPH_CUDA(ctx, up(d_dur, in->ev_duration, sizeof(float) * in->n_events));
    NPH_CUDA(ctx, up(d_time, in->ev_start_time, sizeof(double) * n_time));
    NPH_CUDA(ctx, up(d_smp, in->samples, sizeof(float) * n_smp));
    NPH_CUDA(ctx, up(d_refused, refused.data(), sizeof(unsigned int) * n_reads));

    a.chains = ea.d_chains; a.results = ea.d_results; a.records = ea.d_records; a.ranks_fwd = ea.d_ranks_fwd; a.ranks_rc = ea.d_ranks_rc;
    a.reads = ctx->d_reads.p; a.models = ctx->d_models.p; a.level = ctx->d_level.p;
    a.chain_row = d_chain_row; a.chain_read = d_chain_read; a.treads = d_treads; a.text = d_text; a.ref = d_ref; a.rc_ref = d_rc;
    a.ev_mean = d_mean; a.ev_stdv = d_stdv; a.ev_duration = d_dur; a.ev_start_time = d_time; a.samples = d_smp;
    a.n_chains = (uint32_t)n_chains; a.n_rows = (uint32_t)n_rows; a.opt = *opt;
    a.row_len = d_row_len; a.row_off = d_row_off; a.refused = d_refused;

    const uint32_t n_tiles = (uint32_t)((n_rows + 31) / 32);
    const int grid = (int)std::max<size_t>(1, std::min<size_t>((n_tiles + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 16));
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    if (n_rows) {
        ea_tsv_len_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
        ea_tsv_mask_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    }
    NPH_TRY(nph_scan_exclusive(ctx, d_row_len, (uint32_t)n_rows, d_row_off, d_scan));
    ea_tsv_read_off_kernel<<<(unsigned)(n_reads / 256 + 1), 256, 0, ctx->stream>>>(d_row_off, d_read_row, (uint32_t)n_reads, d_read_off);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    nph_timing_events(ctx, 6);
    NPH_CUDA(ctx, cudaMemcpyAsync(read_off_out, d_read_off, sizeof(uint64_t) * (n_reads + 1), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaMemcpyAsync(refused.data(), d_refused, sizeof(unsigned int) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
    if (row_off_out) NPH_CUDA(ctx, cudaMemcpyAsync(row_off_out, d_row_off, sizeof(uint64_t) * (n_rows + 1), cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (size_t r = 0; r < n_reads; ++r) read_refused_out[r] = refused[r] ? 1 : 0;
    const uint64_t total = read_off_out[n_reads];
    *n_bytes_out = total;
    if (total == 0) return NPH_OK;
    if (total > cap || !tsv_out) {
        ctx->last_error = "tsv_out too small: " + std::to_string(total) + " bytes";
        return NPH_ERR_INVALID;
    }
    NPH_TRY(nph_reserve(ctx, ea.d_tsv, (size_t)total + 16));
    a.out = reinterpret_cast<char*>(ea.d_tsv.p);
    ea_tsv_write_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    NPH_CUDA(ctx, cudaGetLastError());
    NPH_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    nph_timing_events(ctx, 7);
    NPH_CUDA(ctx, cudaMemcpyAsync(tsv_out, ea.d_tsv.p, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    NPH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return NPH_OK;
}
