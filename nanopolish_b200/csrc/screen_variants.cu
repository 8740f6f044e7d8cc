// screen_variants.cu — screen_variants_by_score of `nanopolish variants --consensus` on the device: every candidate of a list
// screened in its own window in one call.
//
// Replaces, for a whole candidate list at once:
//   screen_variants_by_score                  ref: src/nanopolish_call_variants.cpp:364-402
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_window_reads)
//   Haplotype::apply_variant on the window    ref: src/nanopolish_haplotype.cpp:33-75 (decided on the host, per candidate)
//   score_variant_thresholded                 ref: src/common/nanopolish_variant.cpp:765-799, with the -q sets of
//                                             generate_methylated_alternatives (:158-178) as nph_screen_load_methylation forms them
//
// Candidates with the same window (calling_start, |ref_seq|) share its reads and base haplotype.  The host writes the base window of
// every window and the edited window of every candidate that applies as bytes.  Kernels, after the window-read walk of
// window_reads.cu (count -> scan -> fill: each window's event sequences and their event rows) and the rank pool of score_sets.cu
// (nph_set_ranks: both strands of every sequence and of each methylated copy, and which copies differ), the round loop of variants.cu:
//   per round, while any candidate is inside the threshold and has reads left:
//     sv_round_count_kernel   thread per window: the next reads_per_round reads, each scoring the base set and the set of every
//                             live candidate of the window
//     sv_emit_kernel          thread per window: those jobs, read by read; then K1 (nph_score_device_jobs)
//     sv_accumulate_kernel    thread per window: `if (fabs(total) < threshold) total += variant - base` per candidate, reads in order
#include "nph_internal.cuh"
#include "exact_math.cuh"
#include "meth_dev.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr uint32_t kNoSeq = 0xffffffffu;

// a window: [cs, cs + len - 1], its candidates wcand[cand_first, cand_first + n_cand), its base sequence
struct SvWin { int32_t cs, len; uint32_t cand_first, n_cand, base_seq, pad; };

// per candidate: the thresholded total, the reference's DP rows, its variant sequence (kNoSeq: outside the region or not applied),
// whether its total is inside the threshold at the start of the round
struct SvCand { double total; unsigned long long ref_rows; uint32_t seq, alive; };

struct SvWinState { uint32_t done, chunk; };

struct SvCounters { unsigned long long events, ref_events; unsigned int any_left; };

struct SvArgs {
    const nph_meth_record* records;
    const SvWin* wins;
    const NphSetSeq* seqs;
    const uint32_t* wcand;
    SvCand* cands;
    uint32_t n_wins;
    int k, rpr;
    uint32_t flags;
    double threshold;
};

// thread per window: how many jobs it contributes this round (per read the base set and the set of every live candidate)
__global__ void sv_round_count_kernel(const SvArgs a, SvWinState* __restrict__ ws, const uint64_t* __restrict__ pair_off,
                                      uint64_t* __restrict__ job_cnt, const uint32_t* __restrict__ alts)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= a.n_wins) return;
    const SvWin W = a.wins[wi];
    const uint32_t n_reads = (uint32_t)(pair_off[wi + 1] - pair_off[wi]);
    uint32_t per_read = set_size(alts[W.base_seq]);
    bool any = false;
    for (uint32_t c = 0; c < W.n_cand; ++c) {
        const SvCand& C = a.cands[a.wcand[W.cand_first + c]];
        if (!C.alive) continue;
        any = true;
        per_read += set_size(alts[C.seq]);
    }
    SvWinState s = ws[wi];
    s.chunk = any && s.done < n_reads ? min((uint32_t)a.rpr, n_reads - s.done) : 0u;
    ws[wi] = s;
    job_cnt[wi] = (uint64_t)s.chunk * per_read;
}

// appends the jobs of sequence si's set for one read
__device__ __forceinline__ nph_hmm_job* emit_seq(const SvArgs& a, const NphSetTypes& ty, const uint32_t* alts, nph_hmm_job jb,
                                                 const nph_meth_record& R, uint32_t record, uint32_t si, nph_hmm_job* out)
{
    const NphSetSeq S = a.seqs[si];
    jb.n_kmers = S.len - (uint32_t)a.k + 1u;
    return set_jobs(ty, jb, R, record, ty.T ? alts[si] : 0u, S.rank_off, jb.n_kmers, out);
}

__global__ void sv_emit_kernel(const SvArgs a, const SvWinState* __restrict__ ws, const uint64_t* __restrict__ pair_off,
                               const NphWinPair* __restrict__ pairs, const uint64_t* __restrict__ job_off, nph_hmm_job* __restrict__ jobs,
                               unsigned long long* __restrict__ events, const NphSetTypes ty, const uint32_t* __restrict__ alts)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long ev = 0;
    if (wi < a.n_wins && ws[wi].chunk) {
        const SvWinState s = ws[wi];
        const SvWin W = a.wins[wi];
        const NphWinPair* rd = pairs + pair_off[wi] + s.done;
        nph_hmm_job* out = jobs + job_off[wi];
        for (uint32_t r = 0; r < s.chunk; ++r) {
            const NphWinPair P = rd[r];
            const nph_meth_record R = a.records[P.record];
            const nph_hmm_job jb = nph_window_job(R, P, (uint8_t)a.flags);
            nph_hmm_job* const first = out;
            out = emit_seq(a, ty, alts, jb, R, P.record, W.base_seq, out);
            for (uint32_t c = 0; c < W.n_cand; ++c) {
                const SvCand& C = a.cands[a.wcand[W.cand_first + c]];
                if (C.alive) out = emit_seq(a, ty, alts, jb, R, P.record, C.seq, out);
            }
            ev += (unsigned long long)(out - first) * nph_pair_rows(P.e1, P.e2);
        }
    }
    for (int o = 16; o; o >>= 1) ev += __shfl_xor_sync(kFull, ev, o);
    if ((threadIdx.x & 31) == 0 && ev) atomicAdd(events, ev);
}

// thread per window: the round's reads in order, per read the base set's fold once and, for every live candidate, the sequential
// `if (fabs(total) < threshold) total += variant - base` (var_accumulate_kernel's arithmetic, NaN included)
__global__ void sv_accumulate_kernel(const SvArgs a, SvWinState* __restrict__ ws, const uint64_t* __restrict__ pair_off,
                                     const NphWinPair* __restrict__ pairs, const uint64_t* __restrict__ job_off, const float* __restrict__ scores,
                                     SvCounters* __restrict__ ctr, const NphSetTypes ty, const uint32_t* __restrict__ alts)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= a.n_wins) return;
    SvWinState s = ws[wi];
    if (!s.chunk) return;
    const SvWin W = a.wins[wi];
    const float* sc = scores + job_off[wi];
    const NphWinPair* rd = pairs + pair_off[wi] + s.done;
    const uint32_t nb = set_size(ty.T ? alts[W.base_seq] : 0u);
    unsigned long long ref_ev = 0;
    for (uint32_t r = 0; r < s.chunk; ++r) {
        // double base_score = profile_hmm_score_set(...) (a float); a set of one is its score
        const double base_score = (double)nph_score_set_fold(sc, nb, ty.pen[nb - 1], ty.tbl);
        sc += nb;
        const unsigned long long E = nph_pair_rows(rd[r].e1, rd[r].e2);
        for (uint32_t c = 0; c < W.n_cand; ++c) {
            SvCand& C = a.cands[a.wcand[W.cand_first + c]];
            if (!C.alive) continue;
            const uint32_t nc = set_size(ty.T ? alts[C.seq] : 0u);
            const double variant_score = (double)nph_score_set_fold(sc, nc, ty.pen[nc - 1], ty.tbl);
            sc += nc;
            if (fabs(C.total) < a.threshold) {
                C.total = __dadd_rn(C.total, __dsub_rn(variant_score, base_score));
                const unsigned long long rows = (unsigned long long)(nb + nc) * E;
                C.ref_rows += rows;
                ref_ev += rows;
            }
        }
    }
    s.done += s.chunk;
    s.chunk = 0;
    ws[wi] = s;
    const uint32_t n_reads = (uint32_t)(pair_off[wi + 1] - pair_off[wi]);
    bool left = false;
    for (uint32_t c = 0; c < W.n_cand; ++c) {
        SvCand& C = a.cands[a.wcand[W.cand_first + c]];
        if (!C.alive) continue;
        C.alive = fabs(C.total) < a.threshold ? 1u : 0u;
        left = left || (C.alive && s.done < n_reads);
    }
    if (ref_ev) atomicAdd(&ctr->ref_events, ref_ev);
    if (left) atomicOr(&ctr->any_left, 1u);
}

// the host's view of the list: windows, sequences and their bytes, the windows' candidate lists, the initial candidate states
struct SvPlan {
    std::vector<SvWin> wins;
    std::vector<NphSetSeq> seqs;
    std::vector<uint8_t> bytes;
    std::vector<uint32_t> wcand;
    std::vector<SvCand> cands;
    std::vector<uint32_t> cand_win;           // per candidate: its window (kNoSeq: outside the region)
    std::vector<uint8_t> applied;
};

int plan_list(nph_ctx* ctx, const nph_screen_list_params& p, const char* ref, size_t n_ref, const char* alleles, size_t n_allele_bytes,
              const nph_screen_candidate* cands, size_t n, SvPlan& pl)
{
    const int64_t region_end = (int64_t)p.region_start + (int64_t)n_ref - 1;
    std::unordered_map<uint64_t, uint32_t> win_of;          // (calling_start, |ref_seq|) -> window
    std::vector<std::vector<uint32_t>> members;
    pl.cands.assign(n, SvCand{0.0, 0ull, kNoSeq, 0u});
    pl.cand_win.assign(n, kNoSeq);
    pl.applied.assign(n, 0);
    for (size_t i = 0; i < n; ++i) {
        const nph_screen_candidate& c = cands[i];
        const std::string at = "candidate " + std::to_string(i) + ": ";
        if (!nph_slice_ok(c.ref_seq_off, c.ref_seq_len, n_allele_bytes) || !nph_slice_ok(c.alt_seq_off, c.alt_seq_len, n_allele_bytes)) {
            ctx->last_error = at + "an allele outside alleles";
            return NPH_ERR_INVALID;
        }
        if (c.ref_position < 0 || c.ref_position + (int64_t)c.ref_seq_len + p.flank > INT32_MAX) {
            ctx->last_error = at + "ref_position + |ref_seq| + flank outside 0..INT32_MAX (the reference narrows the window's ends to int)";
            return NPH_ERR_INVALID;
        }
        const int64_t cs = c.ref_position - p.flank, ce = c.ref_position + (int64_t)c.ref_seq_len + p.flank;
        if (cs < p.region_start || ce > region_end) continue;                  // are_coordinates_valid: skipped
        const uint64_t key = ((uint64_t)(uint32_t)(int32_t)cs << 32) | c.ref_seq_len;
        auto it = win_of.find(key);
        uint32_t w;
        const int32_t win_off = (int32_t)(cs - p.region_start), len = (int32_t)(ce - cs + 1);
        if (it == win_of.end()) {
            w = (uint32_t)pl.wins.size();
            win_of.emplace(key, w);
            pl.wins.push_back(SvWin{(int32_t)cs, len, 0u, 0u, (uint32_t)pl.seqs.size(), 0u});
            pl.seqs.push_back(NphSetSeq{pl.bytes.size(), 0, (uint32_t)len, 0u});
            pl.bytes.insert(pl.bytes.end(), ref + win_off, ref + win_off + len);
            members.emplace_back();
        } else {
            w = it->second;
        }
        members[w].push_back((uint32_t)i);
        pl.cand_win[i] = w;
        // apply_variant: window.substr(flank, |ref_seq|) == ref_seq (the window holds all |ref_seq| bases)
        if (std::memcmp(ref + win_off + p.flank, alleles + c.ref_seq_off, c.ref_seq_len) != 0) continue;
        pl.applied[i] = 1;
        pl.cands[i].seq = (uint32_t)pl.seqs.size();
        pl.cands[i].alive = 0.0 < (double)p.score_threshold ? 1u : 0u;
        // the edited window: its first flank bases, alt_seq, the bases after ref_seq
        pl.seqs.push_back(NphSetSeq{pl.bytes.size(), 0, (uint32_t)(len - (int32_t)c.ref_seq_len + (int32_t)c.alt_seq_len), 0u});
        pl.bytes.insert(pl.bytes.end(), ref + win_off, ref + win_off + p.flank);
        pl.bytes.insert(pl.bytes.end(), alleles + c.alt_seq_off, alleles + c.alt_seq_off + c.alt_seq_len);
        pl.bytes.insert(pl.bytes.end(), ref + win_off + p.flank + c.ref_seq_len, ref + win_off + len);
    }
    for (size_t w = 0; w < pl.wins.size(); ++w) {
        pl.wins[w].cand_first = (uint32_t)pl.wcand.size();
        pl.wins[w].n_cand = (uint32_t)members[w].size();
        pl.wcand.insert(pl.wcand.end(), members[w].begin(), members[w].end());
    }
    return NPH_OK;
}

} // namespace

extern "C" int nph_screen_variants_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                         const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                         const char* ref_bases, size_t n_ref_bases,
                                         const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                         const nph_meth_record* records, size_t n_records,
                                         const nph_screen_list_params* params, const char* alleles, size_t n_allele_bytes,
                                         const nph_screen_candidate* candidates, size_t n_candidates, double indel_bias,
                                         const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                                         nph_screen_result* out, nph_screen_list_counts* counts_out)
{
    if (!ctx || !params || (n_candidates && (!candidates || !out)) || (n_allele_bytes && !alleles)) return NPH_ERR_INVALID;
    if (n_records && (!records || !first_event || (n_deltas_total && !event_deltas))) return NPH_ERR_INVALID;
    if (!ref_bases || !ev_start_time) return NPH_ERR_INVALID;
    if (n_ref_bases < 1 || n_ref_bases > 0x7fffffffu || (int64_t)params->region_start + (int64_t)n_ref_bases - 1 > INT32_MAX) return NPH_ERR_INVALID;
    const nph_screen_list_params p = *params;
    if (p.k < 1 || p.k > 8) { ctx->last_error = "k outside 1..8"; return NPH_ERR_INVALID; }
    if (p.flank < 0 || 2 * (int64_t)p.flank + 1 < (int64_t)p.k) { ctx->last_error = "2 * flank + 1 below k (a haplotype without a k-mer)"; return NPH_ERR_INVALID; }
    if (p.reads_per_round == 0) { ctx->last_error = "reads_per_round is 0"; return NPH_ERR_INVALID; }
    if (p.alignment_flags & ~(NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP)) { ctx->last_error = "unknown alignment_flags"; return NPH_ERR_INVALID; }
    std::vector<MethDev> md;
    NPH_TRY(nph_region_types(ctx, p.k, meth, n_records, alt_model_ids, md));
    SvPlan pl;
    NPH_TRY(plan_list(ctx, p, ref_bases, n_ref_bases, alleles, n_allele_bytes, candidates, n_candidates, pl));
    nph_screen_list_counts cnt{};
    cnt.n_candidates = n_candidates;
    cnt.n_windows = pl.wins.size();
    const auto finish = [&](const std::vector<uint64_t>& off, const std::vector<SvCand>& st) {
        for (size_t i = 0; i < n_candidates; ++i) {
            const uint32_t w = pl.cand_win[i];
            if (w == kNoSeq) { out[i] = nph_screen_result{std::nan(""), 0u, NPH_SCREEN_OUTSIDE}; continue; }
            const uint32_t nr = off.empty() ? 0u : (uint32_t)(off[w + 1] - off[w]);
            out[i] = pl.applied[i] ? nph_screen_result{st[i].total, nr, NPH_SCREEN_SCREENED} : nph_screen_result{0.0, nr, NPH_SCREEN_NOT_APPLIED};
        }
    };
    if (pl.wins.empty()) {
        finish({}, pl.cands);
        if (counts_out) *counts_out = cnt;
        nph_timing_staged(ctx, 0.f, 0);
        return NPH_OK;
    }
    nph_ctx::ScreenListState& ss = ctx->sl;
    const size_t n_wins = pl.wins.size(), n_seqs = pl.seqs.size(), n_cand = n_candidates;
    const auto run = [&]() -> int {
        NphSetTypes ty;
        NPH_TRY(nph_region_load_types(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, ref_bases, n_ref_bases, event_deltas,
                                      n_deltas_total, first_event, records, n_records, p.k, md, alt_model_ids, ty));
        cudaStream_t st = ctx->stream;
        SvWin* d_wins; NphSetSeq* d_seqs; uint32_t* d_wcand; uint8_t* d_bytes;
        NPH_TRY(nph_carve(ctx, ss.d_in, [&](NphArena& c) {
            d_wins = c.take<SvWin>(n_wins);
            d_seqs = c.take<NphSetSeq>(n_seqs);
            d_wcand = c.take<uint32_t>(pl.wcand.size());
            d_bytes = c.take<uint8_t>(pl.bytes.size());
        }));
        SvWinState* d_ws; uint64_t* d_job_cnt; uint64_t* d_job_off; uint64_t* d_scratch; SvCand* d_cands; uint32_t* d_alts; SvCounters* d_ctr;
        NPH_TRY(nph_carve(ctx, ss.d_state, [&](NphArena& c) {
            d_ws = c.take<SvWinState>(n_wins);
            d_job_cnt = c.take<uint64_t>(n_wins);
            d_job_off = c.take<uint64_t>(n_wins + 1);
            d_scratch = c.take<uint64_t>(nph_scan_scratch(n_wins));
            d_cands = c.take<SvCand>(n_cand);
            d_alts = c.take<uint32_t>(n_seqs);
            d_ctr = c.take<SvCounters>(1);
        }));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_wins, pl.wins.data(), sizeof(SvWin) * n_wins, cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_wcand, pl.wcand.data(), sizeof(uint32_t) * pl.wcand.size(), cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_cands, pl.cands.data(), sizeof(SvCand) * n_cand, cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_bytes, pl.bytes.data(), pl.bytes.size(), cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemsetAsync(d_ws, 0, sizeof(SvWinState) * n_wins, st));
        NPH_CUDA(ctx, cudaMemsetAsync(d_ctr, 0, sizeof(SvCounters), st));
        SvArgs a{ctx->region.ev.d_records.p, d_wins, d_seqs, d_wcand, d_cands, (uint32_t)n_wins, (int)p.k, (int)p.reads_per_round,
                 p.alignment_flags, (double)p.score_threshold};
        // the windows' reads
        std::vector<int2> bounds(n_wins);
        for (size_t w = 0; w < n_wins; ++w) bounds[w] = make_int2(pl.wins[w].cs, pl.wins[w].cs + pl.wins[w].len - 1);
        NphWindowReads wr;
        NPH_TRY(nph_window_reads(ctx, bounds, 0, wr));
        const std::vector<uint64_t>& off = wr.off;
        const uint64_t* d_off = wr.d_off;
        const NphWinPair* d_pairs = wr.d_pairs;
        uint64_t pool = 0;
        NPH_TRY(nph_set_ranks(ctx, pl.seqs, d_seqs, d_bytes, p.k, ty, d_alts, &pool));
        const unsigned wgrid = (unsigned)((n_wins + 255) / 256);
        float kernel_ms = 0.f;
        int launches = 6;
        for (;;) {
            sv_round_count_kernel<<<wgrid, 256, 0, st>>>(a, d_ws, d_off, d_job_cnt, d_alts);
            NPH_CUDA(ctx, cudaGetLastError());
            NPH_TRY(nph_scan_exclusive(ctx, d_job_cnt, (uint32_t)n_wins, d_job_off, d_scratch));
            uint64_t n_jobs = 0;
            NPH_CUDA(ctx, cudaMemcpyAsync(&n_jobs, d_job_off + n_wins, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
            NPH_CUDA(ctx, cudaStreamSynchronize(st));                 // read-back: the round's job count
            if (n_jobs == 0) break;
            NPH_TRY(nph_score_device_jobs(ctx, (size_t)n_jobs, (size_t)pool, indel_bias, [&]() -> int {
                sv_emit_kernel<<<wgrid, 256, 0, st>>>(a, d_ws, d_off, d_pairs, d_job_off, ctx->d_jobs.p, &d_ctr->events, ty, d_alts);
                NPH_CUDA(ctx, cudaGetLastError());
                return NPH_OK;
            }));
            sv_accumulate_kernel<<<wgrid, 256, 0, st>>>(a, d_ws, d_off, d_pairs, d_job_off, ctx->d_scores.p, d_ctr, ty, d_alts);
            NPH_CUDA(ctx, cudaGetLastError());
            float ms = 0.f; int nl = 0;
            if (nph_last_kernel_ms(ctx, &ms, &nl) == NPH_OK) { kernel_ms += ms; launches += nl + 4; }
            cnt.n_rounds += 1;
            cnt.n_jobs += n_jobs;
        }
        std::vector<SvCand> h_cands(n_cand);
        std::vector<uint32_t> h_alts(n_seqs);
        SvCounters h_ctr{};
        NPH_CUDA(ctx, cudaMemcpyAsync(h_cands.data(), d_cands, sizeof(SvCand) * n_cand, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(h_alts.data(), d_alts, sizeof(uint32_t) * n_seqs, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(&h_ctr, d_ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));
        finish(off, h_cands);
        cnt.n_dp_rows = h_ctr.events;
        cnt.n_reference_rows = h_ctr.ref_events;
        // what the device does not run: a candidate that does not apply scores the base set on both sides of every read (its total
        // stays 0); and the jobs every read of every applied candidate would take
        const double thr = (double)p.score_threshold;
        for (size_t w = 0; w < n_wins; ++w) {
            const SvWin& W = pl.wins[w];
            const uint64_t nb = 1u + (uint64_t)__builtin_popcount(h_alts[W.base_seq]);
            uint64_t per_read = nb;
            bool any = false;
            for (uint32_t c = 0; c < W.n_cand; ++c) {
                const uint32_t i = pl.wcand[W.cand_first + c];
                if (!pl.applied[i]) { if (0.0 < thr) cnt.n_reference_rows += 2u * nb * wr.rows[w]; continue; }
                any = true;
                per_read += 1u + (uint64_t)__builtin_popcount(h_alts[pl.cands[i].seq]);
            }
            if (any) cnt.n_jobs_without_exit += (off[w + 1] - off[w]) * per_read;
        }
        cnt.kernel_ms = kernel_ms;
        nph_timing_staged(ctx, kernel_ms, launches);
        return NPH_OK;
    };
    NPH_TRY(run());
    if (counts_out) *counts_out = cnt;
    return NPH_OK;
}
