// score_sets.cu — the -q score sets of `nanopolish variants`: profile_hmm_score_set over a sequence and its methylated copies
// (generate_methylated_alternatives, ref: src/common/nanopolish_variant.cpp:158-178), for the edit screen (variants.cu), list
// screening (screen_variants.cu) and group calling (call_variants.cu).
//
// Here: the checks of the types and of each record's models, the set description the kernels read (NphSetTypes, with
// profile_hmm_score_set's log(n) from host libm), the -q front end of the two one-shot calls, and the rank pool of their
// variable-length sequences.  The device helpers (site_at, meth_copy_rank, set_size, set_jobs) are in meth_dev.cuh; the edit screen
// keeps its own fixed pool and buffers, since other calls may run between its staged load, run and fetch.
//
// Kernel:
//   set_ranks_kernel   a warp per (sequence, alternative): both strands' k-mer ranks, and whether the methylated copy differs from
//                      its sequence (a recognition site anywhere in it)
#include "nph_internal.cuh"
#include "meth_dev.cuh"
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;

__global__ void set_ranks_kernel(const NphSetSeq* __restrict__ seqs, uint32_t n_seqs, const uint8_t* __restrict__ bytes, int k,
                                 uint32_t* __restrict__ pool, const NphSetTypes st, uint32_t* __restrict__ alts)
{
    const int lane = threadIdx.x & 31;
    const uint32_t na = 1u + (uint32_t)st.T;
    for (uint32_t item = blockIdx.x * kWarps + (threadIdx.x >> 5); item < n_seqs * na; item += gridDim.x * kWarps) {
        const NphSetSeq S = seqs[item / na];
        const int a = (int)(item % na);
        const uint8_t* s = bytes + S.seq_off;
        const int L = (int)S.len, nk = L - k + 1;
        uint32_t* fw = pool + S.rank_off + (uint64_t)a * 2u * (uint64_t)nk;
        uint32_t* rc = fw + nk;
        bool site = false;
        for (int p = lane; p < L; p += 32) {
            if (a == 0) {
                if (p >= nk) continue;
                uint8_t c[8];
                for (int i = 0; i < k; ++i) c[i] = nph_dna_code(s[p + i]);
                nph_dna_kmer_ranks(c, 0, k, fw[p], rc[p]);
                continue;
            }
            const MethDev& md = st.types[a - 1];
            site = site || site_at(md, s, p, L) >= 0;
            if (p >= nk) continue;
            // the reverse-strand k-mer at L - p - k holds the same characters back to front: character p + i weighs asize^i
            uint32_t f = 0, r = 0, w = 1;
            for (int i = 0; i < k; ++i) {
                uint32_t cf, cr;
                meth_copy_rank(md, s, L, p + i, cf, cr);
                f = f * md.asize + cf;
                r += cr * w;
                w *= md.asize;
            }
            fw[p] = f; rc[p] = r;
        }
        if (__any_sync(0xffffffffu, site) && lane == 0) atomicOr(alts + item / na, 1u << (a - 1));
    }
}

} // namespace

int nph_screen_types(nph_ctx* ctx, uint32_t k, const nph_screen_methylation& meth, size_t n_records, const uint32_t* alt_model_ids,
                     std::vector<MethDev>& md)
{
    const uint32_t T = meth.n_types;
    if (T > NPH_SCREEN_MAX_TYPES) { ctx->last_error = "nph_screen_methylation: more than NPH_SCREEN_MAX_TYPES types"; return NPH_ERR_INVALID; }
    if (T && n_records && !alt_model_ids) return NPH_ERR_INVALID;
    md.assign(T, MethDev{});
    for (uint32_t t = 0; t < T; ++t) {
        NPH_TRY(nph_meth_alphabet(ctx, meth.alphabets[t], md[t]));
        if (md[t].k != k) { ctx->last_error = "nph_screen_methylation: type " + std::to_string(t) + " has k != params.k"; return NPH_ERR_INVALID; }
    }
    return NPH_OK;
}

int nph_screen_record_check(nph_ctx* ctx, uint32_t k, const std::vector<MethDev>& md, const uint32_t* alt_model_ids, size_t r,
                            const nph_meth_record& R)
{
    const size_t T = md.size();
    const DevModel& mod = ctx->models[R.model_id];
    if (mod.k != k || mod.alphabet_size != 4) { ctx->last_error = "screening record " + std::to_string(r) + ": its model is not a nucleotide model of k = params.k"; return NPH_ERR_INVALID; }
    for (size_t t = 0; t < T; ++t) {
        const uint32_t id = alt_model_ids[r * T + t];
        if (id >= ctx->models.size() || ctx->models[id].k != md[t].k || ctx->models[id].alphabet_size != md[t].asize) {
            ctx->last_error = "screening record " + std::to_string(r) + ": its model of methylation type " + std::to_string(t) +
                              " is out of range or not a model of that alphabet";
            return NPH_ERR_INVALID;
        }
    }
    return NPH_OK;
}

NphSetTypes nph_set_types(const MethDev* d_types, const uint32_t* d_alt_model, const float* tbl, int T)
{
    NphSetTypes st{d_types, d_alt_model, tbl, T, {}};
    for (int n = 1; n <= NPH_SCREEN_MAX_TYPES + 1; ++n) st.pen[n - 1] = log((double)n);     // profile_hmm_score_set's log(num_models)
    return st;
}

int nph_region_types(nph_ctx* ctx, uint32_t k, const nph_screen_methylation* meth, size_t n_records, const uint32_t* alt_model_ids,
                     std::vector<MethDev>& md)
{
    static const nph_screen_methylation none{};
    return nph_screen_types(ctx, k, meth ? *meth : none, n_records, alt_model_ids, md);
}

int nph_region_load_types(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, const double* ev_start_time,
                          size_t n_events_total, const char* ref, size_t n_ref, const int16_t* deltas, size_t n_deltas, const int32_t* first_event,
                          const nph_meth_record* records, size_t n_records, uint32_t k, const std::vector<MethDev>& md,
                          const uint32_t* alt_model_ids, NphSetTypes& st)
{
    NPH_TRY(nph_region_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total, ref, n_ref, deltas, n_deltas, first_event, records,
                            n_records, [&](size_t r, const nph_meth_record& R) { return nph_screen_record_check(ctx, k, md, alt_model_ids, r, R); }));
    const size_t T = md.size();
    MethDev* d_meth; uint32_t* d_alt_models;
    NPH_TRY(nph_carve(ctx, ctx->region.d_types, [&](NphArena& c) {
        d_meth = c.take<MethDev>(T + 1);
        d_alt_models = c.take<uint32_t>(n_records * T + 1);
    }));
    if (T) NPH_CUDA(ctx, cudaMemcpyAsync(d_meth, md.data(), sizeof(MethDev) * T, cudaMemcpyHostToDevice, ctx->stream));
    if (T && n_records) NPH_CUDA(ctx, cudaMemcpyAsync(d_alt_models, alt_model_ids, sizeof(uint32_t) * n_records * T, cudaMemcpyHostToDevice, ctx->stream));
    st = nph_set_types(d_meth, d_alt_models, ctx->d_logsum.p, (int)T);
    return NPH_OK;
}

int nph_set_ranks(nph_ctx* ctx, std::vector<NphSetSeq>& seqs, NphSetSeq* d_seqs, const uint8_t* d_bytes, uint32_t k, const NphSetTypes& st,
                  uint32_t* d_alts, uint64_t* pool)
{
    cudaStream_t s = ctx->stream;
    uint64_t n = 0;
    for (NphSetSeq& q : seqs) {
        q.rank_off = n;
        n += (uint64_t)(1 + st.T) * 2u * (uint64_t)(q.len - k + 1);
    }
    *pool = n;
    NPH_TRY(nph_reserve(ctx, ctx->d_ranks, (size_t)n));
    NPH_CUDA(ctx, cudaMemcpyAsync(d_seqs, seqs.data(), sizeof(NphSetSeq) * seqs.size(), cudaMemcpyHostToDevice, s));
    NPH_CUDA(ctx, cudaMemsetAsync(d_alts, 0, sizeof(uint32_t) * seqs.size(), s));
    const size_t n_items = seqs.size() * (size_t)(1 + st.T);
    const int grid = (int)std::min<size_t>((n_items + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 16);
    set_ranks_kernel<<<grid, kThreads, 0, s>>>(d_seqs, (uint32_t)seqs.size(), d_bytes, (int)k, ctx->d_ranks.p, st, d_alts);
    NPH_CUDA(ctx, cudaGetLastError());
    return NPH_OK;
}
