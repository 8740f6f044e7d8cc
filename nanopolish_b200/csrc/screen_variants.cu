// screen_variants.cu — screen_variants_by_score of `nanopolish variants --consensus` on the device: every candidate of a list
// screened in its own window in one call.
//
// Replaces, for a whole candidate list at once:
//   screen_variants_by_score                  ref: src/nanopolish_call_variants.cpp:364-402
//   AlignmentDB::get_event_subsequences       ref: src/alignment/nanopolish_alignment_db.cpp:172-221 (nph_event_subsequence, shared
//                                             with the edit screen, homopolymer fixing and all-support)
//   Haplotype::apply_variant on the window    ref: src/nanopolish_haplotype.cpp:33-75 (decided on the host, per candidate)
//   score_variant_thresholded                 ref: src/common/nanopolish_variant.cpp:765-799, with the -q sets of
//                                             generate_methylated_alternatives (:158-178) as nph_screen_load_methylation forms them
//
// Candidates with the same window (calling_start, |ref_seq|) share its reads and base haplotype.  Kernels, in the count -> scan ->
// fill shape of all_support.cu, then the round loop of variants.cu:
//   sv_pairs_kernel<false>  a warp per window, the records 32 at a time: the window's event sequences and their event rows
//   (nph_scan_exclusive: each window's first pair; one read-back sizes the pairs)
//   sv_pairs_kernel<true>   the same walk, writing the pairs {record, e1, e2} in record order
//   sv_ranks_kernel         a warp per (sequence, alternative): the k-mer ranks of both strands into a variable-length pool (the
//                           base window of every window, the edited window of every candidate that applies), and whether the
//                           methylated copy of each type differs from its sequence
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

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr uint32_t kNoSeq = 0xffffffffu;

struct SvPair { uint32_t record; int32_t e1, e2; };

// a window: [cs, cs + len - 1], its candidates wcand[cand_first, cand_first + n_cand), its base sequence
struct SvWin { int32_t cs, len; uint32_t cand_first, n_cand, base_seq, pad; };

// a sequence of the rank pool: window bytes [0, flank), the allele (al bytes at alleles[alt_off]), window bytes from flank + rl on.
// The base window has rl = al = 0.  Alternative a (0: nucleotides, 1 + t: methylated copy of type t) has its forward ranks at
// rank_off + a * 2 * nk and its reverse-strand ranks nk further, nk = L - k + 1.
struct SvSeq { uint64_t rank_off, alt_off; int32_t win_off, rl, al, L; };

// per candidate: the thresholded total, the reference's DP rows, its variant sequence (kNoSeq: outside the region or not applied),
// whether its total is inside the threshold at the start of the round
struct SvCand { double total; unsigned long long ref_rows; uint32_t seq, alive; };

struct SvWinState { uint32_t done, chunk; };

struct SvCounters { unsigned long long events, ref_events; unsigned int any_left; };

struct SvArgs {
    const nph_meth_record* records;
    const int32_t* dense;
    const int32_t* first_valid;
    const SvWin* wins;
    const SvSeq* seqs;
    const uint32_t* wcand;
    SvCand* cands;
    const uint8_t* ref;                 // the region reference
    const uint8_t* alleles;
    uint32_t n_records, n_wins, n_seqs;
    int flank, k, T, rpr;
    uint32_t flags;
    double threshold;
};

// the -q types (T = 0: none)
struct SvMeth {
    const MethDev* types;
    const uint32_t* alt_model;          // n_records x T
    uint32_t* alts;                     // per sequence: bit t set when its methylated copy of type t differs from it
    const float* tbl;
    double pen[NPH_SCREEN_MAX_TYPES + 1];   // log(n) for a set of n sequences, host libm
};

__device__ __forceinline__ uint32_t set_size(uint32_t mask) { return 1u + (uint32_t)__popc(mask); }

// FILL = false: per window the number of event sequences and their event rows; FILL = true: the pairs
template <bool FILL>
__global__ void __launch_bounds__(kThreads) sv_pairs_kernel(const SvArgs a, uint64_t* __restrict__ n_pairs, unsigned long long* __restrict__ sum_e,
                                                            const uint64_t* __restrict__ pair_off, SvPair* __restrict__ pairs)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    for (uint32_t wi = warp; wi < a.n_wins; wi += n_warps) {
        const int cs = a.wins[wi].cs, ce = cs + a.wins[wi].len - 1;
        uint64_t n = 0;
        unsigned long long e = 0;
        SvPair* out = FILL ? pairs + pair_off[wi] : nullptr;
        for (uint32_t base = 0; base < a.n_records; base += 32) {
            const uint32_t r = base + lane;
            int e1 = 0, e2 = 0;
            bool in = false;
            if (r < a.n_records) {
                const nph_meth_record R = a.records[r];
                in = nph_event_subsequence(R, a.dense + R.ref_off, a.first_valid[r], cs, ce, e1, e2);
            }
            const unsigned m = __ballot_sync(kFull, in);
            if (FILL && in) out[n + __popc(m & ((1u << lane) - 1u))] = SvPair{r, e1, e2};
            if (in) e += (unsigned long long)(e1 > e2 ? e1 - e2 : e2 - e1) + 1ull;
            n += __popc(m);
        }
        if (!FILL) {
            for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(kFull, e, o);
            if (lane == 0) { n_pairs[wi] = n; sum_e[wi] = e; }
        }
    }
}

// character i of sequence S
__device__ __forceinline__ uint8_t seq_char(const SvArgs& a, const SvSeq& S, int i)
{
    const uint8_t* w = a.ref + S.win_off;
    if (i < a.flank) return w[i];
    if (i < a.flank + S.al) return a.alleles[S.alt_off + (uint64_t)(i - a.flank)];
    return w[i - S.al + S.rl];
}

// site_at (meth_dev.cuh) on the characters of S
__device__ __forceinline__ int seq_site_at(const SvArgs& a, const MethDev& md, const SvSeq& S, int i)
{
    if (i < 0 || i + (int)md.site_len > S.L) return -1;
    for (uint32_t q = 0; q < md.n_sites; ++q) {
        bool eq = true;
        for (uint32_t t = 0; t < md.site_len && eq; ++t) eq = seq_char(a, S, i + (int)t) == (uint8_t)md.site[q][t];
        if (eq) return (int)q;
    }
    return -1;
}

// rank of character p of methylate(S) (fw) or of Alphabet::reverse_complement(methylate(S)) (!fw, p indexing that string): a
// methylated site at s covers [s, s + rl) forward and [L - s - rl, L - s) reversed.  Recognition sites never overlap
// (nph_meth_alphabet), so at most one site covers a position.
__device__ __forceinline__ uint32_t meth_rank(const SvArgs& a, const MethDev& md, const SvSeq& S, int p, bool fw)
{
    const int rl = (int)md.site_len;
    const int t = fw ? p : S.L - 1 - p;                          // the forward position the character comes from
    for (int s = t - rl + 1; s <= t; ++s) {
        const int q = seq_site_at(a, md, S, s);
        if (q < 0) continue;
        return fw ? md.site_m_rank[q][t - s] : md.site_mrc_rank[q][p - (S.L - s - rl)];
    }
    const uint8_t c = seq_char(a, S, t);
    return fw ? md.rank_of[c] : md.comp_rank_of[c];
}

// a warp per (sequence, alternative): both strands' ranks of every k-mer; an alternative's lanes also look for a site at each
// position, and a sequence with one gets its type's bit in sm.alts (generate_methylated_alternatives keeps a copy that differs)
__global__ void __launch_bounds__(kThreads) sv_ranks_kernel(const SvArgs a, uint32_t* __restrict__ pool, const SvMeth sm)
{
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * kWarps + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * kWarps;
    const uint32_t na = 1u + (uint32_t)a.T;
    for (uint32_t item = warp; item < a.n_seqs * na; item += n_warps) {
        const uint32_t si = item / na;
        const int alt = (int)(item % na);
        const SvSeq S = a.seqs[si];
        const int nk = S.L - a.k + 1;
        uint32_t* fw = pool + S.rank_off + (uint64_t)alt * 2u * (uint64_t)nk;
        uint32_t* rc = fw + nk;
        bool site = false;
        for (int p = lane; p < S.L; p += 32) {
            if (alt == 0) {
                if (p >= nk) continue;
                // HMMInputSequence::get_kmer_rank(p, k, rc) of the DNA alphabet (nph_dna_kmer_ranks)
                uint32_t f = 0, r = 0;
                for (int t = 0; t < a.k; ++t) {
                    f = f * 4u + nph_dna_code(seq_char(a, S, p + t));
                    r = r * 4u + (3u - nph_dna_code(seq_char(a, S, p + a.k - 1 - t)));
                }
                fw[p] = f; rc[p] = r;
                continue;
            }
            const MethDev& md = sm.types[alt - 1];
            site = site || seq_site_at(a, md, S, p) >= 0;
            if (p >= nk) continue;
            uint32_t f = 0, r = 0;
            for (int t = 0; t < a.k; ++t) {
                f = f * md.asize + meth_rank(a, md, S, p + t, true);
                r = r * md.asize + meth_rank(a, md, S, S.L - p - a.k + t, false);
            }
            fw[p] = f; rc[p] = r;
        }
        if (__any_sync(kFull, site) && lane == 0) atomicOr(sm.alts + si, 1u << (alt - 1));
    }
}

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

// appends the jobs of sequence si's set for one read: the sequence, then its methylated copies in type order
__device__ __forceinline__ nph_hmm_job* emit_set(const SvArgs& a, const SvMeth& sm, nph_hmm_job jb, const nph_meth_record& R, uint32_t record,
                                                 uint32_t si, nph_hmm_job* out)
{
    const SvSeq S = a.seqs[si];
    const uint32_t nk = (uint32_t)(S.L - a.k + 1);
    const uint32_t mask = a.T ? sm.alts[si] : 0u;
    jb.n_kmers = nk;
    for (int alt = 0; alt <= a.T; ++alt) {
        if (alt && !((mask >> (alt - 1)) & 1u)) continue;
        jb.model_id = alt ? sm.alt_model[(size_t)record * a.T + (alt - 1)] : R.model_id;
        jb.rank_off = S.rank_off + (uint64_t)alt * 2u * nk + (R.rc ? nk : 0u);
        *out++ = jb;
    }
    return out;
}

__global__ void sv_emit_kernel(const SvArgs a, const SvWinState* __restrict__ ws, const uint64_t* __restrict__ pair_off,
                               const SvPair* __restrict__ pairs, const uint64_t* __restrict__ job_off, nph_hmm_job* __restrict__ jobs,
                               unsigned long long* __restrict__ events, const SvMeth sm)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long ev = 0;
    if (wi < a.n_wins && ws[wi].chunk) {
        const SvWinState s = ws[wi];
        const SvWin W = a.wins[wi];
        const SvPair* rd = pairs + pair_off[wi] + s.done;
        nph_hmm_job* out = jobs + job_off[wi];
        for (uint32_t r = 0; r < s.chunk; ++r) {
            const SvPair P = rd[r];
            const nph_meth_record R = a.records[P.record];
            nph_hmm_job jb;
            jb.read = R.read;
            jb.event_start = (uint32_t)P.e1; jb.event_stop = (uint32_t)P.e2;
            jb.stride = R.rc ? -1 : 1;                    // EventAlignmentRecord::stride agrees with rc for every read the HMM accepts
            jb.rc = R.rc; jb.flags = (uint8_t)a.flags; jb.reserved = 0;
            nph_hmm_job* const first = out;
            out = emit_set(a, sm, jb, R, P.record, W.base_seq, out);
            for (uint32_t c = 0; c < W.n_cand; ++c) {
                const SvCand& C = a.cands[a.wcand[W.cand_first + c]];
                if (C.alive) out = emit_set(a, sm, jb, R, P.record, C.seq, out);
            }
            ev += (unsigned long long)(out - first) * ((unsigned long long)(P.e1 > P.e2 ? P.e1 - P.e2 : P.e2 - P.e1) + 1ull);
        }
    }
    for (int o = 16; o; o >>= 1) ev += __shfl_xor_sync(kFull, ev, o);
    if ((threadIdx.x & 31) == 0 && ev) atomicAdd(events, ev);
}

// thread per window: the round's reads in order, per read the base set's fold once and, for every live candidate, the sequential
// `if (fabs(total) < threshold) total += variant - base` (var_accumulate_kernel's arithmetic, NaN included)
__global__ void sv_accumulate_kernel(const SvArgs a, SvWinState* __restrict__ ws, const uint64_t* __restrict__ pair_off,
                                     const SvPair* __restrict__ pairs, const uint64_t* __restrict__ job_off, const float* __restrict__ scores,
                                     SvCounters* __restrict__ ctr, const SvMeth sm)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= a.n_wins) return;
    SvWinState s = ws[wi];
    if (!s.chunk) return;
    const SvWin W = a.wins[wi];
    const float* sc = scores + job_off[wi];
    const SvPair* rd = pairs + pair_off[wi] + s.done;
    const uint32_t nb = set_size(a.T ? sm.alts[W.base_seq] : 0u);
    unsigned long long ref_ev = 0;
    for (uint32_t r = 0; r < s.chunk; ++r) {
        // double base_score = profile_hmm_score_set(...) (a float); a set of one is its score
        const double base_score = (double)nph_score_set_fold(sc, nb, sm.pen[nb - 1], sm.tbl);
        sc += nb;
        const unsigned long long E = (unsigned long long)(rd[r].e1 > rd[r].e2 ? rd[r].e1 - rd[r].e2 : rd[r].e2 - rd[r].e1) + 1ull;
        for (uint32_t c = 0; c < W.n_cand; ++c) {
            SvCand& C = a.cands[a.wcand[W.cand_first + c]];
            if (!C.alive) continue;
            const uint32_t nc = set_size(a.T ? sm.alts[C.seq] : 0u);
            const double variant_score = (double)nph_score_set_fold(sc, nc, sm.pen[nc - 1], sm.tbl);
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

// the host's view of the list: windows, sequences, the windows' candidate lists, the initial candidate states
struct SvPlan {
    std::vector<SvWin> wins;
    std::vector<SvSeq> seqs;
    std::vector<uint32_t> wcand;
    std::vector<SvCand> cands;
    std::vector<uint32_t> cand_win;           // per candidate: its window (kNoSeq: outside the region)
    std::vector<uint8_t> applied;
    uint64_t pool = 0;                        // rank pool entries
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
            pl.seqs.push_back(SvSeq{0, 0, win_off, 0, 0, len});
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
        pl.seqs.push_back(SvSeq{0, c.alt_seq_off, win_off, (int32_t)c.ref_seq_len, (int32_t)c.alt_seq_len,
                                len - (int32_t)c.ref_seq_len + (int32_t)c.alt_seq_len});
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
    static const nph_screen_methylation none{};
    const nph_screen_methylation& mt = meth ? *meth : none;
    std::vector<MethDev> md;
    NPH_TRY(nph_screen_types(ctx, p.k, mt, n_records, alt_model_ids, md));
    const int T = (int)md.size();
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
        NPH_TRY(nph_reads_load(ctx, reads, n_reads, ev_mean, ev_start_time, n_events_total));
        // records index the event deltas, as the edit screen's do
        NPH_TRY(nph_event_records_load(ctx, ss.ev, ref_bases, n_ref_bases, n_deltas_total, true, event_deltas, first_event, nullptr, 0,
                                       records, n_records, 0x3fffffffu, [&](size_t r, const nph_meth_record& R) {
            return nph_screen_record_check(ctx, p.k, md, alt_model_ids, r, R);
        }));
        cudaStream_t st = ctx->stream;
        SvWin* d_wins; SvSeq* d_seqs; uint32_t* d_wcand; uint8_t* d_alleles; MethDev* d_meth; uint32_t* d_alt_models;
        NPH_TRY(nph_carve(ctx, ss.d_in, [&](NphArena& c) {
            d_wins = c.take<SvWin>(n_wins);
            d_seqs = c.take<SvSeq>(n_seqs);
            d_wcand = c.take<uint32_t>(pl.wcand.size());
            d_alleles = c.take<uint8_t>(n_allele_bytes + 1);
            d_meth = c.take<MethDev>((size_t)T + 1);
            d_alt_models = c.take<uint32_t>(n_records * (size_t)T + 1);
        }));
        uint64_t* d_n; unsigned long long* d_sum_e; uint64_t* d_off; uint64_t* d_job_cnt; uint64_t* d_job_off; uint64_t* d_scratch;
        NPH_TRY(nph_carve(ctx, ss.d_counts, [&](NphArena& c) {
            d_n = c.take<uint64_t>(n_wins);
            d_sum_e = c.take<unsigned long long>(n_wins);
            d_off = c.take<uint64_t>(n_wins + 1);
            d_job_cnt = c.take<uint64_t>(n_wins);
            d_job_off = c.take<uint64_t>(n_wins + 1);
            d_scratch = c.take<uint64_t>(nph_scan_scratch(n_wins));
        }));
        SvWinState* d_ws; SvCand* d_cands; uint32_t* d_alts; SvCounters* d_ctr;
        NPH_TRY(nph_carve(ctx, ss.d_state, [&](NphArena& c) {
            d_ws = c.take<SvWinState>(n_wins);
            d_cands = c.take<SvCand>(n_cand);
            d_alts = c.take<uint32_t>(n_seqs);
            d_ctr = c.take<SvCounters>(1);
        }));
        // the rank pool: per sequence (1 + T) alternatives x both strands
        for (SvSeq& s : pl.seqs) {
            s.rank_off = pl.pool;
            pl.pool += (uint64_t)(1 + T) * 2u * (uint64_t)(s.L - (int)p.k + 1);
        }
        NPH_CUDA(ctx, cudaMemcpyAsync(d_wins, pl.wins.data(), sizeof(SvWin) * n_wins, cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_seqs, pl.seqs.data(), sizeof(SvSeq) * n_seqs, cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_wcand, pl.wcand.data(), sizeof(uint32_t) * pl.wcand.size(), cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(d_cands, pl.cands.data(), sizeof(SvCand) * n_cand, cudaMemcpyHostToDevice, st));
        if (n_allele_bytes) NPH_CUDA(ctx, cudaMemcpyAsync(d_alleles, alleles, n_allele_bytes, cudaMemcpyHostToDevice, st));
        if (T) NPH_CUDA(ctx, cudaMemcpyAsync(d_meth, md.data(), sizeof(MethDev) * T, cudaMemcpyHostToDevice, st));
        if (T && n_records) NPH_CUDA(ctx, cudaMemcpyAsync(d_alt_models, alt_model_ids, sizeof(uint32_t) * n_records * T, cudaMemcpyHostToDevice, st));
        NPH_CUDA(ctx, cudaMemsetAsync(d_ws, 0, sizeof(SvWinState) * n_wins, st));
        NPH_CUDA(ctx, cudaMemsetAsync(d_alts, 0, sizeof(uint32_t) * n_seqs, st));
        NPH_CUDA(ctx, cudaMemsetAsync(d_ctr, 0, sizeof(SvCounters), st));
        const int32_t* dense;
        const int32_t* first_valid;
        NPH_TRY(nph_event_records_expand(ctx, ss.ev, &dense, &first_valid));
        SvArgs a{ss.ev.d_records.p, dense, first_valid, d_wins, d_seqs, d_wcand, d_cands, ss.ev.d_ref.p, d_alleles, (uint32_t)n_records,
                 (uint32_t)n_wins, (uint32_t)n_seqs, p.flank, (int)p.k, T, (int)p.reads_per_round, p.alignment_flags, (double)p.score_threshold};
        SvMeth sm{};
        sm.types = d_meth; sm.alt_model = d_alt_models; sm.alts = d_alts; sm.tbl = ctx->d_logsum.p;
        for (int n = 1; n <= 1 + T; ++n) sm.pen[n - 1] = log((double)n);      // profile_hmm_score_set's log(num_models), host libm
        // the windows' reads
        const int grid = (int)std::min<size_t>((n_wins + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 8);
        sv_pairs_kernel<false><<<grid, kThreads, 0, st>>>(a, d_n, d_sum_e, nullptr, nullptr);
        NPH_CUDA(ctx, cudaGetLastError());
        NPH_TRY(nph_scan_exclusive(ctx, d_n, (uint32_t)n_wins, d_off, d_scratch));
        std::vector<uint64_t> off(n_wins + 1);
        NPH_CUDA(ctx, cudaMemcpyAsync(off.data(), d_off, sizeof(uint64_t) * (n_wins + 1), cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaStreamSynchronize(st));                     // the one read-back that sizes the pairs
        const uint64_t n_pairs = off[n_wins];
        NPH_TRY(nph_reserve(ctx, ss.d_pairs, sizeof(SvPair) * (size_t)(n_pairs + 1)));
        SvPair* d_pairs = reinterpret_cast<SvPair*>(ss.d_pairs.p);
        if (n_pairs) {
            sv_pairs_kernel<true><<<grid, kThreads, 0, st>>>(a, nullptr, nullptr, d_off, d_pairs);
            NPH_CUDA(ctx, cudaGetLastError());
        }
        NPH_TRY(nph_reserve(ctx, ctx->d_ranks, (size_t)pl.pool));
        const size_t n_items = n_seqs * (size_t)(1 + T);
        const int rgrid = (int)std::min<size_t>((n_items + kWarps - 1) / kWarps, (size_t)ctx->sm_count * 16);
        sv_ranks_kernel<<<rgrid, kThreads, 0, st>>>(a, ctx->d_ranks.p, sm);
        NPH_CUDA(ctx, cudaGetLastError());
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
            NPH_TRY(nph_score_device_jobs(ctx, (size_t)n_jobs, (size_t)pl.pool, indel_bias, [&]() -> int {
                sv_emit_kernel<<<wgrid, 256, 0, st>>>(a, d_ws, d_off, d_pairs, d_job_off, ctx->d_jobs.p, &d_ctr->events, sm);
                NPH_CUDA(ctx, cudaGetLastError());
                return NPH_OK;
            }));
            sv_accumulate_kernel<<<wgrid, 256, 0, st>>>(a, d_ws, d_off, d_pairs, d_job_off, ctx->d_scores.p, d_ctr, sm);
            NPH_CUDA(ctx, cudaGetLastError());
            float ms = 0.f; int nl = 0;
            if (nph_last_kernel_ms(ctx, &ms, &nl) == NPH_OK) { kernel_ms += ms; launches += nl + 4; }
            cnt.n_rounds += 1;
            cnt.n_jobs += n_jobs;
        }
        std::vector<SvCand> h_cands(n_cand);
        std::vector<uint32_t> h_alts(n_seqs);
        std::vector<unsigned long long> h_sum_e(n_wins);
        SvCounters h_ctr{};
        NPH_CUDA(ctx, cudaMemcpyAsync(h_cands.data(), d_cands, sizeof(SvCand) * n_cand, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(h_alts.data(), d_alts, sizeof(uint32_t) * n_seqs, cudaMemcpyDeviceToHost, st));
        NPH_CUDA(ctx, cudaMemcpyAsync(h_sum_e.data(), d_sum_e, sizeof(unsigned long long) * n_wins, cudaMemcpyDeviceToHost, st));
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
                if (!pl.applied[i]) { if (0.0 < thr) cnt.n_reference_rows += 2u * nb * h_sum_e[w]; continue; }
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
