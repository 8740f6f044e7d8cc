// meth_dev.cuh — a methylation alphabet and its recognition sites as the device kernels use them (ranks, not characters).
// Built and validated once by nph_meth_alphabet (methylation.cu); read by call-methylation (methylation.cu) and by the -q score
// sets of `nanopolish variants` (score_sets.cu: the edit screen, list screening and group calling).
#pragma once
#include "nph_internal.cuh"

struct MethDev {
    int32_t min_separation, min_flank, max_span, min_event_span, region_start, region_end;   // call-methylation's window (variants.cu: unused)
    uint32_t k, asize, n_sites, site_len;
    uint8_t rank_of[256];                                              // Alphabet::rank (unknown symbols rank 0)
    uint8_t comp_rank_of[256];                                         // rank(complement(symbol))
    char    site[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];           // recognition sites, characters
    uint8_t site_m_rank[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];    // ranks of the methylated site
    uint8_t site_mrc_rank[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];  // ranks of what stands on the other strand: reverse(methylated complement)
};

// The alphabet part of p into d (the window fields are zero): reads only k, alphabet_size, bases, complements, n_sites, site_len
// and the three site arrays.  NPH_ERR_INVALID for a malformed alphabet, NPH_ERR_UNSUPPORTED for sites that can overlap each other.
int nph_meth_alphabet(nph_ctx* ctx, const nph_meth_params& p, MethDev& d);

// The -q types of a call (score_sets.cu; nph_screen_load_methylation, nph_screen_variants_batch, nph_call_variant_groups_batch): at
// most NPH_SCREEN_MAX_TYPES, alt_model_ids present when there are types and records, each alphabet well formed and of k.
int nph_screen_types(nph_ctx* ctx, uint32_t k, const nph_screen_methylation& meth, size_t n_records, const uint32_t* alt_model_ids,
                     std::vector<MethDev>& md);
// A record of such a call: its model is a nucleotide model of k, and its model of each type (alt_model_ids[r * T + t]) is in range
// and of that type's alphabet.
int nph_screen_record_check(nph_ctx* ctx, uint32_t k, const std::vector<MethDev>& md, const uint32_t* alt_model_ids, size_t r,
                            const nph_meth_record& R);

// What the kernels of a call need to score a sequence as profile_hmm_score_set does: the set is the sequence, then its
// Alphabet::methylate copy of each -q type where that copy differs from it (generate_methylated_alternatives), in -q order.
struct NphSetTypes {
    const MethDev* types;               // T alphabets, -q order
    const uint32_t* alt_model;          // n_records x T: read->get_model(strand, type t)
    const float* tbl;                   // the context's log-sum table
    int T;                              // 0: no types, every set is its sequence alone
    double pen[NPH_SCREEN_MAX_TYPES + 1];   // log(n) for a set of n sequences, host libm
};
NphSetTypes nph_set_types(const MethDev* d_types, const uint32_t* d_alt_model, const float* tbl, int T);

// The -q front end of the one-shot region calls (list screening, group calling).  nph_region_types: a null meth is none, then
// nph_screen_types.  nph_region_load_types: nph_region_load with every record passing nph_screen_record_check, then the types'
// tables and model ids into ctx->region.d_types, described by st.
int nph_region_types(nph_ctx* ctx, uint32_t k, const nph_screen_methylation* meth, size_t n_records, const uint32_t* alt_model_ids,
                     std::vector<MethDev>& md);
int nph_region_load_types(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, const double* ev_start_time,
                          size_t n_events_total, const char* ref, size_t n_ref, const int16_t* deltas, size_t n_deltas, const int32_t* first_event,
                          const nph_meth_record* records, size_t n_records, uint32_t k, const std::vector<MethDev>& md,
                          const uint32_t* alt_model_ids, NphSetTypes& st);

// A sequence of a variable-length rank pool: its len characters at seq_off of the call's byte array; alternative a (0: the
// nucleotides, 1 + t: the methylated copy of type t) has its forward ranks at rank_off + a * 2 * nk and its reverse-strand ranks nk
// further, nk = len - k + 1.
struct NphSetSeq { uint64_t seq_off, rank_off; uint32_t len, pad; };
// The pool of seqs (list screening, group calling): assigns every rank_off and *pool, uploads seqs to d_seqs and writes the ranks of
// every alternative of every sequence into ctx->d_ranks, and into alts[i] bit t when the copy of type t differs from sequence i.
int nph_set_ranks(nph_ctx* ctx, std::vector<NphSetSeq>& seqs, NphSetSeq* d_seqs, const uint8_t* d_bytes, uint32_t k, const NphSetTypes& st,
                  uint32_t* d_alts, uint64_t* pool);

#ifdef __CUDACC__
// does a complete recognition site start at s[i]?  (is_motif_match reports complete sites only; the partial
// matches match_to_site also knows — string end, string inside a site — never have the full length for len >= site_len)
__device__ __forceinline__ int site_at(const MethDev& d, const uint8_t* __restrict__ s, int i, int n)
{
    if (i < 0 || i + (int)d.site_len > n) return -1;
    for (uint32_t q = 0; q < d.n_sites; ++q) {
        bool eq = true;
        for (uint32_t t = 0; t < d.site_len; ++t) eq = eq && (s[i + t] == (uint8_t)d.site[q][t]);
        if (eq) return (int)q;
    }
    return -1;
}

// ranks of the character at position t of methylate(s), s of n characters: fw on the forward strand, and rc where it lands in
// Alphabet::reverse_complement(methylate(s)), at index n - 1 - t.  A methylated site at q covers [q, q + rl) forward and
// [n - q - rl, n - q) reversed; recognition sites never overlap (nph_meth_alphabet), so at most one site covers a position.
__device__ __forceinline__ void meth_copy_rank(const MethDev& d, const uint8_t* __restrict__ s, int n, int t, uint32_t& fw, uint32_t& rc)
{
    const int rl = (int)d.site_len;
    for (int q0 = t - rl + 1; q0 <= t; ++q0) {
        const int q = site_at(d, s, q0, n);
        if (q < 0) continue;
        fw = d.site_m_rank[q][t - q0];
        rc = d.site_mrc_rank[q][q0 + rl - 1 - t];
        return;
    }
    fw = d.rank_of[s[t]];
    rc = d.comp_rank_of[s[t]];
}

// profile_hmm_score_set's set size of a sequence whose copy of type t differs from it where bit t of mask is set
__device__ __forceinline__ uint32_t set_size(uint32_t mask) { return 1u + (uint32_t)__popc(mask); }

// Appends the jobs of one sequence's set for one read: jb is the read's header (nph_window_job) with n_kmers filled in; the sequence
// with the record's model, then each copy of mask in -q order with the record's model of its type.  Alternative a's forward ranks
// start at rank_base + a * 2 * width, its reverse-strand ranks width further.
__device__ __forceinline__ nph_hmm_job* set_jobs(const NphSetTypes& st, nph_hmm_job jb, const nph_meth_record& R, uint32_t record,
                                                 uint32_t mask, uint64_t rank_base, uint32_t width, nph_hmm_job* out)
{
    for (int a = 0; a <= st.T; ++a) {
        if (a && !((mask >> (a - 1)) & 1u)) continue;
        jb.model_id = a ? st.alt_model[(size_t)record * st.T + (a - 1)] : R.model_id;
        jb.rank_off = rank_base + (uint64_t)a * 2u * width + (R.rc ? width : 0u);
        *out++ = jb;
    }
    return out;
}
#endif
