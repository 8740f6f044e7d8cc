// meth_dev.cuh — a methylation alphabet and its recognition sites as the device kernels use them (ranks, not characters).
// Built and validated once by nph_meth_alphabet (methylation.cu); read by call-methylation (methylation.cu) and by the
// methylation-aware variant screening (variants.cu).
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
#endif
