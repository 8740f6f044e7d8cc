// hmm_viterbi_kernel.cuh — the device side of K3 (Viterbi alignment, SURVEY.md section 8f N1) as a warp-level
// function, shared by the batch kernel (hmm_viterbi.cu: one profile_hmm_align per job) and the eventalign chain
// kernel (eventalign_chain.cu: a read's whole segment chain without leaving the device).
//   profile_hmm_align_r9          ref: src/hmm/nanopolish_profile_hmm_r9.cpp:73-204
//   ProfileHMMViterbiOutputR9     ref: src/hmm/nanopolish_profile_hmm_r9.inl:130-197
#pragma once
#include "hmm_wavefront.cuh"
#include "exact_math.cuh"

namespace nph_vit {

constexpr unsigned kFull = 0xffffffffu;
enum { MV_SAME_M = 0, MV_PREV_M = 1, MV_SAME_B = 2, MV_PREV_B = 3, MV_PREV_K = 4, MV_SOFT = 5 };

// one profile_hmm_align call, as the warp sees it
struct VitJob {
    const float* lv;          // drift-scaled levels of the read (first event of the READ, not of the window)
    DevRead rd;
    float2 tr;                // (lp_mm_self, lp_mm_next) of the read
    DevModelView mv;
    const uint32_t* rk;       // K k-mer ranks, strand-resolved
    int K, E, stride;
    long long e_first;        // HMMInputData::event_start_idx
    bool pre_clip;
};
// per-warp scratch: Gaussians (kpad float4), strip-edge columns M, B, K (untouched for one strip),
// movement codes ((steps + 1) * 32 * C uint16) in global memory; a 2 KB tile in shared memory
struct VitScratch {
    float4* params;
    EdgeRows edge;
    uint16_t* trace;
    uint16_t* tile;           // shared memory, 32 x 32 movement codes: the backtrack's staging corner
};

// running max with the reference's tie rule: a later candidate that equals the max takes the label
__device__ __forceinline__ void vmax(float& mx, int& from, float x, int idx)
{
    mx = x > mx ? x : mx;
    from = (mx == x) ? idx : from;
}

// Fill, backtrack and forward replay of one job by one warp.  Returns the number of states written to out[0..n) in
// ascending event order (0 where the reference would trip an assert: the path enters a -inf cell or block 0, or cap is
// too small); *last_v_out = l_fm of the last state (lane 0's value is the meaningful one).  Requires E >= 2.
// REPLAY = false (the eventalign chain, which never reads l_fm): no forward replay; the states stay where the backtrack
// put them, out[cap - n .. cap) in ascending event order with l_fm = 0, and the one way a path can enter a -inf cell — a
// FROM_SOFT that is not the legitimate start (every -inf cell records FROM_SOFT, and finite transitions out of finite
// cells stay finite) — is caught during the backtrack.
template <int C, bool REPLAY = true>
__device__ __forceinline__ int viterbi_align(const HmmConsts& c, const float* __restrict__ flank, const VitJob& j, const VitScratch& sc,
                                             nph_align_state* out, int cap, float* last_v_out, int lane)
{
    constexpr int STRIP = 32 * C;
    const float NEG = -CUDART_INF_F;
    const float lp_mk = c.lp_mk, lp_mb = c.lp_mb, lp_bb = c.lp_bb, lp_bk = c.lp_bk;
    const float lp_bm_next = c.lp_bm_next, lp_bm_self = c.lp_bm_self, lp_kk = c.lp_kk, lp_km = c.lp_km;
    const float lp_mm_self = j.tr.x, lp_mm_next = j.tr.y;
    const int K = j.K, E = j.E, stride = j.stride;
    const bool pre_clip = j.pre_clip;
    float4* const my_params = sc.params;
    uint16_t* const trace = sc.trace;
    const nph_wave_geom geo = nph_wave_geometry(K, E, C, 32, true);
    const int P = geo.P;
    fill_job_gaussians<32>(my_params, j.mv, j.rd, j.rk, K, geo.kpad, lane, c.log_inv_sqrt_2pi);
    __syncwarp();

    const float* lv = j.lv;
    const long long e_first = j.e_first;
    const int total_steps = geo.total_steps();

    // ---------------------------------- fill ----------------------------------
    float mu[C], sd[C], cc[C], ry[C], Mp[C], Bp[C], Kp[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { mu[c] = 0.f; sd[c] = 1.f; cc[c] = 0.f; ry[c] = 1.f; Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; }
    float Lm_prev = NEG, Lb_prev = NEG, Lk_prev = NEG;
    const int n_strips = geo.n_strips, last_strip = geo.last_strip();
    int r = 1 - lane, s = 0;
    float x_next = 0.f;
    if (r == 1) x_next = lv[e_first];
    float em_next = NEG, eb_next = NEG, ek_next = NEG;

    for (int g = 0; g < total_steps; ++g) {
        float Lm = __shfl_up_sync(kFull, Mp[C - 1], 1);
        float Lb = __shfl_up_sync(kFull, Bp[C - 1], 1);
        float Lk = __shfl_up_sync(kFull, Kp[C - 1], 1);
        if (lane == 0) { Lm = em_next; Lb = eb_next; Lk = ek_next; }
        const bool in_strip = (r >= 1) && (s < n_strips);
        const int col0 = s * STRIP + lane * C;
        const bool live = in_strip && (r <= E) && (col0 < K);
        const float x = x_next;
        if (in_strip && r == 1) {
#pragma unroll
            for (int c = 0; c < C; ++c) { Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; }
            Lm_prev = NEG; Lb_prev = NEG; Lk_prev = NEG;
            if (col0 < K) load_columns<C>(my_params, col0, mu, sd, cc, ry);
        }
        {
            int rn = r + 1, sn = s;
            if (rn > P) { rn = 1; sn = s + 1; }
            if (rn >= 1 && rn <= E && sn < n_strips) {
                x_next = lv[e_first + (long long)(rn - 1) * stride];
                if (lane == 0 && sn > 0) { em_next = sc.edge.a[rn]; eb_next = sc.edge.b[rn]; ek_next = sc.edge.c[rn]; }
            }
        }
        uint16_t tcode[C];
#pragma unroll
        for (int c = 0; c < C; ++c) tcode[c] = 0;
        if (live) {
            float soft = NEG;
            if (col0 == 0 && (r == 1 || pre_clip)) soft = __fadd_rn(0.0f, flank[r - 1]);
            float lm_prev = Lm_prev, lb_prev = Lb_prev, lk_prev = Lk_prev;
            float lm_cur = Lm, lb_cur = Lb, lk_cur = Lk;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const float em = log_gauss(x, mu[c], sd[c], cc[c], ry[c]);
                // MATCH: six candidates in movement order
                float m = __fadd_rn(lp_mm_self, Mp[c]);
                int fm = MV_SAME_M;
                vmax(m, fm, __fadd_rn(lp_mm_next, lm_prev), MV_PREV_M);
                vmax(m, fm, __fadd_rn(lp_bm_self, Bp[c]), MV_SAME_B);
                vmax(m, fm, __fadd_rn(lp_bm_next, lb_prev), MV_PREV_B);
                vmax(m, fm, __fadd_rn(lp_km, lk_prev), MV_PREV_K);
                // the soft-clip candidate is -inf everywhere but in column 0: there it takes part in the chain, elsewhere it can
                // only win the label when every candidate is -inf (a later equal candidate takes the label)
                if (c == 0) vmax(m, fm, soft, MV_SOFT);
                else fm = (m == NEG) ? MV_SOFT : fm;
                m = __fadd_rn(m, em);
                // BAD EVENT: {same M, -inf, same B, -inf, -inf, -inf}.  The -inf candidates between and after the live ones
                // only matter when the running max is still -inf after the last live one: then the last index (SOFT) holds
                // the label; labels they would take earlier are overwritten by the next live candidate (x >= -inf always
                // updates an all--inf chain).
                float b = __fadd_rn(lp_mb, Mp[c]);
                int fb = MV_SAME_M;
                vmax(b, fb, __fadd_rn(lp_bb, Bp[c]), MV_SAME_B);
                fb = (b == NEG) ? MV_SOFT : fb;
                // K-MER SKIP: {-inf, prev M, -inf, prev B, prev K, -inf} of the same row
                float kk = __fadd_rn(lp_mk, lm_cur);
                int fk = MV_PREV_M;
                vmax(kk, fk, __fadd_rn(lp_bk, lb_cur), MV_PREV_B);
                vmax(kk, fk, __fadd_rn(lp_kk, lk_cur), MV_PREV_K);
                fk = (kk == NEG) ? MV_SOFT : fk;

                lm_prev = Mp[c]; lb_prev = Bp[c]; lk_prev = Kp[c];
                lm_cur = m; lb_cur = b; lk_cur = kk;
                Mp[c] = m; Bp[c] = b; Kp[c] = kk;
                tcode[c] = (uint16_t)(fm | (fb << 3) | (fk << 6));
            }
            Lm_prev = Lm; Lb_prev = Lb; Lk_prev = Lk;
            if (lane == 31 && s < last_strip) { sc.edge.a[r] = Mp[C - 1]; sc.edge.b[r] = Bp[C - 1]; sc.edge.c[r] = Kp[C - 1]; }
        }
        // trace line of this step: one contiguous 64*C bytes per warp
#pragma unroll
        for (int c = 0; c < C; ++c) trace[(size_t)g * STRIP + lane * C + c] = tcode[c];
        r += 1;
        if (r > P) { r = 1; s += 1; }
        if (n_strips > 1) __syncwarp();
    }
    __syncwarp();

    // ---------------------------------- backtrack (all lanes walk the same path) ----------------------------------
    int n = 0, status = 0;
    {
        int row = E, kmer = K - 1, st = 2;        // state codes: 0 K, 1 B, 2 M (column % 3 in the reference)
        // The path moves at most one row up and one k-mer left per state, so the next 32 states lie inside the 32 x 32
        // corner of the trace that ends at (row, kmer): the warp stages that corner in shared memory with 32
        // independent loads per lane (lane = k-mer column, 64 contiguous bytes per row) instead of paying one dependent
        // L2 round trip per state.
        bool ended_soft = false;
        int row0 = 0, kmer0 = -1;                 // corner currently staged: rows (row0-32, row0], k-mers (kmer0-32, kmer0]
        while (row > 0) {
            if (kmer0 < 0 || row <= row0 - 32 || kmer <= kmer0 - 32) {
                __syncwarp();
                row0 = row; kmer0 = kmer;
                const int km = kmer0 - lane;
                if (km >= 0) {
                    const int sidx = km / STRIP, rel = km - sidx * STRIP;
                    const uint16_t* src = trace + ((size_t)sidx * P + rel / C) * STRIP + rel;
#pragma unroll 8
                    for (int i = 0; i < 32; ++i) {
                        const int rw = row0 - i;
                        if (rw >= 1) sc.tile[i * 32 + lane] = __ldcg(src + (size_t)(rw - 1) * STRIP);
                    }
                }
                __syncwarp();
            }
            const uint32_t code = sc.tile[(row0 - row) * 32 + (kmer0 - kmer)];
            const int mvt = (st == 2) ? (code & 7) : (st == 1) ? ((code >> 3) & 7) : ((code >> 6) & 7);
            if (n >= cap) { status = 3; break; }
            if (lane == 0) {
                nph_align_state a;
                a.event_idx = (uint32_t)(e_first + (long long)(row - 1) * stride);
                a.kmer_idx = (uint32_t)kmer;
                a.l_fm = 0.f;
                a.state = (st == 2) ? 'M' : (st == 1) ? 'B' : 'K';
                a.reserved[0] = (uint8_t)mvt; a.reserved[1] = 0; a.reserved[2] = 0;
                out[cap - 1 - n] = a;
            }
            ++n;
            if (mvt == MV_SOFT) {
                if (!REPLAY && !(st == 2 && kmer == 0 && (row == 1 || pre_clip))) status = 2;
                ended_soft = true;
                break;
            }
            int nst = 2;
            switch (mvt) {
                case MV_SAME_M: nst = 2; break;
                case MV_PREV_M: kmer -= 1; nst = 2; break;
                case MV_SAME_B: nst = 1; break;
                case MV_PREV_B: kmer -= 1; nst = 1; break;
                case MV_PREV_K: kmer -= 1; nst = 0; break;
            }
            if (st != 0) row -= 1;               // a k-mer skip is silent
            st = nst;
            if (kmer < 0) { status = 2; break; } // block 0: the reference asserts
        }
        if (!REPLAY && !status && !ended_soft) status = 2;    // walked off row 1 without reaching the start state
    }
    __syncwarp();
    if (!REPLAY) {
        *last_v_out = NEG;
        return status ? 0 : n;
    }

    // ---------------------------------- replay forwards: l_fm of every state ----------------------------------
    float last_v = NEG;
    if (!status && lane == 0) {
        float v = NEG;
        for (int i = 0; i < n; ++i) {
            nph_align_state a = out[cap - n + i];
            const int mvt = a.reserved[0];
            const int row = (int)(((long long)a.event_idx - e_first) * stride) + 1;
            float x5 = NEG;
            if (mvt == MV_SOFT) {
                // legitimate only as the first state: MATCH of k-mer 0 at row 1 or with PRE_CLIP; anything else is a -inf cell
                if (i == 0 && a.state == 'M' && a.kmer_idx == 0 && (row == 1 || pre_clip)) x5 = __fadd_rn(0.0f, flank[row - 1]);
                else { status = 2; break; }
            }
            float t;
            if (a.state == 'M') {
                const float tr_ = mvt == MV_SAME_M ? lp_mm_self : mvt == MV_PREV_M ? lp_mm_next : mvt == MV_SAME_B ? lp_bm_self
                                  : mvt == MV_PREV_B ? lp_bm_next : lp_km;
                t = (mvt == MV_SOFT) ? x5 : __fadd_rn(tr_, v);
                const float4 g4 = my_params[a.kmer_idx];
                t = __fadd_rn(t, log_gauss(lv[a.event_idx], g4.x, g4.y, g4.z, g4.w));
            } else if (a.state == 'B') {
                t = __fadd_rn(mvt == MV_SAME_M ? lp_mb : lp_bb, v);
            } else {
                t = __fadd_rn(mvt == MV_PREV_M ? lp_mk : mvt == MV_PREV_B ? lp_bk : lp_kk, v);
            }
            if (t == NEG) { status = 2; break; }  // the reference asserts vm != -inf on every visited cell
            v = t;
            a.l_fm = v;
            a.reserved[0] = 0;
            out[i] = a;                            // compaction to the front: i <= cap - n + i, read before write
        }
        last_v = v;
    }
    const int status_all = __shfl_sync(kFull, status, 0);
    *last_v_out = last_v;
    return status_all ? 0 : n;
}

} // namespace nph_vit
