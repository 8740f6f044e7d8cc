// hmm_classes.h — kernel-class choice for forward-HMM jobs, shared by host and device code.
//
// A class is (C columns per lane, W lanes per job); 32/W jobs share a warp.  W < 32 classes hold
// single-strip jobs (K <= W*C); W == 32 also chains strips for wide jobs.  A job goes to the class that
// minimises modelled issue slots = steps x (per-step overhead + C x per-cell cost) x W/32: 46 per warp step and
// 67 instructions per block-cell.  These are the steady step of the general row loop of hmm_forward_kernel<9|10, 32, false> before
// the full-warp single-strip classes streamed their jobs (cuobjdump -sass, scripts/k1_bounds.py), and the general loop still runs
// every other class.  A streamed job of those classes costs less than the model says: about E steps of 15 + 67 per column plus its
// transition window (DESIGN.md section 3.4); the model has not been re-fitted to it, so every job keeps the class it had before.
#pragma once
#include <stdint.h>
#include "../../include/nph.h"

#ifdef __CUDACC__
#define NPH_HD __host__ __device__ __forceinline__
#else
#define NPH_HD inline
#endif

#define NPH_NUM_WIDTHS 5              // 4, 8, 16, 32 lanes single-strip; 32 lanes with chained strips
#define NPH_MAX_COLS 10
#define NPH_NUM_CLASSES (NPH_NUM_WIDTHS * NPH_MAX_COLS)
#define NPH_STEP_BUCKETS 1024         // step key: exact below 768, then 32-step bins
#define NPH_CHUNK_BUCKETS 8           // level chunk of the job's read (one-shot call), major key
#define NPH_KEY_BUCKETS (NPH_STEP_BUCKETS * NPH_CHUNK_BUCKETS)
#define NPH_MIN_PERIOD 40             // least rows between chained strips: the last lane writes the right edge of row r, and lane 0 reads it P - 32 steps later (hmm_wavefront.cuh)

NPH_HD uint32_t nph_class_width(int wi) { return wi >= 3 ? 32u : (4u << wi); }   // 4, 8, 16, 32, 32 (chained)
NPH_HD bool nph_class_chained(int wi) { return wi == 4; }
NPH_HD int nph_class_index(int C, int wi) { return wi * NPH_MAX_COLS + (C - 1); }

// events of a job's window, both ends included
NPH_HD int nph_job_events(const nph_hmm_job& jb)
{
    return (int)(jb.event_stop > jb.event_start ? jb.event_stop - jb.event_start : jb.event_start - jb.event_stop) + 1;
}

// How K k-mer columns and E event rows lie on the systolic wavefront of a class (C columns per lane, W lanes per job): the one
// statement of the strip rules for the forward and Viterbi kernels, the scheduler and the host-side scratch sizing.  A chained class
// cuts the columns into strips of W*C that follow each other every P rows.
struct nph_wave_geom {
    int K, E, C, strip;
    int n_strips;
    int kpad;           // columns the strips cover
    int P;              // rows between strip starts (one strip: E)
    NPH_HD bool multi_strip() const { return kpad > strip; }
    NPH_HD int last_strip() const { return n_strips - 1; }
    // lane of the group, and column of that lane, that hold k-mer K - 1 in the last strip
    NPH_HD int end_lane() const { return ((K - 1) - last_strip() * strip) / C; }
    NPH_HD int end_slot() const { return ((K - 1) - last_strip() * strip) % C; }
    NPH_HD int total_steps() const { return last_strip() * P + E + end_lane(); }   // until end_lane has done row E of the last strip
};
// may_chain = false only spares the single-strip kernels the division: a job that fits one strip has one strip either way
NPH_HD nph_wave_geom nph_wave_geometry(int K, int E, int C, int W, bool may_chain)
{
    nph_wave_geom g;
    g.K = K; g.E = E; g.C = C; g.strip = W * C;
    g.n_strips = may_chain ? (K + g.strip - 1) / g.strip : 1;
    g.kpad = g.n_strips * g.strip;
    g.P = g.multi_strip() ? (E > NPH_MIN_PERIOD ? E : NPH_MIN_PERIOD) : E;
    return g;
}

// per-step cost: 46 issue slots of per-step work plus the row update, 67 per column (the general row loop; see above)
NPH_HD float nph_class_cost(uint32_t steps, int C, uint32_t W)
{
    return (float)steps * (46.0f + 67.0f * C) * (W * (1.0f / 32.0f));
}

// returns class index; *steps_out = steps in that class
NPH_HD int nph_choose_class(uint32_t K, uint32_t E, uint32_t* steps_out)
{
    float best = 3.0e38f;
    int best_cls = nph_class_index(NPH_MAX_COLS, 4);
    uint32_t best_steps = 0;
    for (int wi = 0; wi < NPH_NUM_WIDTHS; ++wi) {
        const uint32_t W = nph_class_width(wi);
        for (int C = 1; C <= NPH_MAX_COLS; ++C) {
            const bool fits = K <= W * (uint32_t)C;
            if (nph_class_chained(wi) ? fits : !fits) continue;       // single-strip classes take jobs that fit, the chained class the rest
            const uint32_t steps = (uint32_t)nph_wave_geometry((int)K, (int)E, C, (int)W, true).total_steps();   // a job that fits one strip has one strip
            const float cost = nph_class_cost(steps, C, W);
            if (cost < best) { best = cost; best_cls = nph_class_index(C, wi); best_steps = steps; }
        }
    }
    *steps_out = best_steps;
    return best_cls;
}

// position inside a class's slice of the schedule: level chunk ascending (so that jobs whose reads land first
// run first while the rest is still crossing PCIe), then steps descending (longest first, lockstep neighbours alike)
NPH_HD uint32_t nph_key_bucket(uint32_t steps, uint32_t chunk)
{
    uint32_t b = steps < 768u ? steps : 768u + (steps - 768u) / 32u;
    if (b >= (uint32_t)NPH_STEP_BUCKETS) b = (uint32_t)NPH_STEP_BUCKETS - 1u;
    if (chunk >= (uint32_t)NPH_CHUNK_BUCKETS) chunk = (uint32_t)NPH_CHUNK_BUCKETS - 1u;
    return chunk * (uint32_t)NPH_STEP_BUCKETS + ((uint32_t)NPH_STEP_BUCKETS - 1u - b);
}
