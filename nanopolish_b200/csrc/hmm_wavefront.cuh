// hmm_wavefront.cuh — what the forward score (hmm_forward_kernel.cuh) and the Viterbi aligner (hmm_viterbi_kernel.cuh) share of the
// systolic mapping of profile_hmm_fill_generic_r9 (ref: src/hmm/nanopolish_profile_hmm_r9.inl:265-433); nph_wave_geom (hmm_classes.h)
// holds the strip numbers of one job.  Each kernel steps its own rows and strips.
// A group of W lanes owns a job; lane j owns C adjacent k-mer columns and walks the event rows one step behind lane j - 1, whose states
// arrive by three __shfl_up_sync per step.  W == 32 may chain strips of W*C columns: lane 0 enters strip s + 1 the step after it leaves
// strip s, and the strip's right-edge column (three floats per row) travels from the last lane to lane 0 through the warp's edge rows:
// stored at step s*P + r + W - 2, prefetched at step (s + 1)*P + r - 2, so P >= NPH_MIN_PERIOD leaves P - W >= 8 __syncwarp()s between.
#pragma once
#include "nph_internal.cuh"
#include "hmm_classes.h"
#include <math_constants.h>

// per-warp scratch: max_kpad float4 Gaussians and, for chained strips, three edge rows (indexed 1 .. P <= max_period)
inline uint32_t nph_edge_stride(uint32_t max_period) { return max_period + 8; }
inline void nph_wave_scratch(NphArena& a, uint32_t max_kpad, uint32_t max_period, size_t warps, float4** params, float** edge)
{
    *params = a.take<float4>((size_t)max_kpad * warps);
    *edge = a.take<float>(3 * (size_t)nph_edge_stride(max_period) * warps);
}

// the right-edge column of a chained strip, three states by position (which states is the kernel's business)
struct EdgeRows { float* a; float* b; float* c; };

__device__ __forceinline__ float4* warp_params(float4* params, uint32_t kpad_stride, int warp) { return params + (size_t)warp * kpad_stride; }
__device__ __forceinline__ EdgeRows warp_edge_rows(float* edge, uint32_t edge_stride, int warp)
{
    float* const a = edge + (size_t)warp * 3 * edge_stride;
    return EdgeRows{a, a + edge_stride, a + edge_stride + edge_stride};
}

// per-job prologue: the read-scaled Gaussian of every k-mer, padding columns included, by the job's W lanes
template <int W>
__device__ __forceinline__ void fill_job_gaussians(float4* params, const DevModelView& mv, const DevRead& rd, const uint32_t* rk, int K, int kpad,
                                                   int lane_in_group, float log_inv_sqrt_2pi)
{
    for (int i = lane_in_group; i < kpad; i += W) {
        float4 g = nph_pad_gaussian();
        if (i < K) g = nph_scaled_gaussian(mv, rd, rk[i], log_inv_sqrt_2pi);
        params[i] = g;
    }
}

// a lane's C columns, from the scratch into registers
template <int C>
__device__ __forceinline__ void load_columns(const float4* params, int col0, float (&mu)[C], float (&sd)[C], float (&cc)[C], float (&ry)[C])
{
#pragma unroll
    for (int c = 0; c < C; ++c) { const float4 g4 = params[col0 + c]; mu[c] = g4.x; sd[c] = g4.y; cc[c] = g4.z; ry[c] = g4.w; }
}
