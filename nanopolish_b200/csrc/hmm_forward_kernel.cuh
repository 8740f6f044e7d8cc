// hmm_forward_kernel.cuh — K1: the R9 profile-HMM forward score on sm_90a (kernel template).
//
// Replaces, for a whole batch of (sequence, HMMInputData, flags) jobs at once:
//   profile_hmm_score_r9            ref: src/hmm/nanopolish_profile_hmm_r9.cpp:35-65
//   profile_hmm_fill_generic_r9     ref: src/hmm/nanopolish_profile_hmm_r9.inl:265-433
//   ProfileHMMForwardOutputR9       ref: src/hmm/nanopolish_profile_hmm_r9.inl:79-127
//   log_probability_match_r9        ref: src/hmm/nanopolish_emissions.h:57-68
//   get_scaled_gaussian_from_pore_model_state   ref: src/nanopolish_squiggle_read.h:217-226
//   p7_FLogsum                      ref: src/common/logsum.h:55-66
//
// Design (DESIGN.md section 3 has the long form):
//   * the systolic wavefront of hmm_wavefront.cuh: a group of W lanes (W = 4, 8, 16 or 32; 32/W jobs per warp) owns one job, lane j
//     owns C adjacent k-mer columns (M, B, K states and the read-scaled Gaussian of each in registers); nothing of the
//     (E+1) x 3(K+2) matrix the reference mallocs per call is ever stored.  W == 32 also exists with chained strips for jobs wider
//     than 32*C columns; W < 32 classes hold single-strip jobs (K <= W*C).
//   * the 65.5 KB quantised log-sum table lives in shared memory (exact_math.cuh: 7 instructions per sum).
//   * every float operation is issued in the reference's order with explicit round-to-nearest
//     intrinsics (no FMA contraction), IEEE division included, so scores are bit-identical.
//   * persistent CTAs (one per SM); warps pull 32/W jobs at a time, longest first, from an atomic counter.
#pragma once
#include "hmm_wavefront.cuh"
#include "exact_math.cuh"
#include <climits>

namespace nph_fwd {

static_assert(NPH_TBL_SMEM == NPH_LOGSUM_TBL_LEN, "the shared table must cover every index lsum_sat can form");

// Warps per persistent CTA (one CTA per SM).  The full-warp classes hold 16 warps at up to 128 registers; the sub-warp classes of short
// windows need fewer registers (80 at C = 4) and are latency bound on their per-step loads, so they run 24 (C <= 4) or 20 (C <= 6)
// warps.
constexpr int kMaxWarpsPerCta = 24;
template <int C, int W> struct CtaShape { static constexpr int warps = (W == 32) ? 16 : (C <= 4 ? 24 : (C <= 6 ? 20 : 16)); };
constexpr unsigned kFull = 0xffffffffu;

struct FwdParams {
    const float* level;           // drift-scaled event levels, all reads
    const DevRead* reads;
    const float2* trans;          // per read (lp_mm_self, lp_mm_next)
    const DevModelView* models;
    const uint32_t* ranks;
    const nph_hmm_job* jobs;
    const uint32_t* order;        // this class's slice of the schedule
    uint32_t n_jobs;
    unsigned int* counter;
    const float* logsum_g;
    const float* flank;
    float* scores;
    float4* scratch_params;       // per warp: kpad_stride float4 Gaussians (nph_wave_scratch, hmm_wavefront.cuh)
    float* scratch_edge;          // per warp: 3 * edge_stride floats (chained class only)
    uint32_t kpad_stride;
    uint32_t edge_stride;
    uint32_t lsum_bias;           // NPH_LOGSUM_SAT_ADDR_BIAS, passed at run time on purpose (exact_math.cuh)
    uint32_t lsum_scale;          // 4, at run time for the same reason (keeps the table address an IMAD)
    const uint32_t* progress;     // one-shot call: number of level chunks landed so far (nullptr: all resident)
    uint32_t chunk_events;        // events per level chunk (multiple of 32)
    HmmConsts c;
};

// One row of a lane's C columns.  Mp, Bp, Kp, Tp hold the previous row on entry and this row on return (Tp[c] = lp3 + Bp[c]); lm, lt, lk
// are the left neighbour's M, lp3 + B and K, *_prev of the previous row and *_cur of this one.  With with_soft, column 0's match also
// folds soft() (the soft-clip start; -inf where it does not apply), in a second copy of column 0 that the usual row branches past.
template <int C, class SoftFn>
__device__ __forceinline__ void row_update(const float x, const float (&mu)[C], const float (&sd)[C], const float (&cc)[C], const float (&ry)[C],
                                           float (&Mp)[C], float (&Bp)[C], float (&Kp)[C], float (&Tp)[C],
                                           float lm_prev, float lt_prev, float lk_prev, float lm_cur, float lt_cur, float lk_cur,
                                           const float lp_mm_self, const float lp_mm_next, const HmmConsts& k, const bool with_soft, const SoftFn& soft,
                                           const LogsumTable& tb)
{
    auto cell = [&](const int c, const bool fold_soft) {
        const float em = log_gauss(x, mu[c], sd[c], cc[c], ry[c]);
        // match: left fold over {same M, prev M, same B, prev B, prev K, soft}
        float m = __fadd_rn(lp_mm_self, Mp[c]);
        m = lsum_sat(m, __fadd_rn(lp_mm_next, lm_prev), tb);
        m = lsum_sat(m, Tp[c], tb);
        m = lsum_sat(m, lt_prev, tb);
        m = lsum_sat(m, __fadd_rn(k.lp_km, lk_prev), tb);
        if (fold_soft) m = lsum_sat(m, soft(), tb);
        m = __fadd_rn(m, em);
        // bad event: {same M, same B}
        const float b = lsum_sat(__fadd_rn(k.lp_mb, Mp[c]), __fadd_rn(k.lp_bb, Bp[c]), tb);
        // k-mer skip: {prev M, prev B, prev K} of the SAME row
        float kk = lsum_sat(__fadd_rn(k.lp_mk, lm_cur), lt_cur, tb);
        kk = lsum_sat(kk, __fadd_rn(k.lp_kk, lk_cur), tb);
        const float t = __fadd_rn(k.lp_bk, b);

        lm_prev = Mp[c]; lt_prev = Tp[c]; lk_prev = Kp[c];
        lm_cur = m; lt_cur = t; lk_cur = kk;
        Mp[c] = m; Bp[c] = b; Kp[c] = kk; Tp[c] = t;
    };
    if (with_soft) cell(0, true);
    else cell(0, false);
#pragma unroll
    for (int c = 1; c < C; ++c) cell(c, false);
}

// the end-state fold of one row on the lane holding the last k-mer (column end_slot of the lane); post = flank[E - r]
template <int C>
__device__ __forceinline__ float end_fold(float lp_end, const float (&Mp)[C], const float (&Bp)[C], const float (&Kp)[C], const int end_slot, const float post,
                                          const LogsumTable& tb)
{
    float Me = Mp[0], Be = Bp[0], Ke = Kp[0];
#pragma unroll
    for (int c = 1; c < C; ++c) if (c == end_slot) { Me = Mp[c]; Be = Bp[c]; Ke = Kp[c]; }
    lp_end = lsum_sat(lp_end, __fadd_rn(Me, post), tb);
    lp_end = lsum_sat(lp_end, __fadd_rn(Be, post), tb);
    return lsum_sat(lp_end, __fadd_rn(Ke, post), tb);
}

// a job record with what its read, read transitions and model hold for it; waits, when levels are still streaming in, until the
// chunk holding the read's last event has landed (chunks land in order; the progress word is written by a copy queued behind the data)
struct JobIn { nph_hmm_job job; DevRead rd; float2 tr; DevModelView mv; };
__device__ __forceinline__ JobIn fetch_job(const FwdParams& p, const uint32_t job_idx, const bool has_job, const int lane)
{
    JobIn j;
    j.job = p.jobs[job_idx];
    j.rd = p.reads[j.job.read];
    j.tr = p.trans[j.job.read];
    j.mv = p.models[j.job.model_id];
    if (p.progress) {
        uint32_t need = has_job ? (uint32_t)((j.rd.event_off + j.rd.n_events - 1) / p.chunk_events) + 1u : 0u;
        need = __reduce_max_sync(kFull, need);
        if (lane == 0) {
            const volatile uint32_t* pr = p.progress;
            while (*pr < need) __nanosleep(500);
        }
        __syncwarp();
    }
    return j;
}

// Streamed jobs of the full-warp single-strip classes (W = 32, CHAIN = false).
//
// A job with E > 32 rows and neither pre- nor post-clipping runs in three phases: a 33-step window where its lanes enter one by one,
// E - 33 steady steps where every lane is on a row in 1..E, and a window where its lanes leave.  Lane j of the warp does row E of job n
// at step t = j of the window and row 1 of job n + 1 the step after, so the leaving window of job n is the entering window of job
// n + 1, and the warp keeps its wavefront (left neighbour one step ahead on the same job) from job to job.  A warp fills
// and drains once per stream instead of once per job, and the steady loop carries no per-lane test: three shuffles, the lane-0 edge,
// one prefetch and the row update.  Lanes whose columns lie wholly beyond K compute on the padding Gaussians there; only lanes further
// right read their states, and none of them reaches the end fold.
//
// The warp keeps pulling jobs from the class counter while they qualify; the first one that does not ends the stream (after the
// drain) and is returned for the general loop.  The next job's Gaussians are formed after the steady loop, into the other half of the
// warp's parameter line (two lines of 32 * C, hmm_forward.cu sizes it): the lanes' own Gaussians are read back from their half
// afterwards instead of being held in registers through the formation, which needs more registers than the row loop leaves.
__device__ __forceinline__ bool streams(const nph_hmm_job& job, const int E)
{
    return E > 32 && (job.flags & (NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP)) == 0;
}

// what the windows need of a streamed job.  It sits in shared memory, two per warp (the leaving and the entering job), and is read
// only where one lane enters or leaves a job, so that the window does not hold both jobs' numbers in registers next to its row states.
struct StreamJob {
    unsigned long long x_addr;     // address of the level of row 1
    uint32_t idx;
    int E, end_lane, end_slot;
    float lp_mm_self, lp_mm_next;
    int x_step;                    // bytes from one row's level to the next
};

// forms job_idx's Gaussians on the warp's parameter line and its record in *s (lane 0)
template <int C>
__device__ __forceinline__ int stream_job(const FwdParams& p, float4* params, const uint32_t job_idx, const JobIn& j, const int lane, StreamJob* s)
{
    const nph_wave_geom geo = nph_wave_geometry((int)j.job.n_kmers, nph_job_events(j.job), C, 32, false);
    if (lane == 0) {
        s->x_addr = (unsigned long long)(p.level + j.rd.event_off + j.job.event_start);
        s->idx = job_idx;
        s->E = geo.E; s->end_lane = geo.end_lane(); s->end_slot = geo.end_slot();
        s->lp_mm_self = j.tr.x; s->lp_mm_next = j.tr.y;
        s->x_step = j.job.stride * (int)sizeof(float);
    }
    fill_job_gaussians<32>(params, j.mv, j.rd, p.ranks + j.job.rank_off, geo.K, geo.kpad, lane, p.c.log_inv_sqrt_2pi);
    return geo.E;
}

// Runs the stream that starts with job job_idx (which streams()); returns the slot of the job that ended it (>= p.n_jobs: none left).
template <int C>
__device__ uint32_t run_stream(const FwdParams& p, const LogsumTable& tb, const HmmConsts& k, float4* params, int lane, const uint32_t job_idx,
                               const JobIn& first)
{
    // opaque from here: the stream's addresses and lane offsets are formed inside the stream instead of being hoisted out of the
    // kernel's job loop, where they would hold registers through the general loop
    asm volatile("" : "+l"(params), "+r"(lane));
    __shared__ StreamJob s_jobs[CtaShape<C, 32>::warps][2];
    volatile StreamJob* const sj = s_jobs[threadIdx.x >> 5];   // volatile: read at each lane's entry and exit, not kept in registers
    // the entering job's record is sj[n & 1] and its Gaussians are line(n); the leaving job's record is sj[(n + 1) & 1]
    auto line = [&](const int i) { return params + (i & 1) * (32 * C); };
    int n = 0;
    int E = stream_job<C>(p, line(0), job_idx, first, lane, const_cast<StreamJob*>(&sj[0]));

    const float NEG = -CUDART_INF_F;
    float mu[C], sd[C], cc[C], ry[C];
    float Mp[C], Bp[C], Kp[C], Tp[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { mu[c] = 0.f; sd[c] = 1.f; cc[c] = 0.f; ry[c] = 1.f; Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; Tp[c] = NEG; }
    float Lm_prev = NEG, Lt_prev = NEG, Lk_prev = NEG;
    // this lane's job: transitions and the level address of its next row
    float lp_mm_self = 0.f, lp_mm_next = 0.f;
    unsigned long long x_addr = 0;
    int x_step = 0;
    float x_next = 0.f;
    bool has_a = false, has_b = true;
    uint32_t ended_by = p.n_jobs;
    __syncwarp();
    for (;;) {
        volatile StreamJob& a = sj[(n + 1) & 1];
        volatile StreamJob& b = sj[n & 1];
        // window: lane j is on row E + t - j of the leaving job while t <= j, and on row t - j of b after; lane 31 enters b at t = 32
        const int window = has_b ? 33 : a.end_lane + 1;
        for (int t = 0; t < window; ++t) {
            float Lm = __shfl_up_sync(kFull, Mp[C - 1], 1);
            float Lt = __shfl_up_sync(kFull, Tp[C - 1], 1);
            float Lk = __shfl_up_sync(kFull, Kp[C - 1], 1);
            if (lane == 0) { Lm = NEG; Lt = NEG; Lk = NEG; }
            const float x = x_next;
            if (has_b && t == lane + 1) {
                // entering b (after the shuffle: the right neighbour still takes this lane's last row of the leaving job): row 0 and the
                // start column are -inf
#pragma unroll
                for (int c = 0; c < C; ++c) { Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; Tp[c] = NEG; }
                Lm_prev = NEG; Lt_prev = NEG; Lk_prev = NEG;
                load_columns<C>(line(n), lane * C, mu, sd, cc, ry);
                lp_mm_self = b.lp_mm_self; lp_mm_next = b.lp_mm_next;
            }
            // prefetch for the next step; at t == j that is row 1 of b
            if (t == lane) { x_addr = b.x_addr; x_step = b.x_step; }
            if (t < lane ? has_a : has_b) {
                x_next = __ldca(reinterpret_cast<const float*>(x_addr));
                x_addr += x_step;
            }
            if (t <= lane ? has_a : has_b) {
                // the soft-clip start: column 0 at row 1
                row_update<C>(x, mu, sd, cc, ry, Mp, Bp, Kp, Tp, Lm_prev, Lt_prev, Lk_prev, Lm, Lt, Lk, lp_mm_self, lp_mm_next, k, true,
                              [&] { return (lane == 0 && t == 1) ? p.flank[0] : NEG; }, tb);
                Lm_prev = Lm; Lt_prev = Lt; Lk_prev = Lk;
                if (t == lane && lane == a.end_lane) p.scores[a.idx] = end_fold<C>(NEG, Mp, Bp, Kp, a.end_slot, p.flank[0], tb);   // row E
            }
        }
        if (!has_b) break;

        // steady: every lane on b, rows 33 - j .. E - 1 - j
#pragma unroll 1
        for (int g = E - 33; g > 0; --g) {
            float Lm = __shfl_up_sync(kFull, Mp[C - 1], 1);
            float Lt = __shfl_up_sync(kFull, Tp[C - 1], 1);
            float Lk = __shfl_up_sync(kFull, Kp[C - 1], 1);
            if (lane == 0) { Lm = NEG; Lt = NEG; Lk = NEG; }
            const float x = x_next;
            x_next = __ldca(reinterpret_cast<const float*>(x_addr));
            x_addr += x_step;
            row_update<C>(x, mu, sd, cc, ry, Mp, Bp, Kp, Tp, Lm_prev, Lt_prev, Lk_prev, Lm, Lt, Lk, lp_mm_self, lp_mm_next, k, false,
                          [&] { return NEG; }, tb);
            Lm_prev = Lm; Lt_prev = Lt; Lk_prev = Lk;
        }
        has_a = true;

        // the next job, if it streams, into the other half line and the record of the job that left in the last window
        __syncwarp();
        has_b = false;
        const uint32_t slot = nph_warp_pop(p.counter, 1u, lane);
        if (slot < p.n_jobs) {
            const uint32_t n_idx = p.order[slot];
            const JobIn j = fetch_job(p, n_idx, true, lane);
            has_b = streams(j.job, nph_job_events(j.job));
            if (has_b) E = stream_job<C>(p, line(n + 1), n_idx, j, lane, const_cast<StreamJob*>(&sj[(n + 1) & 1]));
            else ended_by = slot;
        }
        load_columns<C>(line(n), lane * C, mu, sd, cc, ry);
        n += 1;
        __syncwarp();
    }
    return ended_by;
}

// CHAIN = false: every job of the class fits one strip (K <= W*C), all strip/edge bookkeeping compiles away.
template <int C, int W, bool CHAIN>
__global__ void __launch_bounds__(CtaShape<C, W>::warps * 32, 1) hmm_forward_kernel(const FwdParams p)
{
    static_assert(W == 4 || W == 8 || W == 16 || W == 32, "group width");
    static_assert(!CHAIN || W == 32, "only full-warp groups chain strips");
    constexpr int G = 32 / W;                 // jobs per warp
    constexpr int kWarpsPerCta = CtaShape<C, W>::warps;
    constexpr int kCtaThreads = kWarpsPerCta * 32;
    constexpr int STRIP = W * C;              // columns per strip
    extern __shared__ float s_tbl[];
    for (int i = threadIdx.x; i < NPH_TBL_SMEM; i += kCtaThreads) s_tbl[i] = p.logsum_g[i];
    __syncthreads();
    const LogsumTable tb = make_logsum_table(s_tbl, p.lsum_bias, p.lsum_scale);

    const int lane = threadIdx.x & 31;
    const int gl = lane & (W - 1);            // lane within the group
    const int grp = lane / W;
    const int warp_global = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    float4* const my_params = warp_params(p.scratch_params, p.kpad_stride, warp_global) + (W < 32 ? grp * STRIP : 0);
    const EdgeRows edge = warp_edge_rows(p.scratch_edge, p.edge_stride, warp_global);   // M, lp3 + B, K of the edge column

    const float NEG = -CUDART_INF_F;
    // lp_bk, lp_bm_next and lp_bm_self are all log(p_third) (nph_api.cu checks that they are bitwise equal), so
    // lp3 + B is one float that serves K-skip at (r, c+1), M-self at (r+1, c) and M-next at (r+1, c+1)
    const HmmConsts& k = p.c;

    uint32_t ended_stream = UINT_MAX;   // full-warp single strip: the job that ended a stream, not yet run
    for (;;) {
        const uint32_t base = ended_stream != UINT_MAX ? ended_stream : nph_warp_pop(p.counter, (unsigned)G, lane);
        ended_stream = UINT_MAX;
        if (base >= p.n_jobs) break;
        const uint32_t slot = base + grp;
        const bool has_job = slot < p.n_jobs;
        const uint32_t job_idx = p.order[has_job ? slot : base];
        const JobIn ji = fetch_job(p, job_idx, has_job, lane);
        const nph_hmm_job& job = ji.job;
        const DevRead& rd = ji.rd;
        const DevModelView& mv = ji.mv;
        const float lp_mm_self = ji.tr.x, lp_mm_next = ji.tr.y;

        const nph_wave_geom geo = nph_wave_geometry((int)job.n_kmers, has_job ? nph_job_events(job) : 0, C, W, CHAIN);
        const int K = geo.K, E = geo.E, stride = job.stride, n_strips = geo.n_strips, P = geo.P;
        if constexpr (W == 32 && !CHAIN) {
            if (streams(job, E)) { ended_stream = run_stream<C>(p, tb, k, my_params, lane, job_idx, ji); continue; }
        }
        const bool pre_clip = (job.flags & NPH_HAF_ALLOW_PRE_CLIP) != 0;
        const bool post_clip = (job.flags & NPH_HAF_ALLOW_POST_CLIP) != 0;

        // formed in FP64 exactly as get_scaled_gaussian_from_pore_model_state does, then narrowed; plus RN(1/sigma')
        if (has_job) fill_job_gaussians<W>(my_params, mv, rd, p.ranks + job.rank_off, K, geo.kpad, gl, p.c.log_inv_sqrt_2pi);
        __syncwarp();

        const float* lv = p.level + rd.event_off;
        const long long e_first = (long long)job.event_start;
        const int last_strip = geo.last_strip(), end_lane = geo.end_lane(), end_slot = geo.end_slot();
        // lanes beyond end_lane own no column of the last strip; the warp runs until its slowest group is done
        const int my_steps = has_job ? geo.total_steps() : 0;
        const int total_steps = (W == 32) ? my_steps : __reduce_max_sync(kFull, my_steps);
        // the soft-clip fold touches column 0 only at row 1 (step 0) unless a job of this warp allows pre-clipping;
        // elsewhere its operand is -inf, and x (+) -inf == x, so the warp skips it
        const bool any_pre_clip = __any_sync(kFull, pre_clip);

        float mu[C], sd[C], cc[C], ry[C];
        float Mp[C], Bp[C], Kp[C], Tp[C];   // Tp[c] = lp3 + Bp[c]
#pragma unroll
        for (int c = 0; c < C; ++c) { mu[c] = 0.f; sd[c] = 1.f; cc[c] = 0.f; ry[c] = 1.f; Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; Tp[c] = NEG; }
        // one strip: each lane's columns are fixed for the whole job
        if (!CHAIN && gl * C < K) load_columns<C>(my_params, gl * C, mu, sd, cc, ry);
        float Lm_prev = NEG, Lt_prev = NEG, Lk_prev = NEG;
        float lp_end = NEG;
        int r = 1 - gl;        // row of this lane at the current step (rows 1..P; <1 = not started)
        int s = 0;             // strip of this lane (always 0 without CHAIN: rows past E are simply not live)
        float x_next = 0.f;
        if (r == 1 && E >= 1) x_next = lv[e_first];
        float em_next = NEG, et_next = NEG, ek_next = NEG;   // group lane 0: prefetched right edge of the previous strip
        // one strip: address of the level of row r + 1, stepped by one IMAD.WIDE (unsigned, so rows < 1 wrap harmlessly)
        const long long x_step = (long long)stride * (long long)sizeof(float);
        unsigned long long x_addr = (unsigned long long)(lv + e_first) + (unsigned long long)((long long)r * x_step);
        // the end fold runs on the lane holding the last k-mer, from row 1 with post-clipping and at row E without
        const int end_row = (gl == end_lane) ? (post_clip ? 1 : E) : INT_MAX;

        for (int g = 0; g < total_steps; ++g) {
            // left neighbour's newest row (its row == my row, computed one step ago)
            float Lm = __shfl_up_sync(kFull, Mp[C - 1], 1, W);
            float Lt = __shfl_up_sync(kFull, Tp[C - 1], 1, W);
            float Lk = __shfl_up_sync(kFull, Kp[C - 1], 1, W);
            if (gl == 0) { Lm = CHAIN ? em_next : NEG; Lt = CHAIN ? et_next : NEG; Lk = CHAIN ? ek_next : NEG; }

            const bool in_strip = (r >= 1) && (!CHAIN || s < n_strips);
            const int col0 = (CHAIN ? s * STRIP : 0) + gl * C;
            const bool live = in_strip && (r <= E) && (col0 < K);
            const float x = x_next;

            if (CHAIN && in_strip && r == 1) {
                // entering a strip: row 0 and the start column are -inf
#pragma unroll
                for (int c = 0; c < C; ++c) { Mp[c] = NEG; Bp[c] = NEG; Kp[c] = NEG; Tp[c] = NEG; }
                Lm_prev = NEG; Lt_prev = NEG; Lk_prev = NEG;
                if (col0 < K) load_columns<C>(my_params, col0, mu, sd, cc, ry);
            }
            // prefetch for the next step: event level and (group lane 0, chained strips) the stored right edge
            {
                int rn = r + 1, sn = s;
                if (CHAIN && rn > P) { rn = 1; sn = s + 1; }
                if (rn >= 1 && rn <= E && (!CHAIN || sn < n_strips)) {
                    x_next = CHAIN ? lv[e_first + (long long)(rn - 1) * stride] : __ldca(reinterpret_cast<const float*>(x_addr));
                    if (CHAIN && gl == 0 && sn > 0) { em_next = edge.a[rn]; et_next = edge.b[rn]; ek_next = edge.c[rn]; }
                }
            }

            if (live) {
                const bool do_end = (!CHAIN || s == last_strip) && r >= end_row;

                row_update<C>(x, mu, sd, cc, ry, Mp, Bp, Kp, Tp, Lm_prev, Lt_prev, Lk_prev, Lm, Lt, Lk, lp_mm_self, lp_mm_next, k, any_pre_clip || g == 0,
                              [&] { return (col0 == 0 && (r == 1 || pre_clip)) ? p.flank[r - 1] : NEG; }, tb);
                Lm_prev = Lm; Lt_prev = Lt; Lk_prev = Lk;

                // the states of the last k-mer's column; with flags 0 this runs once per job
                if (do_end) lp_end = end_fold<C>(lp_end, Mp, Bp, Kp, end_slot, p.flank[E - r], tb);
                if (CHAIN && gl == W - 1 && s < last_strip) { edge.a[r] = Mp[C - 1]; edge.b[r] = Tp[C - 1]; edge.c[r] = Kp[C - 1]; }
            }

            r += 1;
            if (!CHAIN) x_addr += x_step;
            if (CHAIN && r > P) { r = 1; s += 1; }
            if (CHAIN && n_strips > 1) __syncwarp();   // orders lane 31's edge stores before lane 0's later loads
        }

        const float result = __shfl_sync(kFull, lp_end, (lane & ~(W - 1)) + end_lane);
        if (gl == 0 && has_job) p.scores[job_idx] = result;
        __syncwarp();
    }
}

template <int C, int W, bool CHAIN>
int launch_class(nph_ctx* ctx, const FwdParams& base, const nph_ctx::ClassLaunch& cl, int class_idx, cudaStream_t stream)
{
    FwdParams p = base;
    p.order = ctx->d_order.p + cl.first;
    p.n_jobs = (uint32_t)cl.count;
    p.counter = ctx->d_counters.p + class_idx;
    const size_t smem = sizeof(float) * NPH_TBL_SMEM;
    NPH_CUDA(ctx, cudaFuncSetAttribute(hmm_forward_kernel<C, W, CHAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    constexpr int kWarpsPerCta = CtaShape<C, W>::warps;
    int grid = ctx->sm_count;
    const size_t warps_needed = (cl.count + (32 / W) - 1) / (32 / W);
    if ((size_t)grid * kWarpsPerCta > warps_needed) grid = (int)((warps_needed + kWarpsPerCta - 1) / kWarpsPerCta);
    if (grid < 1) grid = 1;
    hmm_forward_kernel<C, W, CHAIN><<<grid, kWarpsPerCta * 32, smem, stream>>>(p);
    NPH_CUDA(ctx, cudaGetLastError());
    return NPH_OK;
}

// one translation unit per group width (parallel compilation); defined in hmm_forward_w*.cu
template <int W, bool CHAIN> int launch_width(nph_ctx* ctx, const FwdParams& base, const nph_ctx::ClassLaunch& cl, int class_idx, cudaStream_t stream);

#define NPH_DEFINE_LAUNCH_WIDTH(W, CHAIN)                                                                              \
    template <> int launch_width<W, CHAIN>(nph_ctx * ctx, const FwdParams& base, const nph_ctx::ClassLaunch& cl, int class_idx, cudaStream_t stream) \
    {                                                                                                           \
        switch (cl.cols_per_lane) {                                                                             \
            case 1: return launch_class<1, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 2: return launch_class<2, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 3: return launch_class<3, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 4: return launch_class<4, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 5: return launch_class<5, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 6: return launch_class<6, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 7: return launch_class<7, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 8: return launch_class<8, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 9: return launch_class<9, W, CHAIN>(ctx, base, cl, class_idx, stream);                                       \
            case 10: return launch_class<10, W, CHAIN>(ctx, base, cl, class_idx, stream);                                     \
        }                                                                                                       \
        return NPH_ERR_STATE;                                                                                   \
    }

} // namespace nph_fwd
