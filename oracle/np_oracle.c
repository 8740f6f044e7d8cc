/* np_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C, CPU restatement of the reference algorithm of the hot path, written from the
 * behaviour of the reference sources (cited per function, paths relative to /root/reference).
 * It exists so that tests/ can check the CUDA path on a box that has no /root/reference, and so
 * that the restatement itself can be pinned against the compiled reference (oracle/_ref) here.
 *
 * PARITY PIN: the reference's own unit tests hold no known-answer vector for
 * profile_hmm_score_r9 / ABEA (the only HMM test is compiled out, src/test/nanopolish_test.cpp:389-455),
 * so this file is pinned against OUTPUTS OF THE REFERENCE ITSELF RUN HERE: tests/test_oracle_vs_ref.py
 * requires bit-identical floats and identical AlignedPair lists from oracle/_ref/libnpref.so, and
 * tests/golden/ holds vectors generated from the compiled reference by scripts/make_golden.py.
 * The pieces the reference's tests do pin (Gaussian pdf known answer, scalings, kmer_rank) are
 * checked in tests/test_oracle_known_answers.py.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this.  The product (libnph.so) never does: it has no CPU path at all.
 *
 * Build: gcc -O2 -std=c99 -ffp-contract=off (no FMA contraction: the reference is built for
 * baseline x86-64, which has no FMA, so every float op is a separately rounded IEEE op).
 */
#include "np_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------------
 * Table-driven log-sum (HMMER's p7_FLogsum as vendored by the reference).
 * ref: src/common/logsum.h:20-21 (16000 entries, scale 1000), :55-66 (lookup rule),
 *      src/common/logsum.cpp:57-69 (table entry = log(1 + exp(-i/1000)) in double -> float).
 * ---------------------------------------------------------------------------------------- */
#define NPO_TBL 16000
static float g_tbl[NPO_TBL];
static int g_init = 0;

void npo_init(void)
{
    if (g_init) return;
    for (int i = 0; i < NPO_TBL; ++i)
        g_tbl[i] = (float)log(1. + exp((double)-i / 1000.f));
    g_init = 1;
}

void npo_logsum_table(float* out) { npo_init(); memcpy(out, g_tbl, sizeof(g_tbl)); }

float npo_logsum(float a, float b)
{
    const float hi = a > b ? a : b;
    const float lo = a < b ? a : b;
    if (lo == -INFINITY || (hi - lo) >= 15.7f) return hi;
    return hi + g_tbl[(int)((hi - lo) * 1000.f)];
}

/* add_logs takes doubles, narrows to float for the lookup, returns double
 * (src/common/nanopolish_common.h:97-104).  Callers store the result in a float. */
static inline float add_logs_f(float a, float b) { return (float)(double)npo_logsum((float)(double)a, (float)(double)b); }

/* ------------------------------------------------------------------------------------------
 * Emissions.  ref: src/hmm/nanopolish_emissions.h:43-68, src/nanopolish_squiggle_read.h:149-154,
 * :168-171, :217-226.
 * ---------------------------------------------------------------------------------------- */
float npo_log_normal_pdf(float x, float mean, float stdv, float log_stdv)
{
    static const double inv_sqrt_2pi = 0.3989422804014327;
    const float log_inv_sqrt_2pi = (float)log(inv_sqrt_2pi);
    float a = (x - mean) / stdv;
    return log_inv_sqrt_2pi - log_stdv + (-0.5f * a * a);
}

float npo_drift_scaled_level(const nph_read* read, const float* ev_mean, const double* ev_start_time, uint32_t event_idx)
{
    const float* m = ev_mean + read->event_off;
    const double* t = ev_start_time + read->event_off;
    float level = m[event_idx];
    float time = (float)(t[event_idx] - t[0]);
    return (float)(level - time * read->drift);   /* float - (float*double) : evaluated in double, narrowed */
}

static inline void scaled_gaussian(const nph_read* read, const npo_model* model, uint32_t rank,
                                   float* mean, float* stdv, float* log_stdv)
{
    *mean = (float)(read->scale * model->level_mean[rank] + read->shift);
    *stdv = (float)(model->level_stdv[rank] * read->var);
    *log_stdv = (float)(model->level_log_stdv[rank] + read->log_var);
}

float npo_log_probability_match(const nph_read* read, const float* ev_mean, const double* ev_start_time,
                                const npo_model* model, uint32_t rank, uint32_t event_idx)
{
    float level = npo_drift_scaled_level(read, ev_mean, ev_start_time, event_idx);
    float gm, gs, gl;
    scaled_gaussian(read, model, rank, &gm, &gs, &gl);
    return npo_log_normal_pdf(level, gm, gs, gl);
}

/* ------------------------------------------------------------------------------------------
 * Transitions.  ref: calculate_transitions, src/hmm/nanopolish_profile_hmm_r9.inl:17-76.
 * Order of out10: mk, mb, mm_self, mm_next, bb, bk, bm_next, bm_self, kk, km.
 * ---------------------------------------------------------------------------------------- */
void npo_transitions(double events_per_base, double indel_bias, float out[10])
{
    double epb = events_per_base * indel_bias;
    if (epb < 1.25) epb = 1.25;
    float p_stay = (float)(1 - (1 / epb));
    float p_skip = 0.0025;
    float p_bad = 0.001;
    float p_bad_self = p_bad;
    float p_skip_self = 0.3;

    float p_mk = p_skip, p_mb = p_bad, p_mm_self = p_stay;
    float p_mm_next = 1.0f - p_mm_self - p_mk - p_mb;
    float p_bb = p_bad_self;
    float p_third = (1.0f - p_bb) / 3;
    float p_kk = p_skip_self;
    float p_km = 1.0f - p_kk;

    /* The reference writes log(p) with a float argument in C++, which selects the float overload
     * std::log(float) == logf, not the double log. */
    out[0] = logf(p_mk);
    out[1] = logf(p_mb);
    out[2] = logf(p_mm_self);
    out[3] = logf(p_mm_next);
    out[4] = logf(p_bb);
    out[5] = logf(p_third);   /* bk */
    out[6] = logf(p_third);   /* bm_next */
    out[7] = logf(p_third);   /* bm_self */
    out[8] = logf(p_kk);
    out[9] = logf(p_km);
}

/* ------------------------------------------------------------------------------------------
 * Clip penalties.  ref: make_pre_flanking / make_post_flanking, profile_hmm_r9.inl:200-260,
 * background emission -3.0f (emissions.h:98-103).  Because the background log-density is a
 * constant, pre_flank[i] depends on i only and post_flank[i] == pre_flank[n-1-i]; one table serves both.
 * ---------------------------------------------------------------------------------------- */
void npo_flank_table(float* out, size_t n)
{
    const double start_to_clip = 0.5, clip_self = 0.9;
    const float bg = -3.0f;
    if (n > 0) out[0] = (float)log(1 - start_to_clip);
    if (n > 1) out[1] = (float)(log(start_to_clip) + bg + log(1 - clip_self));
    for (size_t i = 2; i < n; ++i)
        out[i] = (float)(log(clip_self) + bg + out[i - 1]);
}

/* ------------------------------------------------------------------------------------------
 * Forward fill.  ref: profile_hmm_score_r9 (src/hmm/nanopolish_profile_hmm_r9.cpp:35-65),
 * profile_hmm_forward_initialize_r9 (:21-33), profile_hmm_fill_generic_r9
 * (src/hmm/nanopolish_profile_hmm_r9.inl:265-433), ProfileHMMForwardOutputR9 (:79-127).
 * Column layout: 3*block + {0: k-mer skip, 1: bad event, 2: match} (profile_hmm_r9.h:52-59).
 * ---------------------------------------------------------------------------------------- */
enum { ST_K = 0, ST_B = 1, ST_M = 2, NST = 3 };

static float fold6(const float x[6])
{
    float s = x[0];
    for (int i = 1; i < 6; ++i) s = add_logs_f(s, x[i]);
    return s;
}

static float hmm_fill(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                      const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                      double indel_bias, float* fm, int viterbi, uint8_t* bm,
                      uint32_t* end_row, uint32_t* end_col)
{
    const nph_read* read = &reads[job->read];
    const npo_model* model = &models[job->model_id];
    const uint32_t* ranks = kmer_ranks + job->rank_off;
    const uint32_t n_kmers = job->n_kmers;
    const uint32_t n_blocks = n_kmers + 2;
    const uint32_t n_cols = NST * n_blocks;
    const uint32_t e_start = job->event_start;
    const uint32_t n_events = (job->event_stop > e_start ? job->event_stop - e_start : e_start - job->event_stop) + 1;
    const uint32_t n_rows = n_events + 1;
    const int stride = job->stride;
    const uint32_t flags = job->flags;

    /* initialise: row 0 and block 0 are -inf, the rest is zero-filled by the reference's
     * allocate_matrix (memset) and then overwritten (nanopolish_matrix.h:35-44). */
    for (size_t i = 0; i < (size_t)n_rows * n_cols; ++i) fm[i] = 0.0f;
    for (uint32_t c = 0; c < n_cols; ++c) fm[c] = -INFINITY;
    for (uint32_t r = 0; r < n_rows; ++r) {
        fm[(size_t)r * n_cols + ST_K] = -INFINITY;
        fm[(size_t)r * n_cols + ST_B] = -INFINITY;
        fm[(size_t)r * n_cols + ST_M] = -INFINITY;
    }

    float t[10];
    npo_transitions(read->events_per_base, indel_bias, t);
    const float lp_mk = t[0], lp_mb = t[1], lp_mm_self = t[2], lp_mm_next = t[3], lp_bb = t[4];
    const float lp_bk = t[5], lp_bm_next = t[6], lp_bm_self = t[7], lp_kk = t[8], lp_km = t[9];

    float* pre = (float*)malloc(sizeof(float) * (n_events + 1));
    float* post = (float*)malloc(sizeof(float) * n_events);
    npo_flank_table(pre, n_events + 1);
    for (uint32_t i = 0; i < n_events; ++i) post[i] = pre[n_events - 1 - i];

    const float lp_sm = 0.0f, lp_ms = 0.0f;
    float lp_end = -INFINITY;
    const uint32_t last_kmer = n_kmers - 1;
    const uint32_t last_row = n_rows - 1;

    for (uint32_t row = 1; row < n_rows; ++row) {
        const uint32_t event_idx = e_start + (row - 1) * stride;
        float* cur = fm + (size_t)row * n_cols;
        const float* prv = fm + (size_t)(row - 1) * n_cols;
        for (uint32_t block = 1; block < n_blocks - 1; ++block) {
            const uint32_t ki = block - 1;
            const uint32_t pb = NST * (block - 1), cb = NST * block;
            const float em = npo_log_probability_match(read, ev_mean, ev_start_time, model, ranks[ki], event_idx);
            float x[6];

            x[0] = lp_mm_self + prv[cb + ST_M];
            x[1] = lp_mm_next + prv[pb + ST_M];
            x[2] = lp_bm_self + prv[cb + ST_B];
            x[3] = lp_bm_next + prv[pb + ST_B];
            x[4] = lp_km + prv[pb + ST_K];
            x[5] = (ki == 0 && (event_idx == e_start || (flags & NPH_HAF_ALLOW_PRE_CLIP))) ? lp_sm + pre[row - 1] : -INFINITY;
            if (!viterbi) {
                cur[cb + ST_M] = fold6(x) + em;
            } else {
                float mx = x[0]; uint8_t from = 0;
                for (int i = 1; i < 6; ++i) { mx = x[i] > mx ? x[i] : mx; from = mx == x[i] ? (uint8_t)i : from; }
                cur[cb + ST_M] = mx + em; bm[(size_t)row * n_cols + cb + ST_M] = from;
            }

            x[0] = lp_mb + prv[cb + ST_M];
            x[1] = -INFINITY;
            x[2] = lp_bb + prv[cb + ST_B];
            x[3] = x[4] = x[5] = -INFINITY;
            if (!viterbi) {
                cur[cb + ST_B] = fold6(x) + 0.0f;
            } else {
                float mx = x[0]; uint8_t from = 0;
                for (int i = 1; i < 6; ++i) { mx = x[i] > mx ? x[i] : mx; from = mx == x[i] ? (uint8_t)i : from; }
                cur[cb + ST_B] = mx + 0.0f; bm[(size_t)row * n_cols + cb + ST_B] = from;
            }

            x[0] = -INFINITY;
            x[1] = lp_mk + cur[pb + ST_M];
            x[2] = -INFINITY;
            x[3] = lp_bk + cur[pb + ST_B];
            x[4] = lp_kk + cur[pb + ST_K];
            x[5] = -INFINITY;
            if (!viterbi) {
                cur[cb + ST_K] = fold6(x) + 0.0f;
            } else {
                float mx = x[0]; uint8_t from = 0;
                for (int i = 1; i < 6; ++i) { mx = x[i] > mx ? x[i] : mx; from = mx == x[i] ? (uint8_t)i : from; }
                cur[cb + ST_K] = mx + 0.0f; bm[(size_t)row * n_cols + cb + ST_K] = from;
            }

            if (ki == last_kmer && ((flags & NPH_HAF_ALLOW_POST_CLIP) || row == last_row)) {
                const int order[3] = { ST_M, ST_B, ST_K };
                for (int s = 0; s < 3; ++s) {
                    float v = lp_ms + cur[cb + order[s]] + post[row - 1];
                    if (!viterbi) {
                        lp_end = add_logs_f(lp_end, v);
                    } else if (v > lp_end) {
                        lp_end = v; *end_row = row; *end_col = cb + order[s];
                    }
                }
            }
        }
    }
    free(pre);
    free(post);
    return lp_end;
}

static size_t job_rows(const nph_hmm_job* job)
{
    uint32_t n_events = (job->event_stop > job->event_start ? job->event_stop - job->event_start
                                                            : job->event_start - job->event_stop) + 1;
    return (size_t)n_events + 1;
}

float npo_hmm_score_dump(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                         const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                         double indel_bias, float* fm)
{
    npo_init();
    return hmm_fill(reads, ev_mean, ev_start_time, models, kmer_ranks, job, indel_bias, fm, 0, NULL, NULL, NULL);
}

float npo_hmm_score(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                    const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                    double indel_bias)
{
    npo_init();
    size_t cells = job_rows(job) * (size_t)(NST * (job->n_kmers + 2));
    float* fm = (float*)malloc(sizeof(float) * cells);
    float s = hmm_fill(reads, ev_mean, ev_start_time, models, kmer_ranks, job, indel_bias, fm, 0, NULL, NULL, NULL);
    free(fm);
    return s;
}

/* ------------------------------------------------------------------------------------------
 * Viterbi alignment.  ref: profile_hmm_align_r9, src/hmm/nanopolish_profile_hmm_r9.cpp:73-204 with
 * ProfileHMMViterbiOutputR9 (src/hmm/nanopolish_profile_hmm_r9.inl:130-197).  The backtrack starts at
 * (last row, MATCH of the last k-mer) — not at the best end cell — and stops at a FROM_SOFT movement.
 * Returns the number of states written (ascending event order), or 0 with *status != 0 where the
 * reference would hit an assert (n_events < 2, or the path runs into a -inf cell).
 * ---------------------------------------------------------------------------------------- */
uint32_t npo_hmm_align(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                       const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                       double indel_bias, nph_align_state* out, uint32_t cap, int* status)
{
    npo_init();
    *status = 0;
    const uint32_t n_kmers = job->n_kmers;
    const size_t n_rows = job_rows(job);
    const uint32_t n_events = (uint32_t)n_rows - 1;
    if (n_events < 2) { *status = 1; return 0; }
    const uint32_t n_cols = NST * (n_kmers + 2);
    float* vm = (float*)malloc(sizeof(float) * n_rows * n_cols);
    uint8_t* bm = (uint8_t*)calloc(n_rows * n_cols, 1);
    uint32_t er = 0, ec = 0;
    hmm_fill(reads, ev_mean, ev_start_time, models, kmer_ranks, job, indel_bias, vm, 1, bm, &er, &ec);

    const char sym[3] = { 'K', 'B', 'M' };
    uint32_t row = (uint32_t)n_rows - 1;
    uint32_t col = NST * n_kmers + ST_M;
    uint32_t n = 0;
    while (row > 0) {
        uint32_t event_idx = job->event_start + (row - 1) * job->stride;
        uint32_t block = col / NST;
        uint32_t kmer_idx = block - 1;
        int ps = (int)(col % NST);
        if (block == 0 || vm[(size_t)row * n_cols + col] == -INFINITY) { *status = 2; n = 0; break; }
        if (n < cap) {
            out[n].event_idx = event_idx; out[n].kmer_idx = kmer_idx;
            out[n].l_fm = vm[(size_t)row * n_cols + col]; out[n].state = sym[ps];
            out[n].reserved[0] = out[n].reserved[1] = out[n].reserved[2] = 0;
        } else { *status = 3; n = 0; break; }
        n++;
        int movement = bm[(size_t)row * n_cols + col];
        if (movement == 5) break;                 /* HMT_FROM_SOFT */
        int next_ps = ST_M;
        switch (movement) {
            case 0: next_ps = ST_M; break;                       /* FROM_SAME_M */
            case 1: kmer_idx -= 1; next_ps = ST_M; break;        /* FROM_PREV_M */
            case 2: next_ps = ST_B; break;                       /* FROM_SAME_B */
            case 3: kmer_idx -= 1; next_ps = ST_B; break;        /* FROM_PREV_B */
            case 4: kmer_idx -= 1; next_ps = ST_K; break;        /* FROM_PREV_K */
        }
        if (ps != ST_K) row -= 1;                 /* a k-mer skip is silent: same row */
        col = NST * (kmer_idx + 1) + next_ps;
    }
    for (uint32_t i = 0, j = n ? n - 1 : 0; i < j; ++i, --j) { nph_align_state t = out[i]; out[i] = out[j]; out[j] = t; }
    free(vm); free(bm);
    return n;
}

static double now_s(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

double npo_hmm_score_batch(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                           const npo_model* models, const uint32_t* kmer_ranks,
                           const nph_hmm_job* jobs, size_t n_jobs, double indel_bias, int threads,
                           float* scores_out)
{
    npo_init();
    if (threads < 1) threads = 1;
    double t0 = now_s();
    #pragma omp parallel for schedule(dynamic) num_threads(threads)
    for (size_t j = 0; j < n_jobs; ++j)
        scores_out[j] = npo_hmm_score(reads, ev_mean, ev_start_time, models, kmer_ranks, &jobs[j], indel_bias);
    return now_s() - t0;
}

/* profile_hmm_score_set: score_i - log(n) in double, folded through the table logsum.
 * ref: src/hmm/nanopolish_profile_hmm.cpp:32-56. */
float npo_score_set_combine(const float* scores, uint32_t n_alt)
{
    npo_init();
    double pen = log((double)n_alt);
    double score = scores[0] - pen;
    for (uint32_t i = 1; i < n_alt; ++i) {
        double alt = scores[i] - pen;
        score = (double)npo_logsum((float)score, (float)alt);
    }
    return (float)score;
}

/* ------------------------------------------------------------------------------------------
 * Method-of-moments scaling.  ref: estimate_scalings_using_mom, src/nanopolish_raw_loader.cpp:17-60.
 * (scale is a ratio of second moments, as in the reference.)
 * ---------------------------------------------------------------------------------------- */
void npo_mom(const nph_read* reads, const float* ev_mean, const npo_model* model,
             const uint32_t* kmer_ranks, const nph_abea_job* job, double* shift_out, double* scale_out)
{
    const nph_read* read = &reads[job->read];
    const float* m = ev_mean + read->event_off;
    const uint32_t* ranks = kmer_ranks + job->rank_off;
    size_t n = read->n_events, nk = job->n_kmers;
    double ev_sum = 0.0;
    for (size_t i = 0; i < n; ++i) ev_sum += m[i];
    double k_sum = 0.0, k_sq = 0.0;
    for (size_t i = 0; i < nk; ++i) {
        double l = model->level_mean[ranks[i]];
        k_sum += l;
        k_sq += pow(l, 2.0f);
    }
    double shift = ev_sum / n - k_sum / nk;
    double ev_sq = 0.0;
    for (size_t i = 0; i < n; ++i) ev_sq += pow(m[i] - shift, 2.0);
    *shift_out = shift;
    *scale_out = (ev_sq / n) / (k_sq / nk);
}

/* ------------------------------------------------------------------------------------------
 * Adaptive banded event alignment (Suzuki-Kasahara band, width 100, Viterbi over
 * diag=step / up=stay / left=skip).  ref: src/nanopolish_raw_loader.cpp:77-379; band coordinate
 * algebra :62-75.
 * ---------------------------------------------------------------------------------------- */
#define BW 100
enum { FROM_D = 0, FROM_U = 1, FROM_L = 2 };

/* ll_k_out (n_events + n_kmers + 2 entries, or NULL): the k-mer index of each band's lower-left cell, band 0 first */
static int64_t abea_core(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                         const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* job,
                         nph_aligned_pair* pairs_out, nph_abea_result* res, int32_t* ll_k_out)
{
    const nph_read* read = &reads[job->read];
    const uint32_t* ranks = kmer_ranks + job->rank_off;
    const long n_events = read->n_events;
    const long n_kmers = job->n_kmers;
    const int half_bw = BW / 2;

    const double min_average_log_emission = -5.0;
    const int max_gap_threshold = 50;

    double events_per_kmer = (double)n_events / n_kmers;
    double p_stay = 1 - (1 / (events_per_kmer + 1));
    double epsilon = 1e-10;
    double lp_skip = log(epsilon);
    double lp_stay = log(p_stay);
    double lp_step = log(1.0 - exp(lp_skip) - exp(lp_stay));
    double lp_trim = log(0.01);

    const long n_rows = n_events + 1, n_cols = n_kmers + 1, n_bands = n_rows + n_cols;

    float* bands = (float*)malloc(sizeof(float) * n_bands * BW);
    uint8_t* trace = (uint8_t*)malloc((size_t)n_bands * BW);
    int* ll_e = (int*)malloc(sizeof(int) * n_bands);   /* event index of each band's lower-left cell */
    int* ll_k = (int*)malloc(sizeof(int) * n_bands);   /* k-mer index of it */
    for (long i = 0; i < n_bands * BW; ++i) { bands[i] = -INFINITY; trace[i] = 0; }
#define BAND(b, o) bands[(size_t)(b) * BW + (o)]
#define TRACE(b, o) trace[(size_t)(b) * BW + (o)]

    ll_e[0] = half_bw - 1;
    ll_k[0] = -1 - half_bw;
    ll_e[1] = ll_e[0] + 1;
    ll_k[1] = ll_k[0];

    BAND(0, -1 - ll_k[0]) = 0.0f;                         /* start cell (event -1, kmer -1) */
    { int o = ll_e[1] - 0; BAND(1, o) = (float)lp_trim; TRACE(1, o) = FROM_U; }

    for (long bi = 2; bi < n_bands; ++bi) {
        float ll = BAND(bi - 1, 0), ur = BAND(bi - 1, BW - 1);
        int right;
        if (ll == -INFINITY && ur == -INFINITY) right = (bi % 2 == 1);
        else right = ll < ur;
        if (right) { ll_e[bi] = ll_e[bi - 1]; ll_k[bi] = ll_k[bi - 1] + 1; }
        else       { ll_e[bi] = ll_e[bi - 1] + 1; ll_k[bi] = ll_k[bi - 1]; }

        int trim_offset = -1 - ll_k[bi];
        if (trim_offset >= 0 && trim_offset < BW) {
            long e = ll_e[bi] - trim_offset;
            if (e >= 0 && e < n_events) { BAND(bi, trim_offset) = (float)(lp_trim * (e + 1)); TRACE(bi, trim_offset) = FROM_U; }
            else BAND(bi, trim_offset) = -INFINITY;
        }

        long kmer_min_offset = 0 - ll_k[bi];
        long kmer_max_offset = n_kmers - ll_k[bi];
        long event_min_offset = ll_e[bi] - (n_events - 1);
        long event_max_offset = ll_e[bi] - (-1);
        long min_offset = kmer_min_offset > event_min_offset ? kmer_min_offset : event_min_offset;
        if (min_offset < 0) min_offset = 0;
        long max_offset = kmer_max_offset < event_max_offset ? kmer_max_offset : event_max_offset;
        if (max_offset > BW) max_offset = BW;

        for (long o = min_offset; o < max_offset; ++o) {
            long e = ll_e[bi] - o, k = ll_k[bi] + o;
            long o_up = ll_e[bi - 1] - (e - 1);
            long o_left = (k - 1) - ll_k[bi - 1];
            long o_diag = (k - 1) - ll_k[bi - 2];
            float up = (o_up >= 0 && o_up < BW) ? BAND(bi - 1, o_up) : -INFINITY;
            float left = (o_left >= 0 && o_left < BW) ? BAND(bi - 1, o_left) : -INFINITY;
            float diag = (o_diag >= 0 && o_diag < BW) ? BAND(bi - 2, o_diag) : -INFINITY;
            float em = npo_log_probability_match(read, ev_mean, ev_start_time, model, ranks[k], (uint32_t)e);
            float score_d = (float)(diag + lp_step + em);
            float score_u = (float)(up + lp_stay + em);
            float score_l = (float)(left + lp_skip);
            float mx = score_d; uint8_t from = FROM_D;
            mx = score_u > mx ? score_u : mx;  from = mx == score_u ? FROM_U : from;
            mx = score_l > mx ? score_l : mx;  from = mx == score_l ? FROM_L : from;
            BAND(bi, o) = mx; TRACE(bi, o) = from;
        }
    }

    /* best end cell: any event against the last k-mer, remaining events trimmed (:309-324) */
    float max_score = -INFINITY;
    long cur_e = 0, cur_k = n_kmers - 1;
    int found = 0;
    for (long e = 0; e < n_events; ++e) {
        long bi = (e + 1) + (cur_k + 1);
        long o = ll_e[bi] - e;
        if (o >= 0 && o < BW) {
            float s = (float)(BAND(bi, o) + (double)(unsigned long)(n_events - e) * lp_trim);
            if (s > max_score) { max_score = s; cur_e = e; found = 1; }
        }
    }

    /* The result record of a failed job follows include/nph.h: NO_END_CELL walks no path; PAIRS_OVERFLOW walks the whole
     * path (n_aligned, max_gap) but skips QC.  Either carries only its own bit and avg_log_emission 0. */
    int64_t n_out = 0;
    double sum_emission = 0, n_aligned = 0;
    int cur_gap = 0, max_gap = 0, status = found ? 0 : NPH_ABEA_NO_END_CELL;
    while (found && cur_k >= 0 && cur_e >= 0) {
        if ((uint64_t)n_out < job->pairs_cap) { pairs_out[n_out].ref_pos = (int32_t)cur_k; pairs_out[n_out].read_pos = (int32_t)cur_e; }
        else status |= NPH_ABEA_PAIRS_OVERFLOW;
        n_out++;
        sum_emission += npo_log_probability_match(read, ev_mean, ev_start_time, model, ranks[cur_k], (uint32_t)cur_e);
        n_aligned += 1;
        long bi = (cur_e + 1) + (cur_k + 1);
        long o = ll_e[bi] - cur_e;
        uint8_t from = (o >= 0 && o < BW) ? TRACE(bi, o) : FROM_D;  /* out of band: reference reads out of row */
        if (from == FROM_D) { cur_k -= 1; cur_e -= 1; cur_gap = 0; }
        else if (from == FROM_U) { cur_e -= 1; cur_gap = 0; }
        else { cur_k -= 1; cur_gap += 1; if (cur_gap > max_gap) max_gap = cur_gap; }
    }
    if (!(status & NPH_ABEA_PAIRS_OVERFLOW)) {
        for (int64_t i = 0, j = n_out - 1; i < j; ++i, --j) { nph_aligned_pair t = pairs_out[i]; pairs_out[i] = pairs_out[j]; pairs_out[j] = t; }
    }

    double avg = 0.0;
    if (!status) {
        avg = sum_emission / n_aligned;
        int spanned = pairs_out[0].ref_pos == 0 && pairs_out[n_out - 1].ref_pos == n_kmers - 1;
        if (avg < min_average_log_emission) status |= NPH_ABEA_LOW_EMISSION;
        if (!spanned) status |= NPH_ABEA_NOT_SPANNED;
        if (max_gap > max_gap_threshold) status |= NPH_ABEA_MAX_GAP;
    }

    if (res) {
        res->n_aligned = (uint32_t)n_out;
        res->n_pairs = status ? 0 : (uint32_t)n_out;
        res->status = status;
        res->max_gap = max_gap;
        res->avg_log_emission = avg;
    }
    if (ll_k_out)
        for (long bi = 0; bi < n_bands; ++bi) ll_k_out[bi] = ll_k[bi];
    free(bands); free(trace); free(ll_e); free(ll_k);
    return status ? 0 : n_out;
#undef BAND
#undef TRACE
}

int64_t npo_abea(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                 const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* job,
                 nph_aligned_pair* pairs_out, nph_abea_result* res)
{
    return abea_core(reads, ev_mean, ev_start_time, model, kmer_ranks, job, pairs_out, res, NULL);
}

/* npo_abea, plus the band history: ll_k_out[bi] = k-mer index of band bi's lower-left cell for the n_events + n_kmers + 2
 * bands (the band's columns are k-mers ll_k_out[bi] .. ll_k_out[bi] + 99; the trim column is k-mer -1) */
int64_t npo_abea_bands(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                       const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* job,
                       nph_aligned_pair* pairs_out, nph_abea_result* res, int32_t* ll_k_out)
{
    return abea_core(reads, ev_mean, ev_start_time, model, kmer_ranks, job, pairs_out, res, ll_k_out);
}

double npo_abea_batch(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                      const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* jobs,
                      size_t n_jobs, int threads, nph_aligned_pair* pairs_out, nph_abea_result* res)
{
    if (threads < 1) threads = 1;
    double t0 = now_s();
    #pragma omp parallel for schedule(dynamic) num_threads(threads)
    for (size_t j = 0; j < n_jobs; ++j)
        npo_abea(reads, ev_mean, ev_start_time, model, kmer_ranks, &jobs[j], pairs_out + jobs[j].pairs_off, &res[j]);
    return now_s() - t0;
}

/* ------------------------------------------------------------------------------------------
 * Event detection (scrappie, as called by load_from_raw: src/nanopolish_squiggle_read.cpp:229-235 — the trimmed
 * raw_table is discarded there, so the whole signal is segmented).
 * ref: src/thirdparty/scrappie/event_detection.c: compute_sum_sumsq :35-49, compute_tstat :62-118,
 *      short_long_peak_detector :122-201, create_event(s) :216-266, detect_events :268-319.
 * Returns the number of events (>= 1), events in emission order; -1 if cap is too small.
 * ---------------------------------------------------------------------------------------- */
#include <float.h>
static void tstat_fill(const double* sum, const double* sumsq, size_t n, size_t w, float* t)
{
    const float eta = FLT_MIN, wf = (float)w;
    for (size_t i = 0; i < n; ++i) t[i] = 0.0f;
    if (n < 2 * w || w < 2) return;
    for (size_t i = w; i <= n - w; ++i) {
        double sum1 = sum[i], sumsq1 = sumsq[i];
        if (i > w) { sum1 -= sum[i - w]; sumsq1 -= sumsq[i - w]; }
        float sum2 = (float)(sum[i + w] - sum[i]);
        float sumsq2 = (float)(sumsq[i + w] - sumsq[i]);
        float mean1 = sum1 / wf;
        float mean2 = sum2 / wf;
        float combined_var = sumsq1 / wf - mean1 * mean1 + sumsq2 / wf - mean2 * mean2;
        combined_var = fmaxf(combined_var, eta);
        const float delta_mean = mean2 - mean1;
        t[i] = fabs(delta_mean) / sqrt(combined_var / wf);
    }
}

typedef struct { float threshold; size_t window_length; size_t masked_to; long peak_pos; float peak_value; int valid_peak; } npo_detector;

/* one step of short_long_peak_detector at position i; the boundaries it emits go to peaks[*count] (and their step to
 * step_out[*count] when given) */
static void npo_peak_step(npo_detector* det, const float* const* sig, float peak_height, size_t i, size_t* peaks, uint64_t* step_out,
                          size_t* count)
{
    for (int k = 0; k < 2; ++k) {
        npo_detector* d = &det[k];
        if (d->masked_to >= i) continue;
        float cur = sig[k][i];
        if (d->peak_pos == -1) {
            if (cur < d->peak_value) d->peak_value = cur;
            else if (cur - d->peak_value > peak_height) { d->peak_value = cur; d->peak_pos = (long)i; }
        } else {
            if (cur > d->peak_value) { d->peak_value = cur; d->peak_pos = (long)i; }
            if (k == 0 && d->peak_value > d->threshold) {
                det[1].masked_to = d->peak_pos + d->window_length;
                det[1].peak_pos = -1; det[1].peak_value = FLT_MAX; det[1].valid_peak = 0;
            }
            if (d->peak_value - cur > peak_height && d->peak_value > d->threshold) d->valid_peak = 1;
            if (d->valid_peak && (i - d->peak_pos) > d->window_length / 2) {
                if (step_out) step_out[*count] = i;
                peaks[(*count)++] = (size_t)d->peak_pos;
                d->peak_pos = -1; d->peak_value = cur; d->valid_peak = 0;
            }
        }
    }
}

static void npo_detectors_init(npo_detector* det, const nph_event_params* prm)
{
    const npo_detector d0 = { prm->threshold1, prm->window_length1, 0, -1, FLT_MAX, 0 }, d1 = { prm->threshold2, prm->window_length2, 0, -1, FLT_MAX, 0 };
    det[0] = d0; det[1] = d1;
}

/* npo_detect_events, plus what it saw on the way: the two t-statistic vectors (t1_out, t2_out: n each) and the position of
 * the detector step that emitted each boundary (emit_step_out: n entries; boundary b is the start of event b + 1) */
long long npo_detect_events_trace(const float* raw, size_t n, const nph_event_params* prm, nph_event* out, size_t cap,
                                  float* t1_out, float* t2_out, uint64_t* emit_step_out)
{
    double* sum = (double*)calloc(n + 1, sizeof(double));
    double* sumsq = (double*)calloc(n + 1, sizeof(double));
    float* t1 = (float*)calloc(n, sizeof(float));
    float* t2 = (float*)calloc(n, sizeof(float));
    size_t* peaks = (size_t*)calloc(n, sizeof(size_t));
    for (size_t i = 0; i < n; ++i) { sum[i + 1] = sum[i] + raw[i]; sumsq[i + 1] = sumsq[i] + raw[i] * raw[i]; }
    tstat_fill(sum, sumsq, n, prm->window_length1, t1);
    tstat_fill(sum, sumsq, n, prm->window_length2, t2);
    npo_detector det[2];
    npo_detectors_init(det, prm);
    const float* sig[2] = { t1, t2 };
    size_t peak_count = 0;
    for (size_t i = 0; i < n; ++i) npo_peak_step(det, sig, prm->peak_height, i, peaks, emit_step_out, &peak_count);
    if (t1_out) memcpy(t1_out, t1, n * sizeof(float));
    if (t2_out) memcpy(t2_out, t2, n * sizeof(float));
    size_t ne = 1;
    for (size_t i = 0; i < n; ++i) if (peaks[i] > 0 && peaks[i] < n) ne++;
    long long ret = (long long)ne;
    if (ne > cap) ret = -1;
    else {
        for (size_t ev = 0; ev < ne; ++ev) {
            size_t s = ev == 0 ? 0 : peaks[ev - 1];
            size_t e = ev == ne - 1 ? n : peaks[ev];
            nph_event x;
            x.start = (uint64_t)s;
            x.length = (float)(e - s);
            x.mean = (float)(sum[e] - sum[s]) / x.length;
            const float deltasqr = (sumsq[e] - sumsq[s]);
            const float var = deltasqr / x.length - x.mean * x.mean;
            x.stdv = sqrtf(fmaxf(var, 0.0f));
            out[ev] = x;
        }
    }
    free(sum); free(sumsq); free(t1); free(t2); free(peaks);
    return ret;
}

long long npo_detect_events(const float* raw, size_t n, const nph_event_params* prm, nph_event* out, size_t cap)
{
    return npo_detect_events_trace(raw, n, prm, out, cap, NULL, NULL, NULL);
}

/* The peak detector alone, walked over positions [from, to) of given t-statistic vectors from the state *st (updated in
 * place).  Returns the number of boundaries emitted; the first `cap` of them go to peaks_out (position) and step_out (the
 * step that emitted it). */
size_t npo_peak_walk(const float* t1, const float* t2, const nph_event_params* prm, size_t from, size_t to, npo_peak_state* st,
                     uint64_t* peaks_out, uint64_t* step_out, size_t cap)
{
    npo_detector det[2];
    npo_detectors_init(det, prm);
    for (int k = 0; k < 2; ++k) {
        det[k].masked_to = (size_t)st->masked_to[k]; det[k].peak_pos = (long)st->peak_pos[k];
        det[k].peak_value = st->peak_value[k]; det[k].valid_peak = st->valid_peak[k];
    }
    const float* sig[2] = { t1, t2 };
    size_t count = 0, peaks[2];
    uint64_t steps[2];
    for (size_t i = from; i < to; ++i) {
        size_t c = 0;
        npo_peak_step(det, sig, prm->peak_height, i, peaks, steps, &c);
        for (size_t e = 0; e < c; ++e, ++count)
            if (count < cap) { peaks_out[count] = peaks[e]; step_out[count] = steps[e]; }
    }
    for (int k = 0; k < 2; ++k) {
        st->masked_to[k] = det[k].masked_to; st->peak_pos[k] = det[k].peak_pos;
        st->peak_value[k] = det[k].peak_value; st->valid_peak[k] = det[k].valid_peak;
    }
    return count;
}

/* ------------------------------------------------------------------------------------------
 * trim_and_segment_raw -> trim_raw_by_mad, medianf/madf/quantilef.
 * ref: src/thirdparty/scrappie/scrappie_common.c:9-190 (pinned against the compiled reference in
 * tests/test_oracle_vs_ref.py).  Returns 1 and the surviving [start, end) or 0 where the reference returns an empty
 * table or trips its own assert.
 * ---------------------------------------------------------------------------------------- */
static int npo_floatcmp(const void* x, const void* y)
{
    float d = *(const float*)x - *(const float*)y;
    return d > 0 ? 1 : -1;
}

static float npo_quantilef(const float* x, size_t nx, float p, float* space)
{
    memcpy(space, x, nx * sizeof(float));
    qsort(space, nx, sizeof(float), npo_floatcmp);
    const size_t idx = p * (nx - 1);
    const float remf = p * (nx - 1) - idx;
    float out;
    if (idx < nx - 1) out = (1.0 - remf) * space[idx] + remf * space[idx + 1];
    else out = space[idx];
    return out;
}

static float npo_madf(const float* x, size_t n, float* space, float* absdiff)
{
    const float mad_scaling_factor = 1.4826;
    if (n == 1) return 0.0f;
    const float med = npo_quantilef(x, n, 0.5f, space);
    for (size_t i = 0; i < n; ++i) absdiff[i] = fabsf(x[i] - med);
    const float mad = npo_quantilef(absdiff, n, 0.5f, space);
    return mad * mad_scaling_factor;
}

/* npo_trim_raw and what it saw: mad_out[nchunk] the chunks' MADs, stat_out = {threshold, interpolated (0/1)},
 * kept_out = {first chunk above the threshold, last chunk above it} ({nchunk, -1} when none is).  Returns like npo_trim_raw. */
int npo_trim_trace(const float* raw, size_t n, int trim_start, int trim_end, int varseg_chunk, float varseg_thresh,
                   uint32_t* start_out, uint32_t* end_out, float* mad_out, float* stat_out, int64_t* kept_out)
{
    *start_out = 0; *end_out = 0;
    const size_t chunk = (size_t)varseg_chunk;
    const size_t nchunk = n / chunk;
    if (stat_out) { stat_out[0] = 0.0f; stat_out[1] = 0.0f; }
    if (kept_out) { kept_out[0] = (int64_t)nchunk; kept_out[1] = -1; }
    if (nchunk == 0) return 0;
    size_t start = 0, end = nchunk * chunk;
    float* madarr = (float*)malloc(nchunk * sizeof(float));
    float* space = (float*)malloc((nchunk > chunk ? nchunk : chunk) * sizeof(float));
    float* absdiff = (float*)malloc(chunk * sizeof(float));
    for (size_t i = 0; i < nchunk; ++i) madarr[i] = npo_madf(raw + i * chunk, chunk, space, absdiff);
    const float thresh = npo_quantilef(madarr, nchunk, varseg_thresh, space);
    if (mad_out) memcpy(mad_out, madarr, nchunk * sizeof(float));
    if (stat_out) { stat_out[0] = thresh; stat_out[1] = (size_t)(varseg_thresh * (nchunk - 1)) < nchunk - 1 ? 1.0f : 0.0f; }
    for (size_t i = 0; i < nchunk; ++i) { if (madarr[i] > thresh) break; start += chunk; }
    for (size_t i = nchunk; i > 0; --i) { if (madarr[i - 1] > thresh) break; end -= chunk; }
    if (kept_out) { kept_out[0] = (int64_t)(start / chunk); kept_out[1] = (int64_t)(end / chunk) - 1; }
    free(madarr); free(space); free(absdiff);
    if (!(end > start)) return 0;                /* assert(rt.end > rt.start) */
    start += (size_t)trim_start;
    if (end < (size_t)trim_end) return 0;
    end -= (size_t)trim_end;
    if (start >= end) return 0;
    *start_out = (uint32_t)start; *end_out = (uint32_t)end;
    return 1;
}

int npo_trim_raw(const float* raw, size_t n, int trim_start, int trim_end, int varseg_chunk, float varseg_thresh,
                 uint32_t* start_out, uint32_t* end_out)
{
    return npo_trim_trace(raw, n, trim_start, trim_end, varseg_chunk, varseg_thresh, start_out, end_out, NULL, NULL, NULL);
}

/* ------------------------------------------------------------------------------------------
 * The tail of SquiggleRead::load_from_raw after ABEA: base_to_event_map + events_per_base
 * (src/nanopolish_squiggle_read.cpp:273-302), get_eventalignment_for_1d_basecalls (:340-391), recalibrate_model with
 * scale_var = true, scale_drift = false (src/nanopolish_methyltrain.cpp:204-307) and the QC (:319-336).
 * PARITY UNPINNED for this function: squiggle_read.cpp / methyltrain.cpp need HDF5 and Eigen 3.3.7 (Makefile:59),
 * neither present, so the reference cannot be compiled here.  The solve restates Eigen's FullPivLU for a 2x2 system
 * (largest-entry pivot by row+column swap, rank threshold epsilon*2*maxpivot, unit-lower / upper substitution).
 * ---------------------------------------------------------------------------------------- */
static void npo_full_piv_lu_solve_2x2(double a00, double a01, double a11, double b0, double b1, double* x0, double* x1, int* piv)
{
    double m[2][2] = {{a00, a01}, {a01, a11}};
    double b[2] = {b0, b1};
    int pr = 0, pc = 0;
    double big = fabs(m[0][0]);
    if (fabs(m[1][0]) > big) { big = fabs(m[1][0]); pr = 1; pc = 0; }       /* column-major scan, first maximum wins */
    if (fabs(m[0][1]) > big) { big = fabs(m[0][1]); pr = 0; pc = 1; }
    if (fabs(m[1][1]) > big) { big = fabs(m[1][1]); pr = 1; pc = 1; }
    *x0 = 0.0; *x1 = 0.0;
    piv[0] = pr; piv[1] = pc; piv[2] = 0;     /* pivot row, pivot column, rank */
    if (big == 0.0) return;
    double t;
    if (pr == 1) { t = m[0][0]; m[0][0] = m[1][0]; m[1][0] = t; t = m[0][1]; m[0][1] = m[1][1]; m[1][1] = t; t = b[0]; b[0] = b[1]; b[1] = t; }
    if (pc == 1) { t = m[0][0]; m[0][0] = m[0][1]; m[0][1] = t; t = m[1][0]; m[1][0] = m[1][1]; m[1][1] = t; }
    const double l = m[1][0] / m[0][0];
    const double u11 = m[1][1] - l * m[0][1];
    const double c1 = b[1] - l * b[0];
    double maxpivot = big;
    if (fabs(u11) > maxpivot) maxpivot = fabs(u11);
    const double thr = 2.220446049250313e-16 * 2.0 * maxpivot;
    double y0, y1;
    if (fabs(u11) > thr) { y1 = c1 / u11; y0 = (b[0] - y1 * m[0][1]) / m[0][0]; piv[2] = 2; }
    else { y1 = 0.0; y0 = b[0] / m[0][0]; piv[2] = 1; }
    if (pc == 1) { *x0 = y1; *x1 = y0; } else { *x0 = y0; *x1 = y1; }
}

/* npo_recalibrate and what it saw: sums_out = {A00, A01, A11, B0, B1} of the normal equations, piv_out = {pivot row, pivot
 * column, rank (0: all zero, 1, 2)} of the solve (-1 where it did not run), m_kmers_out[n_used] the k-mer of each 'M' event. */
void npo_recalibrate_trace(const nph_read* reads, const float* ev_mean, const npo_model* model, const uint32_t* kmer_ranks,
                           const nph_abea_job* job, const nph_aligned_pair* pairs, uint32_t n_pairs,
                           nph_event_range* b2e /* n_kmers */, nph_calibration* out, double* sums_out, int32_t* piv_out,
                           uint32_t* m_kmers_out /* n_kmers */)
{
    double sums_[5]; int32_t piv_[3];
    double* sums = sums_out ? sums_out : sums_;
    int32_t* pv = piv_out ? piv_out : piv_;
    for (int i = 0; i < 5; ++i) sums[i] = 0.0;
    pv[0] = pv[1] = pv[2] = -1;
    const nph_read* read = &reads[job->read];
    const float* m = ev_mean + read->event_off;
    const uint32_t* ranks = kmer_ranks + job->rank_off;
    const size_t n_kmers = job->n_kmers;
    const nph_aligned_pair* pr = pairs + job->pairs_off;
    out->shift = read->shift; out->scale = read->scale; out->drift = read->drift; out->var = read->var;
    out->events_per_base = 0.0; out->n_used = 0; out->status = NPH_CAL_OK;
    for (size_t k = 0; k < n_kmers; ++k) { b2e[k].start = -1; b2e[k].stop = -1; }
    if (n_pairs == 0) { out->status = NPH_CAL_NOT_ALIGNED; return; }

    size_t max_event = 0, min_event = (size_t)-1, prev_event_idx = (size_t)-1;
    for (size_t i = 0; i < n_pairs; ++i) {
        size_t k_idx = (size_t)pr[i].ref_pos, event_idx = (size_t)pr[i].read_pos;
        if (event_idx != prev_event_idx) {
            if (b2e[k_idx].start == -1) b2e[k_idx].start = (int32_t)event_idx;
            b2e[k_idx].stop = (int32_t)event_idx;
        }
        if (event_idx > max_event) max_event = event_idx;
        if (event_idx < min_event) min_event = event_idx;
        prev_event_idx = event_idx;
    }
    out->events_per_base = (double)(max_event - min_event) / n_kmers;

    /* 'M' events of get_eventalignment_for_1d_basecalls, gathered as recalibrate_model does */
    double* raw_events = (double*)malloc(n_kmers * sizeof(double));
    double* level_means = (double*)malloc(n_kmers * sizeof(double));
    double* level_stdvs = (double*)malloc(n_kmers * sizeof(double));
    size_t n = 0, prev_kmer_rank = (size_t)-1;
    for (size_t ki = 0; ki < n_kmers; ++ki) {
        if (b2e[ki].start == -1) continue;
        for (size_t event_idx = (size_t)b2e[ki].start; event_idx <= (size_t)b2e[ki].stop; ++event_idx) {
            size_t kmer_rank = ranks[ki];
            if (prev_kmer_rank != kmer_rank) {
                raw_events[n] = m[event_idx];
                level_means[n] = model->level_mean[kmer_rank];
                level_stdvs[n] = model->level_stdv[kmer_rank];
                if (m_kmers_out) m_kmers_out[n] = (uint32_t)ki;
                ++n;
            }
            prev_kmer_rank = kmer_rank;
        }
    }
    out->n_used = (uint32_t)n;
    if (n >= 200) {
        double A00 = 0., A01 = 0., A11 = 0., B0 = 0., B1 = 0.;
        for (size_t i = 0; i < n; ++i) {
            double inv_var = 1. / (level_stdvs[i] * level_stdvs[i]);
            double mu = level_means[i];
            double e = raw_events[i];
            A00 += inv_var; A01 += mu * inv_var;
            A11 += mu * mu * inv_var;
            B0 += e * inv_var;
            B1 += mu * e * inv_var;
        }
        sums[0] = A00; sums[1] = A01; sums[2] = A11; sums[3] = B0; sums[4] = B1;
        double shift, scale;
        int piv[3];
        npo_full_piv_lu_solve_2x2(A00, A01, A11, B0, B1, &shift, &scale, piv);
        pv[0] = piv[0]; pv[1] = piv[1]; pv[2] = piv[2];
        double var = 0.;
        for (size_t i = 0; i < n; ++i) {
            double yi = (raw_events[i] - shift - scale * level_means[i]);
            var += yi * yi / (level_stdvs[i] * level_stdvs[i]);
        }
        var /= n;
        var = sqrt(var);
        out->shift = shift; out->scale = scale; out->drift = 0.0; out->var = var;
        if (var > 2.5) out->status |= NPH_CAL_HIGH_VAR;
        else if (out->events_per_base > 5.0) out->status |= NPH_CAL_TOO_MANY_STAYS;
    } else {
        out->status = NPH_CAL_TOO_FEW_EVENTS;
    }
    free(raw_events); free(level_means); free(level_stdvs);
}

void npo_recalibrate(const nph_read* reads, const float* ev_mean, const npo_model* model, const uint32_t* kmer_ranks,
                     const nph_abea_job* job, const nph_aligned_pair* pairs, uint32_t n_pairs,
                     nph_event_range* b2e /* n_kmers */, nph_calibration* out)
{
    npo_recalibrate_trace(reads, ev_mean, model, kmer_ranks, job, pairs, n_pairs, b2e, out, NULL, NULL, NULL);
}

int npo_max_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------------------------
 * The poly(A) and detect-polyi tail callers, per read after loading: SegmentationHMM / DPISegmentationHMM ::segment_squiggle,
 * the read rate, estimate_polya_length and the QC, and for detect-polyi BernoulliHMM::segmentation and
 * post_boolhmm_detetection_qc.
 * ref: src/nanopolish_polya_estimator.cpp:204-509, :564-599, :638-722; src/nanopolish_detect_polyi.cpp:177-518, :563-756, :973-997.
 * Textbook form, on purpose unlike the device's walk: the full backpointer table, the explicit backtrack (p[n-1] = TRANSCRIPT,
 * p[j] = bptr[j][p[j+1]] for j = n-2 .. 1, p[0] = START), the boundary scan over the labels, the read rate through a sort
 * and, for poly(I), the Bernoulli Viterbi with its own stored backpointers.
 * ---------------------------------------------------------------------------------------- */
enum { TL_S = 0, TL_L, TL_A, TL_P, TL_C, TL_T };

static float tl_pdf(float x, float mean, float sd)          /* normal_pdf */
{
    const float a = (x - mean) / sd;
    return ((float)0.3989422804014327 / sd) * expf((-0.5f * a) * a);
}

static float tl_log_prob(float p) { return p > 0.00f ? logf(p) : -INFINITY; }
static float tl_max(float a, float b) { return (a < b) ? b : a; }   /* std::max */

static int tl_dcmp(const void* x, const void* y)
{
    const double a = *(const double*)x, b = *(const double*)y;
    return (a > b) - (a < b);
}

int npo_polya_trace(int polyi, const float* x, uint32_t n, const float* dur, uint32_t n_events,
                    const int32_t* map_start, const int32_t* map_stop, uint32_t n_kmers, double sample_rate,
                    double scale, double shift, double var, uint32_t suffix_clip, npo_tail_result* out,
                    uint8_t* labels_out, uint16_t* ties_out, uint8_t* bits_out)
{
    if (n < 2 || n_kmers == 0) return 0;
    for (uint32_t k = 0; k < n_kmers; ++k)
        if (map_start[k] != -1 && !(map_start[k] >= 0 && map_start[k] <= map_stop[k] && (uint32_t)map_stop[k] < n_events)) return 0;
    /* a NaN duration in a mapped span makes the sort's order undefined */
    for (uint32_t k = 0; k < n_kmers; ++k)
        if (map_start[k] != -1)
            for (int32_t e = map_start[k]; e <= map_stop[k]; ++e)
                if (isnan(dur[e])) return 0;

    /* the emission Gaussians (:232-250, detect_polyi.cpp:233-255), scaled as the HMM's constructor does (:310-354) */
    static const float G[8][2] = {{70.2737f, 3.7743f}, {110.973f, 5.237f}, {79.347f, 8.3702f}, {63.3126f, 2.7464f},
                                  {108.883f, 3.257f}, {79.679f, 6.966f}, {105.784f, 16.022f}, {108.498f, 5.257f}};
    float gm[8], gs[8], gl[8];
    for (int g = 0; g < 8; ++g) {
        gm[g] = (float)shift + (float)scale * G[g][0];
        gs[g] = (float)var * G[g][1];
        gl[g] = logf(gs[g]);
    }
    const float lisp = (float)log(0.3989422804014327);
#define TL_LPDF(xx, g) ((lisp - gl[g]) + ((-0.5f * (((xx) - gm[g]) / gs[g])) * (((xx) - gm[g]) / gs[g])))
    const float lSS = tl_log_prob(0.10f), lSL = tl_log_prob(0.90f), lLL = tl_log_prob(0.90f), lLA = tl_log_prob(0.10f);
    const float lAA = tl_log_prob(0.95f), lAP = tl_log_prob(0.05f), lPP = tl_log_prob(0.89f), lPC = tl_log_prob(0.01f);
    const float lPT = tl_log_prob(0.10f), lCP = tl_log_prob(0.99f), lCC = tl_log_prob(0.01f), lTT = tl_log_prob(1.00f);

    uint8_t (*bp)[6] = (uint8_t (*)[6])malloc((size_t)n * 6);
    uint8_t* reg = (uint8_t*)malloc(n);
    float v[6];
    for (uint32_t i = 0; i < n; ++i) {
        /* row 0 emits the LAST sample (:385-386) */
        const float xi = x[i == 0 ? n - 1 : i];
        const float xx = (xi > 200.0f || xi < 40.0f) ? 100.0f : xi;
        float e[6];
        e[TL_S] = logf(0.50f * tl_pdf(xx, gm[0], gs[0]) + 0.50f * 0.00476f);
        e[TL_L] = TL_LPDF(xx, 1);
        e[TL_A] = logf(0.874f * tl_pdf(xx, gm[2], gs[2]) + 0.126f * tl_pdf(xx, gm[3], gs[3]));
        e[TL_P] = polyi ? logf(0.500f * tl_pdf(xx, gm[4], gs[4]) + 0.500f * tl_pdf(xx, gm[7], gs[7])) : TL_LPDF(xx, 4);
        e[TL_C] = (xx > 70.0f && xx < 140.0f) ? -4.2485f : -INFINITY;
        e[TL_T] = logf(0.346f * tl_pdf(xx, gm[5], gs[5]) + 0.654f * tl_pdf(xx, gm[6], gs[6]));
        if (i == 0) {
            v[TL_S] = tl_log_prob(1.00f) + e[TL_S];
            v[TL_L] = -INFINITY + e[TL_L];
            v[TL_A] = v[TL_P] = v[TL_C] = v[TL_T] = -INFINITY;
            memset(bp[0], 0, 6);
            if (ties_out) ties_out[0] = 0;
            continue;
        }
        const float s_s = v[TL_S] + lSS, s_l = v[TL_S] + lSL, l_l = v[TL_L] + lLL, l_a = v[TL_L] + lLA;
        const float a_a = v[TL_A] + lAA, a_p = v[TL_A] + lAP, p_p = v[TL_P] + lPP, p_c = v[TL_P] + lPC, p_t = v[TL_P] + lPT;
        const float c_c = v[TL_C] + lCC, c_p = v[TL_C] + lCP, t_t = v[TL_T] + lTT;
        v[TL_S] = s_s + e[TL_S];
        v[TL_L] = tl_max(l_l, s_l) + e[TL_L];
        v[TL_A] = tl_max(a_a, l_a) + e[TL_A];
        v[TL_P] = tl_max(p_p, tl_max(a_p, c_p)) + e[TL_P];
        v[TL_C] = tl_max(c_c, p_c) + e[TL_C];
        v[TL_T] = tl_max(p_t, t_t) + e[TL_T];
        /* the backpointers of step i (:411-444): strict <, POLYA's in its precedence P, A, C */
        bp[i][TL_S] = TL_S;
        bp[i][TL_L] = s_l < l_l ? TL_L : TL_S;
        bp[i][TL_A] = l_a < a_a ? TL_A : TL_L;
        bp[i][TL_P] = (a_p < p_p && c_p < p_p) ? TL_P : (p_p < a_p && c_p < a_p) ? TL_A : TL_C;
        bp[i][TL_C] = p_c < c_c ? TL_C : TL_P;
        bp[i][TL_T] = p_t < t_t ? TL_T : TL_P;
        if (ties_out) {
            /* bit 2r: rule r's comparison tied at finite scores, bit 2r + 1: at -inf; rules L, A, P-is-P, P-is-A, C, T */
            const float pa[6][2][2] = {{{s_l, l_l}, {s_l, l_l}}, {{l_a, a_a}, {l_a, a_a}}, {{a_p, p_p}, {c_p, p_p}},
                                       {{p_p, a_p}, {c_p, a_p}}, {{p_c, c_c}, {p_c, c_c}}, {{p_t, t_t}, {p_t, t_t}}};
            uint16_t m = 0;
            for (int r = 0; r < 6; ++r)
                for (int q = 0; q < 2; ++q)
                    if (pa[r][q][0] == pa[r][q][1]) m |= (uint16_t)(isinf(pa[r][q][0]) ? 2u << (2 * r) : 1u << (2 * r));
            ties_out[i] = m;
        }
    }
#undef TL_LPDF
    reg[n - 1] = TL_T;
    for (uint32_t j = n - 2; j >= 1 && j < n; --j) reg[j] = bp[j][reg[j + 1]];
    reg[0] = TL_S;
    free(bp);

    /* the boundary scan (:474-499) and the sentinel rule (:500-506) */
    uint64_t ix[5] = {0, 1, 2, 3, 0};
    for (uint32_t i = 0; i < n; ++i) {
        const int nx = i + 1 < n ? reg[i + 1] : -1;
        if (reg[i] == TL_S && nx == TL_L) ix[0] = i;
        if (reg[i] == TL_L && nx == TL_A) ix[1] = i;
        if (reg[i] == TL_A && nx == TL_P) ix[2] = i;
        if (reg[i] == TL_P && nx == TL_T) ix[3] = i;
        if (reg[i] == TL_C) ix[4] += 1;
    }
    out->sentinel = (ix[1] == 1 || ix[2] == 2 || ix[3] == 3);
    if (out->sentinel) { ix[1] = (uint64_t)n - 3; ix[2] = (uint64_t)n - 2; ix[3] = (uint64_t)n - 1; }
    if (labels_out) memcpy(labels_out, reg, n);
    free(reg);
    for (int k = 0; k < 5; ++k) out->seg[k] = ix[k];

    /* the read rate (:564-599): per-k-mer durations summed in event order, sorted, 1 / element [n / 2] */
    double* d = (double*)malloc(sizeof(double) * n_kmers);
    for (uint32_t k = 0; k < n_kmers; ++k) {
        double s = 0.0;
        if (map_start[k] != -1)
            for (int32_t e = map_start[k]; e <= map_stop[k]; ++e) s += (double)dur[e];
        d[k] = s;
    }
    qsort(d, n_kmers, sizeof(double), tl_dcmp);
    const uint32_t r = n_kmers / 2;
    out->median[0] = r > 0 ? d[r - 1] : NAN;
    out->median[1] = d[r];
    out->median[2] = r + 1 < n_kmers ? d[r + 1] : NAN;
    const double rate = 1.0 / d[r];
    free(d);

    /* estimate_polya_length (:638-662) and the QC (:672-722), in size_t and double as the reference has them */
    const uint64_t ld = ix[1], ad = ix[2], pa = ix[3];
    const double len = (double)(pa - (ad + 1)) / sample_rate * rate + -5.0;
    out->read_rate = rate;
    out->polya_length = (0.0 < len) ? len : 0.0;
    const double n_adapter = (double)((ad + 1) - ld), n_polya = (double)(pa - (ad + 1));
    const double adapter_length = (double)(ad - (ld - 1)) / sample_rate * rate;
    out->qc = NPH_POLYA_PASS;
    if (n_adapter < 200.0 || n_polya < 200.0) out->qc = NPH_POLYA_NOREGION;
    else if (adapter_length > 300.0) out->qc = NPH_POLYA_ADAPTER;
    else if (suffix_clip > 200) out->qc = NPH_POLYA_SUFFCLIP;

    out->polyi_last = out->polya_first = out->detected = -1;
    out->bernoulli = 0;
    out->tail_mean = NAN;
    if (!polyi) return 1;

    /* BernoulliHMM::segmentation(samples, adapter + 1, polya) (detect_polyi.cpp:728-756) */
    const int start = (int)(ad + 1), stop = (int)pa;
    out->polyi_last = out->polya_first = -1;
    if (stop - start >= 100) {
        const int m = stop - start;
        float* y = (float*)malloc(sizeof(float) * m);
        uint8_t* b = (uint8_t*)malloc(m);
        uint8_t* bpA = (uint8_t*)malloc(m);
        uint8_t* lab = (uint8_t*)malloc(m);
        float sum = 0.0f;
        for (int i = 0; i < m; ++i) { y[i] = (float)(((double)x[start + i] - shift) / scale); sum += y[i]; }
        const float mean = sum / (float)m;                         /* instance_mean (:655-659) */
        out->bernoulli = 1;
        out->tail_mean = mean;
        for (int i = 0; i < m; ++i) {                               /* log_lkhd_ratio_sequence (:652-675) */
            const float s = (y[i] - mean) + 108.000f;
            const float xx = (s > 200.0f || s < 40.0f) ? 100.0f : s;
            const float lI = logf(tl_pdf(xx, 108.498f, 5.257f)), lA = logf(tl_pdf(xx, 108.883f, 3.257f));
            b[i] = (lI / lA) > 1.0f;
        }
        const float lII = tl_log_prob(0.90f), lIA = tl_log_prob(0.10f), lAA = tl_log_prob(1.00f);
        const float eI[2] = {logf(1.0f - 0.72304f), logf(0.72304f)}, eA[2] = {logf(1.0f - 0.92154f), logf(0.92154f)};
        float vI = tl_log_prob(1.00f) + eI[b[0]], vA = -INFINITY + eA[b[0]];
        bpA[0] = 0;
        for (int i = 1; i < m; ++i) {                               /* viterbi (:678-725) */
            const float i2i = vI + lII, i2a = vI + lIA, a2a = vA + lAA;
            vI = i2i + eI[b[i]];
            vA = tl_max(i2a, a2a) + eA[b[i]];
            bpA[i] = a2a < i2a ? 0 : 1;
        }
        lab[m - 1] = vI < vA ? 1 : 0;
        for (int j = m - 2; j >= 1; --j) lab[j] = lab[j + 1] == 0 ? 0 : bpA[j];
        lab[0] = 0;
        for (int i = 0; i < m; ++i) {
            if (lab[i] == 0) out->polyi_last = i;
            if (lab[i] == 1 && out->polya_first < 0) out->polya_first = i;
        }
        if (bits_out) memcpy(bits_out, b, m);
        free(y); free(b); free(bpA); free(lab);
    }
    const int region_length = (int)(pa - (ad + 1));
    const int polyi_found = out->polyi_last > 200, polya_found = out->polya_first > 0 && region_length - out->polya_first > 200;
    out->detected = polyi_found ? (polya_found ? NPH_POLYI_A_PLUS_I : NPH_POLYI_POLYI_ONLY)
                                : (polya_found ? NPH_POLYI_POLYA_ONLY : NPH_POLYI_NONE);
    return 1;
}
