/* np_oracle.h — TEST INFRASTRUCTURE ONLY (see np_oracle.c). */
#ifndef NP_ORACLE_H
#define NP_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#include "../include/nph.h"   /* POD batch structs only; no product code is linked */

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    const double* level_mean;
    const double* level_stdv;
    const double* level_log_stdv;
    uint32_t n_states;
} npo_model;

void  npo_init(void);
float npo_logsum(float a, float b);
void  npo_logsum_table(float* out16000);
void  npo_transitions(double events_per_base, double indel_bias, float out10[10]);
void  npo_flank_table(float* out, size_t n);
float npo_log_normal_pdf(float x, float mean, float stdv, float log_stdv);
float npo_drift_scaled_level(const nph_read* read, const float* ev_mean, const double* ev_start_time, uint32_t event_idx);
float npo_log_probability_match(const nph_read* read, const float* ev_mean, const double* ev_start_time,
                                const npo_model* model, uint32_t rank, uint32_t event_idx);

float npo_hmm_score(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                    const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                    double indel_bias);
/* Optional: dump the whole forward matrix of one job (rows (E+1) x cols 3*(K+2), row-major). */
float npo_hmm_score_dump(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                         const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                         double indel_bias, float* matrix_out);
double npo_hmm_score_batch(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                           const npo_model* models, const uint32_t* kmer_ranks,
                           const nph_hmm_job* jobs, size_t n_jobs, double indel_bias, int threads,
                           float* scores_out);
float npo_score_set_combine(const float* scores, uint32_t n_alt);

uint32_t npo_hmm_align(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                       const npo_model* models, const uint32_t* kmer_ranks, const nph_hmm_job* job,
                       double indel_bias, nph_align_state* out, uint32_t cap, int* status);

int64_t npo_abea(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                 const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* job,
                 nph_aligned_pair* pairs_out, nph_abea_result* res);
int64_t npo_abea_bands(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                       const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* job,
                       nph_aligned_pair* pairs_out, nph_abea_result* res, int32_t* ll_k_out);
double npo_abea_batch(const nph_read* reads, const float* ev_mean, const double* ev_start_time,
                      const npo_model* model, const uint32_t* kmer_ranks, const nph_abea_job* jobs,
                      size_t n_jobs, int threads, nph_aligned_pair* pairs_out, nph_abea_result* res);
void npo_mom(const nph_read* reads, const float* ev_mean, const npo_model* model,
             const uint32_t* kmer_ranks, const nph_abea_job* job, double* shift_out, double* scale_out);
long long npo_detect_events(const float* raw, size_t n, const nph_event_params* prm, nph_event* out, size_t cap);
long long npo_detect_events_trace(const float* raw, size_t n, const nph_event_params* prm, nph_event* out, size_t cap,
                                  float* t1_out, float* t2_out, uint64_t* emit_step_out);
/* the state of short_long_peak_detector's two detectors (index 0 = short, 1 = long); peak_pos -1 = no peak yet */
typedef struct { uint64_t masked_to[2]; int64_t peak_pos[2]; float peak_value[2]; int32_t valid_peak[2]; } npo_peak_state;
size_t npo_peak_walk(const float* t1, const float* t2, const nph_event_params* prm, size_t from, size_t to, npo_peak_state* st,
                     uint64_t* peaks_out, uint64_t* step_out, size_t cap);
int npo_trim_raw(const float* raw, size_t n, int trim_start, int trim_end, int varseg_chunk, float varseg_thresh,
                 uint32_t* start_out, uint32_t* end_out);
void npo_recalibrate(const nph_read* reads, const float* ev_mean, const npo_model* model, const uint32_t* kmer_ranks,
                     const nph_abea_job* job, const nph_aligned_pair* pairs, uint32_t n_pairs,
                     nph_event_range* b2e, nph_calibration* out);
/* the same with what they saw (tests/prep_cases.py checks its edge claims on these) */
int npo_trim_trace(const float* raw, size_t n, int trim_start, int trim_end, int varseg_chunk, float varseg_thresh,
                   uint32_t* start_out, uint32_t* end_out, float* mad_out, float* stat_out, int64_t* kept_out);
void npo_recalibrate_trace(const nph_read* reads, const float* ev_mean, const npo_model* model, const uint32_t* kmer_ranks,
                           const nph_abea_job* job, const nph_aligned_pair* pairs, uint32_t n_pairs,
                           nph_event_range* b2e, nph_calibration* out, double* sums_out, int32_t* piv_out, uint32_t* m_kmers_out);
int npo_max_threads(void);
/* one read of the poly(A) (polyi = 0) or detect-polyi (polyi = 1) tail caller: the answer and what it saw.  seg, read_rate,
 * polya_length, qc, polyi_last, polya_first and detected are the nph_polyi_result fields (-1 for the last three under poly(A));
 * sentinel: whether segment_squiggle's sentinel rule fired; median: the sorted per-k-mer durations at n_kmers / 2 - 1, n_kmers / 2
 * and n_kmers / 2 + 1 (NaN where absent); bernoulli: whether the Bernoulli stage ran (poly(I), a tail of 100 samples or more);
 * tail_mean: its float mean (NaN where it did not run; a tail holding a NaN sample also has a NaN mean). */
typedef struct {
    uint64_t seg[5];
    double   read_rate, polya_length;
    int32_t  qc, polyi_last, polya_first, detected;
    int32_t  sentinel, bernoulli;
    float    tail_mean;
    double   median[3];
} npo_tail_result;
/* Returns 0, computing nothing, where nph_polya_batch refuses the job (n < 2, no k-mer, a bad map entry, a NaN duration in a
 * mapped span).  Optional traces: labels_out[n] the backtracked state of every sample (0..5 = S L A P C T); ties_out[n] per step,
 * bit 2r for a tie of rule r's comparison at finite scores and bit 2r + 1 for one at -inf, rules L, A, P-from-P, P-from-A, C,
 * T; bits_out[polya - adapter - 1] the Bernoulli stage's bits. */
int npo_polya_trace(int polyi, const float* x, uint32_t n, const float* dur, uint32_t n_events,
                    const int32_t* map_start, const int32_t* map_stop, uint32_t n_kmers, double sample_rate,
                    double scale, double shift, double var, uint32_t suffix_clip, npo_tail_result* out,
                    uint8_t* labels_out, uint16_t* ties_out, uint8_t* bits_out);

#ifdef __cplusplus
}
#endif
#endif
