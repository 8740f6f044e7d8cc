/* nph.h — C ABI of the H100-native nanopolish HMM engine (libnph.so).
 *
 * This is the drop-in boundary for the ONE hot path this repository accelerates
 * (SURVEY.md section 8):
 *
 *   1. the R9 profile-HMM forward score
 *        profile_hmm_score            ref: src/hmm/nanopolish_profile_hmm.cpp:23-30
 *        profile_hmm_score_r9         ref: src/hmm/nanopolish_profile_hmm_r9.cpp:35-65
 *        profile_hmm_fill_generic_r9  ref: src/hmm/nanopolish_profile_hmm_r9.inl:265-433
 *        profile_hmm_score_set        ref: src/hmm/nanopolish_profile_hmm.cpp:32-56
 *   2. the adaptive banded event-to-sequence alignment
 *        adaptive_banded_simple_event_align   ref: src/nanopolish_raw_loader.cpp:77-379
 *        estimate_scalings_using_mom          ref: src/nanopolish_raw_loader.cpp:17-60
 *   3. (section 8f "next" row N1) the Viterbi alignment with the same fill
 *        profile_hmm_align_r9         ref: src/hmm/nanopolish_profile_hmm_r9.cpp:73-204
 *   4. (row N4) the raw-signal prologue that produces the reads the calls above consume
 *        SquiggleRead::load_from_raw  ref: src/nanopolish_squiggle_read.cpp:226-336
 *        trim_and_segment_raw         ref: src/thirdparty/scrappie/scrappie_common.c:122-190
 *        detect_events                ref: src/thirdparty/scrappie/event_detection.c:268-319
 *        recalibrate_model            ref: src/nanopolish_methyltrain.cpp:204-307
 *
 * The reference has no FFI layer: its seam is those C++ free functions, called with
 * HMMInputData / HMMInputSequence / SquiggleRead.  The C++ mirror of that call surface
 * lives in nanopolish_b200/host/ and lowers onto the functions below; INTEGRATION.md shows
 * the binding a nanopolish maintainer would add.
 *
 * Conventions
 *   - plain C, plain pointers and sizes; no C++/torch/CUDA types in any signature
 *     (a CUDA stream is passed as void*).
 *   - every function returns NPH_OK (0) or a negative nph_status; nothing throws, nothing
 *     calls exit().  nph_strerror() gives a message, nph_last_error(ctx) the CUDA detail.
 *   - the caller owns every host buffer for the duration of the call; the context owns
 *     all device memory.  A context is bound to one device and one stream and must not be
 *     used from two threads at once (use one context per OpenMP thread, or a mutex).
 *   - there is NO CPU fallback: without a CUDA device nph_create() fails with
 *     NPH_ERR_NO_DEVICE and nothing else can be called.
 *   - results are bit-identical to the reference's float arithmetic (same operation order,
 *     same quantised table logsum, IEEE add/mul/div, no FMA contraction); see DESIGN.md.
 */
#ifndef NPH_H
#define NPH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NPH_VERSION_MAJOR 0
#define NPH_VERSION_MINOR 1

typedef enum {
    NPH_OK = 0,
    NPH_ERR_NO_DEVICE = -1,   /* no usable CUDA device / driver: there is no CPU path */
    NPH_ERR_CUDA = -2,        /* a CUDA runtime call failed; see nph_last_error */
    NPH_ERR_INVALID = -3,     /* bad argument (null pointer, out-of-range index, ...) */
    NPH_ERR_NOMEM = -4,       /* device or host allocation failed */
    NPH_ERR_STATE = -5,       /* call sequence error (e.g. score before load) */
    NPH_ERR_UNSUPPORTED = -6  /* a shape the kernels do not handle (documented limits) */
} nph_status;

/* flags of profile_hmm_score / profile_hmm_align.
 * ref: src/hmm/nanopolish_profile_hmm.h:34-38 (HAF_ALLOW_PRE_CLIP, HAF_ALLOW_POST_CLIP) */
#define NPH_HAF_ALLOW_PRE_CLIP  1u
#define NPH_HAF_ALLOW_POST_CLIP 2u

typedef struct nph_ctx nph_ctx;

/* One strand of one SquiggleRead: the part of it the hot path reads.
 * ref: SquiggleRead::events[strand] (src/nanopolish_squiggle_read.h:277-299),
 *      SquiggleScalings (:63-93), events_per_base[strand] (:293). 64 bytes. */
typedef struct {
    uint64_t event_off;       /* first event of this read in ev_mean[] / ev_start_time[] */
    uint32_t n_events;
    uint32_t reserved;
    double scale;             /* SquiggleScalings::scale   */
    double shift;             /*                 ::shift   */
    double drift;             /*                 ::drift   */
    double var;               /*                 ::var     */
    double log_var;           /*                 ::log_var (= log(var), cached by set4/set6) */
    double events_per_base;   /* SquiggleRead::events_per_base[strand] */
} nph_read;

/* One profile_hmm_score call == one (HMMInputSequence, HMMInputData, flags) triple.
 * ref: HMMInputData (src/common/nanopolish_common.h:53-62).  The sequence is passed as the
 * k-mer ranks HMMInputSequence::get_kmer_rank(ki, k, rc) returns for ki = 0..n_kmers-1
 * (src/hmm/nanopolish_hmm_input_sequence.h:76-91), i.e. already strand-resolved. 32 bytes. */
typedef struct {
    uint64_t rank_off;        /* first k-mer rank of this job in kmer_ranks[] */
    uint32_t read;            /* index into reads[] */
    uint32_t model_id;        /* from nph_model_upload: HMMInputData::pore_model */
    uint32_t event_start;     /* HMMInputData::event_start_idx */
    uint32_t event_stop;      /* HMMInputData::event_stop_idx (inclusive) */
    uint32_t n_kmers;         /* sequence.length() - k + 1 */
    int8_t   stride;          /* HMMInputData::event_stride: +1, or -1 when event_stop < event_start */
    uint8_t  rc;              /* HMMInputData::rc (informational: ranks are already resolved) */
    uint8_t  flags;           /* NPH_HAF_* */
    uint8_t  reserved;
} nph_hmm_job;

/* One adaptive_banded_simple_event_align call: a whole read against its basecalled sequence. */
typedef struct {
    uint64_t rank_off;        /* first k-mer rank (forward strand, alphabet->kmer_rank) in kmer_ranks[] */
    uint64_t pairs_off;       /* where this read's AlignedPairs go in pairs_out[] (in pairs) */
    uint32_t read;            /* index into reads[] (scalings as set by the MoM estimate: drift 0, var 1) */
    uint32_t n_kmers;
    uint32_t pairs_cap;       /* room at pairs_off, in pairs; n_events + n_kmers always suffices */
    uint32_t reserved;
} nph_abea_job;

/* ref: AlignedPair (src/alignment/nanopolish_anchor.h:18-22) */
typedef struct { int32_t ref_pos; int32_t read_pos; } nph_aligned_pair;

/* status of one ABEA job.  The reference returns an empty vector for every failure
 * (src/nanopolish_raw_loader.cpp:365-372); n_pairs is 0 in exactly those cases. */
#define NPH_ABEA_OK              0
#define NPH_ABEA_LOW_EMISSION    1   /* avg_log_emission < -5.0 */
#define NPH_ABEA_NOT_SPANNED     2   /* path does not run from k-mer 0 to k-mer n_kmers-1 */
#define NPH_ABEA_MAX_GAP         4   /* more than 50 consecutive skipped k-mers */
#define NPH_ABEA_NO_END_CELL     8   /* last k-mer column never inside the band (reference behaviour undefined) */
#define NPH_ABEA_PAIRS_OVERFLOW 16   /* pairs_cap too small */
/* The record of a job that fails:
 *   NPH_ABEA_NO_END_CELL    : no path is walked.  status is that bit alone; n_aligned 0, max_gap 0, avg_log_emission 0.
 *   NPH_ABEA_PAIRS_OVERFLOW : the whole path is walked but QC is not run.  status is that bit alone; n_aligned and max_gap
 *                             are the path's, avg_log_emission is 0.  The job's slot holds pairs in no defined order.
 *   otherwise               : QC ran on the whole path; status is the bit-or of the QC bits (LOW_EMISSION, NOT_SPANNED,
 *                             MAX_GAP) and n_aligned, max_gap and avg_log_emission are the path's.
 * n_pairs is 0 for every failure.  A job never writes outside [pairs_off, pairs_off + pairs_cap). */
typedef struct {
    uint32_t n_pairs;         /* 0 when the reference would have returned an empty vector */
    int32_t  status;          /* bit-or of NPH_ABEA_* */
    int32_t  max_gap;         /* longest run of skipped k-mers on the path */
    uint32_t n_aligned;       /* path length before QC (== n_pairs when status == 0) */
    double   avg_log_emission;   /* mean emission over the path, summed in path order in FP64 */
} nph_abea_result;

/* One Viterbi state of profile_hmm_align.  ref: HMMAlignmentState (src/common/nanopolish_common.h:65-73);
 * l_posterior and log_transition_probability are left for the host wrapper (section 8f N1). */
typedef struct {
    uint32_t event_idx;
    uint32_t kmer_idx;
    float    l_fm;
    char     state;           /* 'M', 'B' (bad event) or 'K' (k-mer skip) */
    uint8_t  reserved[3];
} nph_align_state;

/* ---- context ------------------------------------------------------------------------- */

/* Create a context on CUDA device `device` with its own non-blocking stream. */
int nph_create(nph_ctx** ctx_out, int device);
/* Same, but run everything on the caller's stream (a cudaStream_t passed as void*; NULL = legacy
 * default stream).  Lets a host framework time/sequence the kernels with its own events. */
int nph_create_on_stream(nph_ctx** ctx_out, int device, void* cuda_stream);
int nph_destroy(nph_ctx* ctx);
const char* nph_strerror(int status);
const char* nph_last_error(const nph_ctx* ctx);
int nph_version(void);                              /* major*1000 + minor */
int nph_sync(nph_ctx* ctx);                         /* wait for everything queued on the context's stream */
void* nph_stream(nph_ctx* ctx);                     /* the cudaStream_t the kernels run on */

/* PoreModel::states as three parallel arrays (level_mean, level_stdv, level_log_stdv).
 * ref: PoreModelStateParams (src/pore_model/nanopolish_poremodel.h:20-36). Uploaded once per model. */
int nph_model_upload(nph_ctx* ctx, const double* level_mean, const double* level_stdv,
                     const double* level_log_stdv, uint32_t n_states, uint32_t k,
                     uint32_t alphabet_size, uint32_t* model_id_out);

/* ---- profile_hmm_score ------------------------------------------------------------------
 * One-shot form, host buffers in, host scores out (synchronous):
 *   scores_out[j] == profile_hmm_score(sequence_j, data_j, flags_j)   for j in [0, n_jobs)
 * with hmm_indel_bias_factor (src/hmm/nanopolish_profile_hmm_r9.cpp:19) == indel_bias.
 * A job with event range or k-mer count the reference would assert on yields NPH_ERR_INVALID. */
int nph_hmm_score_batch(nph_ctx* ctx,
                        const nph_read* reads, size_t n_reads,
                        const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                        const uint32_t* kmer_ranks, size_t n_ranks_total,
                        const nph_hmm_job* jobs, size_t n_jobs,
                        double indel_bias, float* scores_out);

/* Staged form of the same computation, for callers that keep a batch resident in HBM
 * (bench.py's device-resident timing, multi-GPU shards, repeated scoring with new jobs):
 *   nph_reads_load   : H2D of events + scalings, then the per-read device prologue
 *                      (drift-scaled levels get_drift_scaled_level, squiggle_read.h:149-154;
 *                       transitions calculate_transitions, profile_hmm_r9.inl:17-76)
 *   nph_hmm_jobs_load: H2D of ranks + jobs, scheduling order
 *   nph_hmm_score    : launches the forward kernel(s) on the context's stream (asynchronous);
 *                      scores go to scores_dev if non-NULL (device pointer, n_jobs floats)
 *                      else to an internal device buffer
 *   nph_hmm_scores_fetch: D2H of the internal score buffer + stream sync                    */
int nph_reads_load(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                   const float* ev_mean, const double* ev_start_time, size_t n_events_total);
int nph_hmm_jobs_load(nph_ctx* ctx, const uint32_t* kmer_ranks, size_t n_ranks_total,
                      const nph_hmm_job* jobs, size_t n_jobs, double indel_bias);
int nph_hmm_score(nph_ctx* ctx, float* scores_dev);
int nph_hmm_scores_fetch(nph_ctx* ctx, float* scores_out, size_t n_jobs);

/* The same computation with the sequences as BASE CODES instead of k-mer ranks — one byte per base on the wire and in HBM instead
 * of four per k-mer; the forward kernel forms each k-mer's rank from the codes while it scales the k-mer's Gaussian.
 * seq_codes holds, per job, the alphabet ranks Alphabet::rank(c) of the n_kmers + k - 1 symbols of the string the job's strand
 * reads: HMMInputSequence's m_seq for rc == 0, its m_rc_seq for rc == 1 (so that k-mer i is what get_kmer_rank(i, k, rc)
 * ranks: the k symbols at i, resp. at length - i - k; src/hmm/nanopolish_hmm_input_sequence.h:76-91).  In these calls
 * nph_hmm_job::rank_off is the offset of the job's first code in seq_codes, and nph_hmm_job::rc selects the direction.
 * A code outside the job's model alphabet yields NPH_ERR_INVALID. */
int nph_hmm_score_batch_seq(nph_ctx* ctx,
                            const nph_read* reads, size_t n_reads,
                            const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                            const uint8_t* seq_codes, size_t n_codes_total,
                            const nph_hmm_job* jobs, size_t n_jobs,
                            double indel_bias, float* scores_out);
int nph_hmm_jobs_load_seq(nph_ctx* ctx, const uint8_t* seq_codes, size_t n_codes_total,
                          const nph_hmm_job* jobs, size_t n_jobs, double indel_bias);

/* profile_hmm_score_set (ref: src/hmm/nanopolish_profile_hmm.cpp:32-56): combine the per-sequence
 * scores of each group of n_alt consecutive jobs, host side, in double through the table logsum:
 *   out[g] = (+)_i ( scores[g*n_alt + i] - log(n_alt) ).  Pure host arithmetic on fetched scores. */
int nph_score_set_combine(const float* scores, size_t n_groups, uint32_t n_alt, float* out);

/* ---- adaptive_banded_simple_event_align -------------------------------------------------
 * One-shot, host buffers (synchronous). pairs_out receives, for job j, results[j].n_pairs
 * AlignedPairs at pairs_out + jobs[j].pairs_off in the reference's order (ascending).
 * Both forms return NPH_ERR_INVALID for a k-mer rank >= the model's n_states, and for a batch with an event level outside
 * [-NPH_ABEA_MAX_LEVEL, NPH_ABEA_MAX_LEVEL] (NaN included) anywhere in the loaded events.  The device Gaussian is exact where
 * |level - mu'| < 2^12 (exact_math.cuh), which these levels keep for any model mean below 2048 pA.  Outside it the device and
 * the reference part: +-inf turns the device's division into NaN where the reference's gives -inf, and from
 * |level - mu'| / sigma' >= 2^64 the device's square overflows to -inf where the reference's (-0.5f * a) * a stays finite. */
#define NPH_ABEA_MAX_LEVEL 2048.0f
int nph_abea_batch(nph_ctx* ctx,
                   const nph_read* reads, size_t n_reads,
                   const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                   const uint32_t* kmer_ranks, size_t n_ranks_total,
                   const nph_abea_job* jobs, size_t n_jobs, uint32_t model_id,
                   nph_aligned_pair* pairs_out, size_t pairs_total, nph_abea_result* results);
/* Staged form (reads via nph_reads_load). */
int nph_abea_jobs_load(nph_ctx* ctx, const uint32_t* kmer_ranks, size_t n_ranks_total,
                       const nph_abea_job* jobs, size_t n_jobs, uint32_t model_id, size_t pairs_total);
int nph_abea_run(nph_ctx* ctx);
int nph_abea_fetch(nph_ctx* ctx, nph_aligned_pair* pairs_out, size_t pairs_total,
                   nph_abea_result* results, size_t n_jobs);

/* estimate_scalings_using_mom for each job's read/sequence: out[j] = {shift, scale} (drift 0, var 1).
 * NPH_ERR_INVALID for a k-mer rank >= the model's n_states. */
int nph_mom_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                  const float* ev_mean, size_t n_events_total,
                  const uint32_t* kmer_ranks, size_t n_ranks_total,
                  const nph_abea_job* jobs, size_t n_jobs, uint32_t model_id, double* shift_scale_out);

/* ---- profile_hmm_align (Viterbi; section 8f N1) ------------------------------------------
 * states_out receives, for job j, n_states_out[j] HMMAlignmentStates at states_out + states_off[j] in ascending
 * event order; states_off has n_jobs + 1 entries and states_off[j+1] - states_off[j] is the room for job j
 * (n_events + n_kmers always suffices).  n_states_out[j] == 0 and scores_out[j] == -inf where the reference would
 * trip an assert (fewer than two events, or the best path runs into a -inf cell) and where the room is shorter than the
 * path.  Offsets must not decrease (NPH_ERR_INVALID); states_out before states_off[0] is left untouched.
 * scores_out (optional) = l_fm of the last state.
 * Limit: the movement trace of the batch's largest window, 2 * (steps + 1) * 32*C bytes per warp (C = 1..8 columns per
 * lane, steps ~ E * ceil(K / 32C) + K/C), is kept for every resident warp; the number of resident CTAs shrinks so that the
 * traces stay within 16 GiB, and a batch whose largest window needs more than that for a single CTA of 16 warps returns
 * NPH_ERR_UNSUPPORTED: about E*K > 5.4e8, from K = E = 23 046 on for a square window.  On a 132-SM H100 the cap starts
 * at about K = E = 1 983.
 * ref: profile_hmm_align_r9, src/hmm/nanopolish_profile_hmm_r9.cpp:73-204. */
int nph_hmm_align_batch(nph_ctx* ctx,
                        const nph_read* reads, size_t n_reads,
                        const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                        const uint32_t* kmer_ranks, size_t n_ranks_total,
                        const nph_hmm_job* jobs, size_t n_jobs, double indel_bias,
                        nph_align_state* states_out, const uint64_t* states_off,
                        uint32_t* n_states_out, float* scores_out);
/* The same against the reads a preceding nph_reads_load left resident in HBM: eventalign re-aligns one ~100-base
 * segment per read per round (align_read_to_ref, src/alignment/nanopolish_eventalign.cpp:691-823), each round's
 * jobs depending on the previous round's paths, so the events go up once and only jobs/states travel per round. */
int nph_hmm_align(nph_ctx* ctx,
                  const uint32_t* kmer_ranks, size_t n_ranks_total,
                  const nph_hmm_job* jobs, size_t n_jobs, double indel_bias,
                  nph_align_state* states_out, const uint64_t* states_off,
                  uint32_t* n_states_out, float* scores_out);

/* ---- eventalign: a read's whole segment chain on the device (section 8f N1) ------------------------------
 * align_read_to_ref (src/alignment/nanopolish_eventalign.cpp:612-827) walks one BAM-aligned segment of a read in
 * ~100-base steps: pick the aligned pair ~100 reference bases ahead (get_end_pair :196-207), the event nearest to its
 * read k-mer (SquiggleRead::get_closest_event_to, src/nanopolish_squiggle_read.cpp:160-186), profile_hmm_align over
 * that window, emit up to 50 event alignments (all of them in the last section), restart from the last one emitted.
 * Each step depends on the previous path, so one warp walks one chain from start to end: cursor, Viterbi fill,
 * backtrack and emission stay on the device, and a batch of reads is ONE launch instead of one per step.
 * A chain is one BAM segment (the pieces between N operations) of one read strand, already trimmed to the region and
 * to the read's last k-mer by the caller (trim_aligned_pairs_to_ref_region / _to_kmer, :166-193).
 * Reads: the batch a preceding nph_reads_load left resident. */
typedef struct {
    uint64_t pair_off;        /* this segment's aligned pairs (ref_pos ascending, read_pos = BAM query k-mer) in pairs[] */
    uint64_t map_off;         /* the read's base_to_event_map[*].indices[strand].start in event_map_start[] (-1: none) */
    uint64_t rank_off;        /* the record's reference in ref_ranks_fwd[] / ref_ranks_rc[]: entry p = rank of the k-mer at
                                 reference offset p (fwd) / of its reverse complement as HMMInputSequence resolves it (rc) */
    uint64_t out_off;         /* where this chain's records go in records_out[] */
    uint32_t read;            /* index into the resident reads */
    uint32_t model_id;
    uint32_t n_pairs;
    uint32_t map_len;         /* base_to_event_map.size() */
    uint32_t ref_len;         /* ref_seq.length(); ref_len - k + 1 rank entries */
    uint32_t read_seq_len;    /* read_sequence.size() (SquiggleRead::flip_k_strand) */
    uint32_t out_cap;         /* room at out_off; abs(last_event - first_event) + 2 always suffices */
    int32_t  ref_offset;      /* record->core.pos */
    int32_t  first_event;     /* get_closest_event_to of the segment's first pair (after flip_k_strand if reversed) */
    int32_t  last_event;      /* ... of its last pair */
    uint8_t  do_base_rc;      /* bam_is_rev(record) */
    uint8_t  rc;              /* HMMInputData::rc == rc_flags[strand] */
    uint8_t  k;
    uint8_t  reserved;
} nph_ea_chain;
/* one EventAlignment (src/alignment/nanopolish_eventalign.h:54-71) without its strings: ref_kmer and model_kmer are
 * substrings of the reference at ref_position (model_kmer reverse-complemented for rc reads, NNNNNN for 'B') */
typedef struct { int32_t ref_position; int32_t event_idx; uint8_t hmm_state; uint8_t reserved[3]; } nph_ea_record;
#define NPH_EA_OK               0
#define NPH_EA_WINDOW_TOO_LARGE 1   /* a window has more k-mers or events than the kernel's single-strip scratch holds:
                                       re-run this read through nph_hmm_align rounds (records so far are valid) */
#define NPH_EA_RC_STRIDE        2   /* event order disagrees with rc (the reference asserts, profile_hmm_r9.inl:275) */
#define NPH_EA_OUT_OVERFLOW     4   /* out_cap too small */
#define NPH_EA_BAD_EVENT        8   /* a cursor event lies outside the read */
typedef struct { uint32_t n_records; uint32_t n_windows; int32_t status; uint32_t reserved; } nph_ea_result;
int nph_eventalign_chain(nph_ctx* ctx,
                         const nph_aligned_pair* pairs, size_t n_pairs_total,
                         const int32_t* event_map_start, size_t n_map_total,
                         const uint32_t* ref_ranks_fwd, const uint32_t* ref_ranks_rc, size_t n_ranks_total,
                         const nph_ea_chain* chains, size_t n_chains, double indel_bias,
                         nph_ea_record* records_out, size_t records_total, nph_ea_result* results_out);
/* The staged form: the same inputs, checks and launch, but only the results come back; the records stay on the device, where
 * nph_eventalign_tsv formats them and nph_eventalign_records_fetch copies them out (nph_eventalign_chain is the two in one
 * call).  They stay valid until the next call on this context that loads reads or uses the alignment scratch (any alignment,
 * ABEA or raw-read call); after that the two consumers return NPH_ERR_STATE. */
int nph_eventalign_chain_run(nph_ctx* ctx,
                             const nph_aligned_pair* pairs, size_t n_pairs_total,
                             const int32_t* event_map_start, size_t n_map_total,
                             const uint32_t* ref_ranks_fwd, const uint32_t* ref_ranks_rc, size_t n_ranks_total,
                             const nph_ea_chain* chains, size_t n_chains, double indel_bias,
                             size_t records_total, nph_ea_result* results_out);
int nph_eventalign_records_fetch(nph_ctx* ctx, nph_ea_record* records_out, size_t records_total);

/* ---- eventalign.tsv on the device -----------------------------------------------------------------------
 * The rows of emit_event_alignment_tsv (src/alignment/nanopolish_eventalign.cpp:398-484) for the records of the last
 * nph_eventalign_chain_run, formatted where they are: one row per record, chains in the order given, records in order, the
 * bytes of consecutive rows adjacent.  What a row needs beyond the resident records, rank tables, models and reads comes in
 * flat arrays: per output read (one BAM record: all its chains) the names, the upper-cased, disambiguated reference and its
 * reverse complement, the strand's unscaled event means, stdv and duration (one per event of the read), and for
 * --signal-index / --samples the events' start times and the raw samples. */
typedef struct {
    uint64_t contig_off, name_off;       /* in text[] */
    uint64_t ref_off;                    /* in ref[] and rc_ref[]: ref_len characters, as the read's chains index them */
    uint64_t event_off;                  /* in ev_mean[], ev_stdv[], ev_duration[], ev_start_time[]: n_events entries */
    uint64_t sample_off, n_samples;      /* in samples[] (--samples) */
    uint64_t read_idx;                   /* printed as %zu without -n */
    uint64_t sample_start_time;          /* SquiggleRead::sample_start_time */
    double   sample_rate, drift;
    uint32_t contig_len, name_len, ref_len, n_events;
    uint32_t strand_idx;                 /* 0 't', 1 'c' */
    uint32_t reserved;
} nph_ea_tsv_read;
typedef struct {
    const nph_ea_tsv_read* reads; size_t n_reads;
    const uint32_t* chain_read;          /* per chain of the run: its output read, non-decreasing */
    const char* text; size_t n_text;
    const char* ref; const char* rc_ref; size_t n_ref;
    const float* ev_mean; const float* ev_stdv; const float* ev_duration;
    const double* ev_start_time;         /* may be NULL without --signal-index / --samples */
    size_t n_events;
    const float* samples; size_t n_samples;   /* may be NULL without --samples */
} nph_ea_tsv_batch;
typedef struct { uint8_t print_read_names, scale_events, write_signal_index, write_samples; } nph_ea_tsv_options;
/* Refusals are per read: a read with a value the exact formatter does not take (a non-finite or huge stdv, duration, level or
 * sample, the 0 / 0 of an event mean of exactly zero at a 'B' state, a sample range outside the read's samples under --samples)
 * or with a chain whose status is not NPH_EA_OK gets no bytes and read_refused_out[read] = 1; the caller formats it with the C
 * library.  read_off_out: n_reads + 1 byte offsets; row_off_out (may be NULL): one per record + 1.  tsv_out is best
 * page-locked.  cap too small: NPH_ERR_INVALID with *n_bytes_out set and the offset tables filled.  NPH_ERR_STATE without
 * resident records. */
int nph_eventalign_tsv(nph_ctx* ctx, const nph_ea_tsv_batch* in, const nph_ea_tsv_options* opt, char* tsv_out, size_t cap,
                       uint64_t* row_off_out, uint64_t* read_off_out, uint8_t* read_refused_out, uint64_t* n_bytes_out);

/* ---- call-methylation: window enumeration + both scores per motif group on the device (section 8f N3) -----
 * calculate_methylation_for_read (src/basemods/nanopolish_basemods.cpp:238-457) from "Scan the sequence for motifs"
 * (:301) to the two profile_hmm_score calls (:383-392), for a whole BamProcessor batch in one call: the motif scan,
 * the grouping of sites closer than min_separation, the window (min_flank either side, span <= max_span, not within
 * min_separation of the alignment start), AlignmentDB::_find_by_ref_bounds on the read's event alignment
 * (src/alignment/nanopolish_alignment_db.cpp:688-731), the region filter, the unmethylated / methylated
 * HMMInputSequence pair (Alphabet::methylate, reverse_complement with its methylated-site units) as k-mer ranks, and the
 * two forward scores.  Nothing O(bases) or O(groups) is left to the host: it hands over the reference substring and
 * the event alignment of each (record, strand) and receives one nph_meth_site per scored group.
 * A record = one BAM record x one strand of its read.  ref_bases holds ref_seq of every record: the reference over
 * [record->core.pos, bam_endpos], already through gDNAAlphabet.disambiguate() (upper-case ACGT).  aligned_events holds
 * EventAlignmentRecord::aligned_events (ref_pos ascending, read_pos = event index; alignment_db.cpp:50-91). */
#define NPH_METH_MAX_SITES 4
#define NPH_METH_MAX_SITE_LEN 8
#define NPH_METH_MAX_WINDOW 1024     /* max_span + 2 * min_flank + 1 must not exceed this */
typedef struct {
    uint64_t ref_off;         /* first base of this record's ref_seq in ref_bases[] */
    uint64_t pair_off;        /* first aligned_events entry in aligned_events[] */
    uint32_t read;            /* index into reads[]: events[strand] of the record's SquiggleRead */
    uint32_t model_id;        /* sr.get_model(strand, methylation_type): the model over the methylation alphabet */
    uint32_t ref_len;         /* ref_seq.size() */
    uint32_t n_pairs;
    int32_t  ref_start_pos;   /* record->core.pos */
    uint8_t  rc;              /* EventAlignmentRecord::rc -> HMMInputData::rc */
    uint8_t  strand;          /* informational (sites of the two strands of one read are merged by the caller) */
    uint8_t  reserved[2];
} nph_meth_record;            /* 40 bytes */
typedef struct {
    int32_t  min_separation;  /* MethylationCallingParameters::min_separation (10), basemods.h:56 */
    int32_t  min_flank;       /* ::min_flank (10) */
    int32_t  max_span;        /* 200: groups spanning more are skipped, basemods.cpp:336 */
    int32_t  min_event_span;  /* 10: abs(e2 - e1) <= 10 skips the group, :363 */
    int32_t  region_start;    /* -1: no restriction (the -w window), :398-401 */
    int32_t  region_end;
    uint32_t k;               /* sr.get_model_k(strand) */
    uint32_t alphabet_size;   /* of the methylation alphabet (5 for cpg: ACGMT) */
    char     bases[8];        /* its symbols in rank order, NUL padded ("ACGMT") */
    char     complements[8];  /* complement of each symbol, same order ("TGCGA") */
    uint32_t n_sites;         /* Alphabet::num_recognition_sites() (1 for cpg, 2 for dcm) */
    uint32_t site_len;        /* Alphabet::recognition_length() */
    char     sites[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];                        /* get_recognition_site(i): "CG" */
    char     sites_methylated[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];             /* ..._methylated(i): "MG" */
    char     sites_methylated_complement[NPH_METH_MAX_SITES][NPH_METH_MAX_SITE_LEN];  /* ..._methylated_complement(i): "GM" */
} nph_meth_params;
/* One scored group of one record == the strand-specific half of a ScoredSite (basemods.h:25-43). */
typedef struct {
    int32_t  start_position;  /* first motif site of the group, reference coordinates */
    int32_t  end_position;    /* last motif site of the group */
    uint32_t n_motif;
    uint32_t record;          /* index into records[] */
    float    ll_unmethylated; /* profile_hmm_score(unmethylated, data, PRE_CLIP | POST_CLIP) */
    float    ll_methylated;
} nph_meth_site;              /* 24 bytes */
/* One-shot: host buffers in, host sites out (synchronous).  site_off_out has n_records + 1 entries: the sites of
 * record r are sites_out[site_off_out[r] .. site_off_out[r+1]) in ascending start_position.  sites_cap is the room in
 * sites_out; sum over records of (ref_len / (min_separation + 1) + 2) always suffices, NPH_ERR_INVALID if it was too
 * small (nph_last_error says how many were needed).  n_scored_events_out (optional): sum over groups of 2 * (abs(e2 - e1) + 1),
 * the unit of the events/s metric.  A group whose event indices lie outside its read (the reference would read out of
 * bounds) or whose clamped window is shorter than k yields NPH_ERR_INVALID. */
int nph_methylation_batch(nph_ctx* ctx,
                          const nph_read* reads, size_t n_reads,
                          const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                          const char* ref_bases, size_t n_ref_total,
                          const nph_aligned_pair* aligned_events, size_t n_pairs_total,
                          const nph_meth_record* records, size_t n_records,
                          const nph_meth_params* params, double indel_bias,
                          uint64_t* site_off_out, nph_meth_site* sites_out, size_t sites_cap,
                          uint64_t* n_scored_events_out);
/* The same with the event alignments in COMPACT form — 2 bytes per reference base instead of 8 per aligned pair, which matters
 * because this call is PCIe bound (the event alignment is larger than the events themselves).  event_deltas runs parallel to
 * ref_bases (entry ref_off + o belongs to reference offset o of the record): NPH_METH_NO_PAIR where aligned_events has no entry
 * with ref_pos == ref_start_pos + o (a deleted reference base, the record's boundary k-mers), else that entry's event index
 * minus the event index of the previous entry (minus first_event[record] for the record's first entry).  The device rebuilds
 * the (ref_pos, event index) list by a prefix sum; results are identical to the pair form.  records[].pair_off / n_pairs are
 * ignored.  Requires strictly increasing ref_pos inside a record (true of every EventAlignmentRecord) and event-index steps
 * that fit an int16 (a caller that meets a larger step uses the pair form). */
#define NPH_METH_NO_PAIR (-32768)
int nph_methylation_batch_compact(nph_ctx* ctx,
                                  const nph_read* reads, size_t n_reads,
                                  const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                  const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total,
                                  const int32_t* first_event,
                                  const nph_meth_record* records, size_t n_records,
                                  const nph_meth_params* params, double indel_bias,
                                  uint64_t* site_off_out, nph_meth_site* sites_out, size_t sites_cap,
                                  uint64_t* n_scored_events_out);
int nph_methylation_load_compact(nph_ctx* ctx, const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total,
                                 const int32_t* first_event, const nph_meth_record* records, size_t n_records,
                                 const nph_meth_params* params, double indel_bias);
/* Staged form against the reads a preceding nph_reads_load left resident:
 *   nph_methylation_load : H2D of the reference bases, event alignments and records
 *   nph_methylation_run  : enumerate -> schedule -> score -> fill the site records, all on the device
 *                          (two small read-backs inside: the counts that size the job arrays, the schedule summary)
 *   nph_methylation_fetch: D2H of the offsets and site records */
int nph_methylation_load(nph_ctx* ctx, const char* ref_bases, size_t n_ref_total,
                         const nph_aligned_pair* aligned_events, size_t n_pairs_total,
                         const nph_meth_record* records, size_t n_records,
                         const nph_meth_params* params, double indel_bias);
int nph_methylation_run(nph_ctx* ctx);
/* counts of the most recent nph_methylation_run: scored groups, forward jobs (2 per group), scored events */
int nph_methylation_counts(nph_ctx* ctx, uint64_t* n_sites_out, uint64_t* n_jobs_out, uint64_t* n_scored_events_out);
int nph_methylation_fetch(nph_ctx* ctx, uint64_t* site_off_out, nph_meth_site* sites_out, size_t sites_cap);
/* The site records of the most recent nph_methylation_run where they lie in device memory (valid until the next call on
 * this context; ordered behind the run on the context's stream), for a caller that ships them GPU to GPU — a multi-GPU
 * driver gathering every rank's records with NCCL — without a host hop. */
int nph_methylation_sites_dev(nph_ctx* ctx, const nph_meth_site** sites_dev_out, uint64_t* n_sites_out);
/* The rows of methylation_calls.tsv for the most recent nph_methylation_run, formatted on the device — the reference's writer
 * (src/nanopolish_call_methylation.cpp:113-140: chromosome, strand, start, end, read_name, log_lik_ratio, log_lik_methylated,
 * log_lik_unmethylated, num_calling_strands, num_motifs, sequence; "%.2lf" for the three likelihoods) applied to every site
 * record in record order, for records that are their read's only scored strand (num_calling_strands 1; every 1D read).
 * contig: the chromosome name of the batch; read_names + name_off (n_records + 1 offsets into read_names, no terminators):
 * the read name of each record; is_reverse[n_records]: bam1_is_rev of each record ('-' / '+').  tsv_out receives
 * *n_bytes_out bytes (no terminator).  NPH_ERR_INVALID with *n_bytes_out set if cap was too small; NPH_ERR_UNSUPPORTED if a
 * likelihood is not finite or beyond 2^52 (the C library's arbitrary-precision path: fetch the sites and format on the host). */
int nph_methylation_tsv(nph_ctx* ctx, const char* contig, const char* read_names, const uint32_t* name_off,
                        const uint8_t* is_reverse, char* tsv_out, size_t cap, uint64_t* n_bytes_out);
/* One-shot of the whole caller: nph_methylation_batch_compact's inputs in, methylation_calls.tsv rows out (the site
 * records never cross PCIe).  On NPH_ERR_UNSUPPORTED (see nph_methylation_tsv) the batch has been scored: the caller
 * may nph_methylation_fetch the records and format them itself. */
int nph_methylation_batch_compact_tsv(nph_ctx* ctx,
                                      const nph_read* reads, size_t n_reads,
                                      const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                      const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total,
                                      const int32_t* first_event,
                                      const nph_meth_record* records, size_t n_records,
                                      const nph_meth_params* params, double indel_bias,
                                      const char* contig, const char* read_names, const uint32_t* name_off, const uint8_t* is_reverse,
                                      char* tsv_out, size_t cap, uint64_t* n_bytes_out,
                                      uint64_t* n_sites_out, uint64_t* n_scored_events_out);

/* ---- call-methylation: per-site methylation frequency accumulated on the device ------------------------------------------
 * The table the reference's scripts/calculate_methylation_frequency.py builds from methylation_calls.tsv (chromosome, start, end,
 * num_motifs_in_group, called_sites, called_sites_methylated, methylated_frequency, group_sequence), kept on the device while
 * batches are scored, so that a caller who wants frequencies needs neither the TSV nor the script.  Folding the batches in order
 * gives the script's output for the concatenation of the batches' TSV rows, byte for byte:
 *   a row is skipped when abs(llr) < call_threshold * num_motifs (llr: the row's printed "%.2lf" log_lik_ratio, as the script
 *   parses it) and is methylated when llr > 0; it counts num_motifs calls at (chromosome, start, end), or, with split_groups and
 *   num_motifs > 1, one call per "CG" of its sequence column (overlapping matches too) at (chromosome, start + offset of that CG
 *   from the first, same) with group size 1 and sequence "split-group"; a key keeps the group size and sequence of the first row
 *   that created it.
 * The accumulator belongs to the context (freed by nph_destroy) and grows on the device as keys arrive. */
typedef struct {
    double   call_threshold;  /* -c (2.0) */
    uint32_t split_groups;    /* -s: nonzero splits multi-site groups into their CpGs */
    uint32_t reserved;
} nph_methfreq_params;
/* Empties the accumulator and sets its parameters (NULL: the script's defaults, 2.0 and no split).  A context starts with an
 * empty accumulator and the defaults. */
int nph_methfreq_reset(nph_ctx* ctx, const nph_methfreq_params* params);
/* Folds the rows of the most recent call-methylation run on this context (the rows nph_methylation_tsv would write, in its
 * order; the same one-strand contract) under contig_id (< 2^20; its name is given to nph_methfreq_tsv).  Call it before the
 * next run on the context: the run replaces the site records.  One small read-back; no per-site work on the host.
 * NPH_ERR_STATE without a run.  A refused batch leaves the accumulator unchanged: NPH_ERR_UNSUPPORTED for a likelihood that is
 * not finite or beyond 2^52, a printed ratio of 2^53 / 100 or more, a negative start or a group spanning 2^13 bases or more;
 * NPH_ERR_INVALID for a group whose sequence column would start before its record's reference (as nph_methylation_tsv). */
int nph_methfreq_add(nph_ctx* ctx, uint32_t contig_id);
/* distinct keys, calls counted (rows that passed the threshold; one per CpG of a split group), rows skipped by the threshold */
int nph_methfreq_counts(nph_ctx* ctx, uint64_t* n_keys_out, uint64_t* n_calls_out, uint64_t* n_ambiguous_out);
/* The frequency table so far: the header and one row per key, sorted by (name, start, end) as Python sorts them (names bytewise).
 * names + name_off (n_contigs + 1 offsets into names, no terminators): the name of each contig id.  out receives *n_bytes_out
 * bytes (no terminator); the accumulator is kept, so folding may go on.  NPH_ERR_INVALID with *n_bytes_out set if cap was too
 * small; NPH_ERR_INVALID for duplicate names or a folded contig id without a name. */
int nph_methfreq_tsv(nph_ctx* ctx, const char* names, const uint32_t* name_off, uint32_t n_contigs,
                     char* out, size_t cap, uint64_t* n_bytes_out);

/* ---- variants: candidate screening on the device (section 8f N2, BASELINE configs[4]) -----------------------------
 * generate_candidate_single_base_edits (src/nanopolish_call_variants.cpp:288-361) for a reference region: at every position i
 * the window [i - flank, i + 1 + flank] (22 bases for flank 10), up to nine candidate edits of base i — for j in ACGT order
 * the substitution to j and the insertion of j behind it (both skipped when j is the reference base), then the deletion of
 * base i (skipped when it equals base i - 1) — each scored with score_variant_thresholded
 * (src/common/nanopolish_variant.cpp:765-799): over the event sequences of the window
 * (AlignmentDB::get_event_subsequences, src/alignment/nanopolish_alignment_db.cpp:172-221: every record whose event alignment
 * bounds the window, event span below 20 events per base), in record order,
 *     if (fabs(total) < score_threshold) total += profile_hmm_score_set(variant) - profile_hmm_score_set(base)
 * — the reference's single-thread semantics (its `omp parallel for` makes the exit point racy).  The early exit is honoured
 * in the work done: reads are scored reads_per_round at a time, and only candidates whose total is still inside the
 * threshold get jobs in the next round (a candidate that leaves it mid-round ignores the rest of that round, exactly like the
 * sequential loop).  Window enumeration, the k-mer ranks of the ten sequences per position and strand, job emission, the
 * forward scores and the accumulation all run on the device; the host drives the rounds (one count read-back per round).
 * No methylation alternatives (opt::methylation_types empty, the default); nph_screen_edits_batch_methylation below takes -q types.
 * Records: nph_meth_record with ref_off = offset of the record's compact event alignment in event_deltas[] (ref_len entries,
 * entry o <-> reference position ref_start_pos + o; NPH_METH_NO_PAIR / steps as in nph_methylation_batch_compact),
 * pair_off / n_pairs unused, model_id = the read's base model.  Record order = AlignmentDB's m_event_records order.
 * ref_bases: the region's reference, ref_bases[p] = base at position region_start + p, n_ref_bases = region_end - region_start + 1
 * (AlignmentDB's m_region_start .. m_region_end inclusive); positions screened: region_start .. region_end - 1. */
#define NPH_SCREEN_SLOTS 9          /* per position: j = 0..3 (ACGT): slot 2j = substitution to j, 2j + 1 = insertion of j; slot 8 = deletion */
typedef struct {
    int32_t  flank;               /* opt::screen_flanking_sequence (10); the window must fit NPH_SCREEN_MAX_WINDOW */
    uint32_t score_threshold;     /* opt::screen_score_threshold (100) */
    uint32_t alignment_flags;     /* NPH_HAF_* handed to profile_hmm_score_set */
    uint32_t k;                   /* k of the reads' base model (nucleotide alphabet) */
    uint32_t reads_per_round;     /* reads of a position scored between two early-exit tests (8) */
    int32_t  region_start;        /* m_region_start */
} nph_screen_params;
#define NPH_SCREEN_MAX_WINDOW 64
/* qualities_out: NPH_SCREEN_SLOTS doubles per screened position (position region_start + p at p * NPH_SCREEN_SLOTS): the
 * Variant::quality score_variant_thresholded returns; NaN for a candidate the reference does not generate (j == reference base,
 * redundant deletion) and for positions whose window leaves the region (are_coordinates_valid fails: the reference skips them).
 * n_reads_out (optional): event sequences per position.  n_scored_events_out (optional): DP rows scored in all rounds. */
int nph_screen_edits_batch(nph_ctx* ctx,
                           const nph_read* reads, size_t n_reads,
                           const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                           const char* ref_bases, size_t n_ref_bases,
                           const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                           const nph_meth_record* records, size_t n_records,
                           const nph_screen_params* params, double indel_bias,
                           double* qualities_out, uint32_t* n_reads_out, uint64_t* n_scored_events_out);
/* Staged form (reads resident): load, run (all rounds; asynchronous device work between the per-round read-backs), fetch. */
int nph_screen_load(nph_ctx* ctx, const char* ref_bases, size_t n_ref_bases, const int16_t* event_deltas, size_t n_deltas_total,
                    const int32_t* first_event, const nph_meth_record* records, size_t n_records,
                    const nph_screen_params* params, double indel_bias);
int nph_screen_run(nph_ctx* ctx);
/* counters of the most recent nph_screen_run: rounds; forward jobs and scored events (DP rows) actually run; what scoring every
 * read of every candidate (no early exit) would have cost in jobs (valid after nph_screen_fetch); and the DP rows the reference's
 * own loop scores for the same result — base and variant sequence per (candidate, read) until the candidate's total leaves the
 * threshold — the unit in which this workload's throughput is compared with the CPU arm (here the base haplotype of a read is
 * scored once per round for all its candidates, the reference scores it once per candidate) */
int nph_screen_counts(nph_ctx* ctx, uint32_t* n_rounds_out, uint64_t* n_jobs_out, uint64_t* n_scored_events_out, uint64_t* n_jobs_without_exit_out,
                      uint64_t* n_reference_events_out);
/* reference_rows_out (optional, one per position): the position's share of nph_screen_counts' n_reference_events */
int nph_screen_fetch(nph_ctx* ctx, double* qualities_out, uint32_t* n_reads_out, uint64_t* reference_rows_out);

/* Methylation-aware screening (`variants -q cpg`, `-q dam,dcm`): opt::methylation_types non-empty.  Every sequence the screening
 * scores (the base window and its nine edited versions) becomes profile_hmm_score_set's set (src/common/nanopolish_variant.cpp:158-178):
 * the sequence itself, then for each type in -q order Alphabet::methylate of it where that changes it (sites matched on the
 * window's characters: an N never completes one), scored against the read's model of that type; the set is folded with log(n)
 * penalties through the table log-sum.  An edit can create or destroy a site, so a candidate and its base can have different
 * numbers of alternatives.  Qualities are those of score_variant_thresholded(..., methylation_types); n_reference_events counts
 * (n(base) + n(variant)) x E per (candidate, read) added, n(s) = 1 + alternatives of s.  With n_types = 0 this is nph_screen_*. */
#define NPH_SCREEN_MAX_TYPES 4
typedef struct {
    uint32_t n_types;                                  /* opt::methylation_types.size() */
    uint32_t reserved;
    nph_meth_params alphabets[NPH_SCREEN_MAX_TYPES];   /* get_alphabet_by_name(type t), in -q order; only k, alphabet_size, bases, complements,
                                                          n_sites, site_len and the three site arrays are read */
} nph_screen_methylation;                              /* 616 bytes */
/* nph_screen_load plus the types.  alt_model_ids: n_records x n_types, entry r * n_types + t = read->get_model(strand, type t) of
 * record r.  NPH_ERR_INVALID: n_types > NPH_SCREEN_MAX_TYPES, a malformed alphabet, an alphabet whose k is not params.k, a model id out of
 * range or whose model's k / alphabet size differ from its alphabet's; NPH_ERR_UNSUPPORTED: recognition sites that can overlap each
 * other.  A refused load leaves nph_screen_run at NPH_ERR_STATE.  nph_screen_run / _counts / _fetch serve both loads. */
int nph_screen_load_methylation(nph_ctx* ctx, const char* ref_bases, size_t n_ref_bases, const int16_t* event_deltas, size_t n_deltas_total,
                                const int32_t* first_event, const nph_meth_record* records, size_t n_records,
                                const nph_screen_params* params, double indel_bias,
                                const nph_screen_methylation* meth, const uint32_t* alt_model_ids);
/* One-shot form: nph_screen_edits_batch with the types. */
int nph_screen_edits_batch_methylation(nph_ctx* ctx,
                                       const nph_read* reads, size_t n_reads,
                                       const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                       const char* ref_bases, size_t n_ref_bases,
                                       const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                       const nph_meth_record* records, size_t n_records,
                                       const nph_screen_params* params, double indel_bias,
                                       const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                                       double* qualities_out, uint32_t* n_reads_out, uint64_t* n_scored_events_out);

/* ---- event detection (section 8f N4: the step before ABEA) --------------------------------------
 * scrappie's detect_events as load_from_raw calls it: t-statistics over two windows on prefix sums, a short/long
 * peak detector, events between consecutive boundaries.
 * ref: src/thirdparty/scrappie/event_detection.c:35-319, event_detection.h:15-29 (parameters),
 *      src/nanopolish_squiggle_read.cpp:229-235 (call site). */
typedef struct {
    uint32_t window_length1, window_length2;   /* 3, 6 for DNA; 7, 14 for RNA */
    float threshold1, threshold2, peak_height;  /* 1.4, 9.0, 0.2 for DNA; 2.5, 9.0, 1.0 for RNA */
    uint32_t reverse_events;  /* nph_load_from_raw_batch only: 1 for direct RNA, whose events load_from_raw turns
                                 around to 5'->3' after the MoM estimate (src/nanopolish_squiggle_read.cpp:262-265) */
} nph_event_params;
/* scrappie's event_t reduced to what it computes here (pos/state are always -1 there) */
typedef struct { uint64_t start; float length; float mean; float stdv; uint32_t reserved; } nph_event;
typedef struct {
    uint64_t sample_off;      /* first raw sample of this read in raw[] (picoamps as float, like Fast5Data::rt.raw) */
    uint64_t event_off;       /* where this read's events go in events_out[] */
    uint32_t n_samples;
    uint32_t event_cap;       /* room at event_off; n_samples always suffices, n_samples/2 does in practice */
} nph_raw_read;
/* events_out[reads[i].event_off ...] receives n_events_out[i] events in scrappie's order; n_events_out[i] == 0 with
 * NPH_ERR_UNSUPPORTED returned if some event_cap was too small (nothing else can fail: every signal has >= 1 event). */
int nph_detect_events_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_raw_read* reads, size_t n_reads,
                            const nph_event_params* params, nph_event* events_out, size_t events_total, uint32_t* n_events_out);

/* ---- raw-signal trimming (section 8f N4: the step before event detection) --------------------------
 * trim_and_segment_raw(rt, trim_start, trim_end, varseg_chunk, varseg_thresh) on a raw_table that starts at
 * {start 0, end n_samples}: median absolute deviation per chunk, chunks at or below the varseg_thresh quantile of
 * those MADs dropped from both ends, then the fixed trims.  ranges_out[i] is the surviving [start, end) relative to
 * reads[i].sample_off; {0, 0} where the reference returns an empty table (or would trip its assert: fewer samples
 * than one chunk, or no chunk above the threshold).  Only sample_off and n_samples of nph_raw_read are used.
 * ref: src/thirdparty/scrappie/scrappie_common.c:9-190; call site src/nanopolish_squiggle_read.cpp:226-233
 *      (trim_start 200, trim_end 10, varseg_chunk 100, varseg_thresh 0.0).  varseg_chunk <= 128.
 * NPH_ERR_INVALID, before anything runs, for a NaN or infinite sample anywhere in raw[0, n_samples_total): the MADs are order
 * statistics, and with a NaN the reference's order depends on the C library's qsort. */
typedef struct { uint32_t start, end; } nph_raw_range;
int nph_trim_raw_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_raw_read* reads, size_t n_reads,
                       int32_t trim_start, int32_t trim_end, int32_t varseg_chunk, float varseg_thresh,
                       nph_raw_range* ranges_out);

/* ---- calibration after ABEA (section 8f N4: the step between ABEA and the HMM) ---------------------
 * For each ABEA job (same jobs[], kmer_ranks[], pairs[] and results[] as nph_abea_batch took and returned):
 *   base_to_event_out[rank_off + ki] = SquiggleRead::base_to_event_map[ki].indices[strand]   ({-1,-1}: no events)
 *   events_per_base                   = (max_event - min_event) / n_kmers
 *   shift, scale, var                 = recalibrate_model(read, model, strand,
 *                                           get_eventalignment_for_1d_basecalls(...), scale_var=true, scale_drift=false)
 * and the QC that follows.  reads[] carries the scalings the read has before the call (the MoM estimate); they come
 * back unchanged when the read is not recalibrated.  base_to_event_out may be NULL; its entries at ranks no job covers are
 * {-1,-1}.  The jobs' rank ranges [rank_off, rank_off + n_kmers) must not overlap (each job's map is built in place at its
 * rank_off): NPH_ERR_INVALID, before anything runs, when two of them do.
 * ref: src/nanopolish_squiggle_read.cpp:270-336,340-391; src/nanopolish_methyltrain.cpp:204-307. */
typedef struct { int32_t start, stop; } nph_event_range;      /* IndexPair, src/nanopolish_squiggle_read.h:32-37 */
#define NPH_CAL_OK              0
#define NPH_CAL_NOT_ALIGNED     1   /* ABEA returned no pairs: events cleared, events_per_base = 0 */
#define NPH_CAL_TOO_FEW_EVENTS  2   /* fewer than 200 'M' events: not recalibrated, events cleared */
#define NPH_CAL_HIGH_VAR        4   /* var > MIN_CALIBRATION_VAR (2.5): events cleared */
#define NPH_CAL_TOO_MANY_STAYS  8   /* events_per_base > 5.0: events cleared */
typedef struct {
    double shift, scale, drift, var;   /* arguments of SquiggleScalings::set4 */
    double events_per_base;
    uint32_t n_used;                   /* 'M' events that entered the normal equations */
    int32_t status;                    /* NPH_CAL_*; non-zero = the reference drops the read */
} nph_calibration;
int nph_recalibrate_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads, const float* ev_mean, size_t n_events_total,
                          const uint32_t* kmer_ranks, size_t n_ranks_total, const nph_abea_job* jobs, size_t n_jobs,
                          uint32_t model_id, const nph_aligned_pair* pairs, size_t pairs_total,
                          const nph_abea_result* results, nph_event_range* base_to_event_out, nph_calibration* calibrations_out);

/* ---- the whole read prologue in one call (section 8f N4) ------------------------------------------------
 * SquiggleRead::load_from_raw for a batch of reads: trim_and_segment_raw (200, 10, 100, 0.0) -> detect_events ->
 * SquiggleEvent conversion -> estimate_scalings_using_mom -> adaptive_banded_simple_event_align -> base_to_event_map,
 * events_per_base, recalibrate_model and the QC, chained on the device (the samples cross PCIe once, events never
 * come back in between).  ref: src/nanopolish_squiggle_read.cpp:226-336.
 * DNA: params = event_detection_defaults, a 6-mer nucleotide model.  Direct RNA: params = event_detection_rna with
 * reverse_events = 1, the 5-mer u_to_t_rna model, ranks of the sequence with U replaced by T (:206-213); the events
 * come back in 5'->3' order, each keeping the start time it had in acquisition order (so start times descend).
 * Outputs, per job j:  events [event_off_out[j], event_off_out[j+1]) of the four event arrays (compact, job order;
 * SquiggleEvent::log_stdv = logf(stdv) is left to the caller's libm), calibrations_out[j] (status != 0: the reference
 * clears the read's events; the arrays still hold them), base_to_event_out[rank_off + ki] (optional).
 * A read that trims to nothing (the reference aborts on it) gets no events and NPH_CAL_EMPTY_AFTER_TRIM.
 * NPH_ERR_UNSUPPORTED if events_cap is too small (n_samples_total / 3 always suffices).  NPH_ERR_INVALID for a k-mer rank
 * >= the model's n_states, and for any sample of raw[0, n_samples_total) outside [-NPH_ABEA_MAX_LEVEL, NPH_ABEA_MAX_LEVEL] (NaN
 * included; samples outside every job's slice too), before any step runs: an event's level is a mean of its samples, so this
 * keeps the events inside the range nph_abea_batch takes.  NPH_ERR_INVALID too, before any step runs, when two jobs' rank
 * ranges [rank_off, rank_off + n_kmers) overlap (as for nph_recalibrate_batch); base_to_event_out entries no live job
 * covers are {-1,-1}. */
#define NPH_CAL_EMPTY_AFTER_TRIM 16
typedef struct {
    uint64_t sample_off;      /* first raw sample (picoamps, float) of this read in raw[] */
    uint64_t rank_off;        /* first k-mer rank of the basecalled sequence in kmer_ranks[] (forward strand) */
    uint32_t n_samples;
    uint32_t n_kmers;         /* read_sequence.length() - k + 1 */
    double   sample_rate;     /* Fast5Data::channel_params.sample_rate */
} nph_raw_job;
int nph_load_from_raw_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total,
                            const uint32_t* kmer_ranks, size_t n_ranks_total,
                            const nph_raw_job* jobs, size_t n_jobs, uint32_t model_id, const nph_event_params* params,
                            uint64_t* event_off_out, float* ev_mean_out, float* ev_stdv_out, double* ev_start_time_out,
                            float* ev_duration_out, size_t events_cap,
                            nph_event_range* base_to_event_out, nph_calibration* calibrations_out);

/* The surviving sample range [start, end) of each job of the most recent nph_load_from_raw_batch on this context,
 * relative to the job's sample_off ({0, 0}: nothing survived).  It is what load_from_raw keeps with SRF_LOAD_RAW_SAMPLES
 * (samples[i] = rt.raw[rt.start + i], sample_start_time = 0; src/nanopolish_squiggle_read.cpp:251-258), which eventalign's
 * --samples / --signal-index read back.  NPH_ERR_STATE if n_jobs is not that call's job count. */
int nph_last_trim_ranges(nph_ctx* ctx, nph_raw_range* ranges_out, size_t n_jobs);

/* ---- poly(A) tail segmentation and length (nanopolish polya) ---------------------------------------------
 * Per read, what estimate_polya_for_single_read computes after loading (src/nanopolish_polya_estimator.cpp:786-813):
 * SegmentationHMM(scale, shift, var).segment_squiggle over the read's samples (:204-509: the 6-state Viterbi over every raw
 * sample, its backtrack and the region boundaries), estimate_unaligned_duration_profile (:564-599: 1 / the median per-k-mer
 * duration), estimate_polya_length (:638-662) and the three QC checks with their priority (:672-722, :803-813).
 * Inputs follow nph_load_from_raw_batch's outputs: ev_duration[event_off + e] is the read's SquiggleEvent::duration,
 * base_to_event[rank_off + ki] its base_to_event_map[ki].indices[0].  raw[sample_off ..] is the read's WHOLE raw signal
 * (SquiggleRead::samples with SRF_LOAD_RAW_SAMPLES, acquisition order, not reversed for direct RNA).
 * A job with loaded == 0 (the read is missing from the index) or n_events == 0 (load_from_raw cleared its events: any
 * NPH_CAL_* status != 0) is not computed: its result carries NPH_POLYA_READ_FAILED_LOAD and -1 values (:760-777).  NPH_ERR_INVALID, before anything runs, for a loaded job with fewer than 2 samples
 * (the reference's backtrack loop wraps), no k-mer, a sample, event or map slice outside the call's arrays, or a map entry
 * other than {-1, *} or {start, stop} with 0 <= start <= stop < n_events (the reference asserts), or a NaN duration in a mapped
 * span (the reference sorts the per-k-mer durations with std::sort, whose order with a NaN is undefined; +-inf durations and NaN
 * samples are computed as the reference computes them).  Secondary records and the
 * suffix clip (the length of the record's LAST CIGAR operation, whatever its type) are the caller's to take from the BAM. */
#define NPH_POLYA_PASS             0
#define NPH_POLYA_NOREGION         1   /* fewer than 200 adapter or poly(A) samples */
#define NPH_POLYA_ADAPTER          2   /* estimated adapter length > 300 nt */
#define NPH_POLYA_SUFFCLIP         3   /* suffix_clip > 200 */
#define NPH_POLYA_READ_FAILED_LOAD 4
typedef struct {
    uint64_t sample_off;      /* first raw sample (picoamps, float) of the read in raw[] */
    uint64_t event_off;       /* first event duration of the read in ev_duration[] */
    uint64_t rank_off;        /* first base_to_event entry of the read in base_to_event[] */
    uint32_t n_samples;       /* SquiggleRead::samples.size() */
    uint32_t n_kmers;         /* base_to_event_map.size() = read_sequence.length() - k + 1 */
    uint32_t n_events;        /* events[0].size() */
    uint32_t suffix_clip;     /* bam_cigar_oplen of the record's last CIGAR operation */
    double   sample_rate;
    double   scale, shift, var;   /* scalings[0]; the HMM takes them as floats */
    uint32_t loaded;          /* 0: READ_FAILED_LOAD (the read is not in the index) */
    uint32_t reserved;
} nph_polya_job;
typedef struct {
    uint64_t start, leader, adapter, polya;   /* Segmentation: final sample index of START, LEADER, ADAPTER, POLYA/CLIFF */
    uint64_t cliffs;                          /* CLIFF samples on the path */
    double   read_rate;                       /* 1 / median per-k-mer duration (may be inf) */
    double   polya_length;                    /* max(0, duration * rate - 5) */
    int32_t  qc;                              /* NPH_POLYA_* */
    uint32_t reserved;
} nph_polya_result;
int nph_polya_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_polya_job* jobs, size_t n_jobs,
                    const float* ev_duration, size_t n_events_total, const nph_event_range* base_to_event, size_t n_ranks_total,
                    nph_polya_result* results_out);

/* ---- poly(I) / poly(A) tail detection (nanopolish detect-polyi) -------------------------------------------
 * Per read, what dpi_estimate_polya_for_single_read computes after loading (src/nanopolish_detect_polyi.cpp:1061-1095): the
 * segmentation, read rate, length and QC of nph_polya_batch with DPISegmentationHMM (:177-518, whose POLYA emission is an even
 * mixture of two Gaussians, :291-295), then BernoulliHMM::segmentation over the tail's samples [adapter + 1, polya) (:728-756)
 * and post_boolhmm_detetection_qc (:973-997).  Same jobs, inputs and refusals as nph_polya_batch, plus NPH_ERR_INVALID for a
 * loaded job with n_samples >= 2^31: the reference passes the tail's bounds as int and would read before the samples.
 * A READ_FAILED_LOAD result has seg as nph_polya_batch gives it and -1 in polyi_last, polya_first and detected. */
#define NPH_POLYI_NONE       0   /* "NONE" */
#define NPH_POLYI_POLYA_ONLY 1   /* "POLYA-ONLY": polya_first > 0 and tail samples - polya_first > 200 */
#define NPH_POLYI_POLYI_ONLY 2   /* "POLYI-ONLY": polyi_last > 200 */
#define NPH_POLYI_A_PLUS_I   3   /* "A+I": both */
typedef struct {
    nph_polya_result seg;     /* as nph_polya_batch, under DPISegmentationHMM; seg.qc is the row's qc_tag */
    int32_t  polyi_last;      /* BernoulliSegmentation::polyi: last poly(I) index in the tail, or -1 */
    int32_t  polya_first;     /* BernoulliSegmentation::polya: first poly(A) index in the tail, or -1 */
    int32_t  detected;        /* NPH_POLYI_*, the row's detected column */
    uint32_t reserved;
} nph_polyi_result;
int nph_detect_polyi_batch(nph_ctx* ctx, const float* raw, size_t n_samples_total, const nph_polya_job* jobs, size_t n_jobs,
                           const float* ev_duration, size_t n_events_total, const nph_event_range* base_to_event,
                           size_t n_ranks_total, nph_polyi_result* results_out);

/* ---- phase-reads: SNP allele calls and qualities (ref: phase_single_read, src/nanopolish_phase_reads.cpp:178-347) -----------
 * One record = one BAM record, strand 0 of its read, in the compact event alignment of nph_methylation_batch_compact: ref_bases
 * holds the record's fetched reference, upper-cased (std::toupper) and NOT disambiguated; model_id is the read's base model (a
 * nucleotide model); strand stays 0.  variants is the caller's list sorted by position (sortByPosition), and var_range[2r],
 * var_range[2r + 1] the [lower_bound(pos), upper_bound(bam_endpos)) range of record r in it.
 * Per variant of a range, in list order: skipped unless is_snp; the window [p - 30, p + 30] (opt::min_flanking_sequence) must be
 * bounded by AlignmentDB::_find_by_ref_bounds (the reference's event/bp ratio test never skips); the centre base must equal
 * ref_base (Haplotype::apply_variant).  Such a site gets two forward scores (the 61-base reference window and the window with
 * alt_base at its centre; HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, the record's EventAlignmentRecord::stride) and one
 * nph_phase_call.  The calls of record r are calls_out[call_off_out[r] .. call_off_out[r + 1]) in list order.
 * NPH_ERR_INVALID: a record, model or variant range out of bounds (lo > hi included); a model that is not a nucleotide model;
 * calls_cap too small (nph_last_error states the count needed; the sum of hi - lo always suffices); a job the scorer refuses.
 * n_scored_events_out (optional): sum over sites of 2 * (abs(e2 - e1) + 1). */
#define NPH_PHASE_FLANK 30
typedef struct {
    int32_t  ref_position;    /* Variant::ref_position */
    char     ref_base;        /* ref_seq[0] */
    char     alt_base;        /* alt_seq[0] */
    uint8_t  is_snp;          /* Variant::is_snp(): both alleles one base long */
    uint8_t  reserved;
} nph_phase_variant;          /* 8 bytes */
typedef struct {
    uint32_t record;          /* index into records[] */
    uint32_t variant;         /* index into variants[] */
    float    ref_score;       /* profile_hmm_score of the reference window */
    float    alt_score;       /* of the window with the alternative base */
    char     call;            /* alt_base if alt_score > ref_score, else ref_base */
    uint8_t  qual;            /* q_char: (int)min(30, -10 log10 p_wrong) + 33, the byte the reference stores in the record's QUAL */
    uint8_t  reserved[2];
} nph_phase_call;             /* 20 bytes */
int nph_phase_reads_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                          const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                          const char* ref_bases, const int16_t* event_deltas, size_t n_ref_total, const int32_t* first_event,
                          const nph_meth_record* records, size_t n_records,
                          const nph_phase_variant* variants, size_t n_variants, const uint32_t* var_range,
                          double indel_bias, uint64_t* call_off_out,
                          nph_phase_call* calls_out, size_t calls_cap, uint64_t* n_scored_events_out);

/* ---- variants --fix-homopolymers: the length likelihoods of every homopolymer of a haplotype (ref: fix_homopolymers,
 * src/nanopolish_call_variants.cpp:541-780) ------------------------------------------------------------------------------
 * The reference scans the haplotype for runs of 3..9 equal bases and, per run that passes its skip tests, scores every candidate
 * length L = 3..9 against the run's event sequences.  The scan, the calling range (Haplotype::
 * get_enclosing_reference_range_for_haplotype_range, substr_by_reference), the call and its application stay with the caller;
 * this call takes one nph_hp_window per surviving run and returns the two likelihood vectors the reference builds for it:
 *   the window's event sequences  AlignmentDB::get_event_subsequences over [ref_calling_start, ref_calling_end] (the records of
 *                                 nph_screen_edits_batch, in record order: bounded by _find_by_ref_bounds, event/bp ratio below 20);
 *                                 total_reads counts them (the TotalReads INFO value)
 *   per sequence, in record order, skipped when abs(e_start - e_stop) < 10 (scored_reads counts the rest):
 *     local_avg = fabs(get_time(e_start) - get_time(e_stop)) / seq_len, get_time(e) = float(start_time[e] - start_time[0]);
 *     rate = (1 / local_avg) * 2.461964
 *     per L: the variant sequence = the calling sequence with the run erased to, or extended to, L bases at edit_offset;
 *       event_lik[L - 3]    += profile_hmm_score(variant, sequence, 0)                    (K1)
 *       sum_duration         = sum over k-mer slots k0 + 2 .. k0 + L + 1, ascending, of each slot's durations: the float
 *                              ev_duration of every non-K state of profile_hmm_align(variant, sequence, 0) (K3) on that k-mer,
 *                              added in double in path order (DurationModel::generate_aligned_durations)
 *       duration_lik[L - 3] += sum_duration > 0.00025 ? log_gamma_sum(sum_duration, {2.461964, rate}, L) : 0
 * all in double with the reference's operation order; the log-gamma terms run on the host with its libm (DESIGN.md).
 * Records: nph_meth_record in the compact form of nph_screen_edits_batch, model_id a nucleotide 6-mer model.  The reads must be
 * PORETYPE_R9 reads: the reference adds the duration term only for those, and this call always adds it.
 * ref_bases: the region's reference, ref_bases[p] = base at region_start + p (AlignmentDB's m_region_start .. m_region_end).
 * NPH_ERR_INVALID: a window with k != 6 (the reference asserts), hp_length outside 3..9, a calling sequence outside calling_seqs,
 * edit_offset + hp_length past the calling sequence (the reference throws or reads out of bounds), k0 + hp_length + k + 1 past
 * it (slot k0 + L + 1 would index past the variant sequence's k-mers), a calling range outside the region;
 * min_flanking_sequence < 7; a record or model out of bounds or not a nucleotide 6-mer model; a job the forward scorer refuses;
 * a job profile_hmm_align finds no path for (the reference asserts).  NPH_ERR_UNSUPPORTED: a window so long that one CTA's
 * Viterbi movement trace would exceed 16 GiB (the limit of nph_hmm_align).  The Viterbi states of the jobs are held in consecutive
 * chunks of (window, read) pairs under 1 GiB of device memory, (E_max + K_max) x 16 bytes per job. */
#define NPH_HP_MIN_LENGTH 3
#define NPH_HP_MAX_LENGTH 9
#define NPH_HP_LENGTHS 7
typedef struct {
    int32_t  region_start;            /* AlignmentDB::m_region_start */
    int32_t  min_flanking_sequence;   /* opt::min_flanking_sequence (30); the caller's scan used it, checked >= 7 */
    uint32_t max_chunk_pairs;         /* (window, read) pairs per chunk of Viterbi states: 0 = as many as fit the 1 GiB budget */
    uint32_t reserved;
} nph_hp_params;                      /* 16 bytes */
typedef struct {
    uint64_t seq_off;                 /* first byte of the calling sequence in calling_seqs[] */
    uint32_t seq_len;                 /* calling_sequence.size() */
    int32_t  ref_calling_start;       /* the enclosing reference range of the calling window */
    int32_t  ref_calling_end;
    uint32_t edit_offset;             /* hap_hp_start - hap_calling_start (after the enclosing range moved hap_calling_start) */
    uint32_t k0;                      /* hap_hp_start - hap_calling_start - k + 1 */
    uint32_t hp_length;               /* 3..9 */
    char     hp_base;
    uint8_t  reserved[3];
    uint32_t k;                       /* the reads' base-model k: 6 */
} nph_hp_window;                      /* 40 bytes */
typedef struct {
    uint32_t total_reads;             /* event sequences of the window (TotalReads) */
    uint32_t scored_reads;            /* of those, the ones with abs(e_start - e_stop) >= 10 */
    double   event_lik[NPH_HP_LENGTHS];     /* event_likelihoods[L], L = 3..9 */
    double   duration_lik[NPH_HP_LENGTHS];  /* duration_likelihoods[L] */
} nph_hp_likelihoods;                 /* 120 bytes */
typedef struct {
    uint64_t n_windows, n_pairs;      /* windows; scored (window, read) pairs */
    uint64_t n_jobs;                  /* 7 per pair, each one forward and one Viterbi fill */
    uint64_t n_dp_rows;               /* event rows of both fills over all jobs */
    uint32_t n_chunks;                /* chunks of Viterbi states */
    uint32_t reserved;
    double   host_ms;                 /* the host's log-gamma terms and fold.  nph_last_kernel_ms after the call: the forward kernels,
                                         the state-offset kernel, K3 and the duration kernel of every chunk (not the pair, scan, emit
                                         or scheduling kernels) */
} nph_hp_counts;                      /* 48 bytes */
int nph_homopolymer_likelihoods_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                      const float* ev_mean, const double* ev_start_time, const float* ev_duration, size_t n_events_total,
                                      const char* ref_bases, size_t n_ref_bases,
                                      const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                      const nph_meth_record* records, size_t n_records,
                                      const nph_hp_params* params, const char* calling_seqs, size_t n_seq_bytes,
                                      const nph_hp_window* windows, size_t n_windows, double indel_bias,
                                      nph_hp_likelihoods* out, nph_hp_counts* counts_out);

/* ---- variants --calculate-all-support: the A/C/G/T read support of every called variant (ref: annotate_variants_with_all_support,
 * src/common/nanopolish_variant.cpp:801-859) -------------------------------------------------------------------------------------
 * Per variant, in input order and each on its own:
 *   the window                    calling_start = ref_position - flank, calling_end = ref_position + flank: the 2 * flank + 1 bases
 *                                 ref_bases[calling_start - region_start ..] (substr_by_reference of the unedited region)
 *   four haplotypes, b in "ACGT"  apply_variant of {ref_seq, alt_seq = b} on a fresh window: it applies when window.substr(flank,
 *                                 ref_seq_len) == ref_seq byte for byte (substr clamps, so a ref_seq longer than flank + 1 bases never
 *                                 applies), and then ref_seq is replaced by b; otherwise the haplotype is the window.  `applied`
 *                                 reports the outcome (it does not depend on b)
 *   the window's event sequences  AlignmentDB::get_event_subsequences over [calling_start, calling_end] (the records of
 *                                 nph_screen_edits_batch, in record order: bounded by _find_by_ref_bounds, event/bp ratio below 20);
 *                                 n_reads counts them
 *   per sequence, in record order s[hi] = profile_hmm_score(haplotype hi, sequence, alignment_flags) (K1), a float;
 *                                 sum = s[0], then sum = add_logs(s[hi], sum) for hi = 1..3 (p7_FLogsum on floats);
 *                                 support[hi] += exp(double(s[hi]) - double(sum)), in double
 *   support[hi] /= n_reads        (0 / 0 with no sequence: a NaN, which the reference prints as -nan)
 * K1 and the log-sum run on the device, exp, the sum over sequences and the division on the host with its libm (DESIGN.md).
 * Records: nph_meth_record in the compact form of nph_screen_edits_batch, model_id a nucleotide model of k = params->k.
 * ref_bases: the region's reference, ref_bases[p] = base at region_start + p (AlignmentDB's m_region_start .. m_region_end).
 * NPH_ERR_INVALID: k outside 1..8; flank + 1 < k (a haplotype without a k-mer); alignment_flags other than NPH_HAF_*; a ref_seq
 * outside ref_seqs; a window outside the region (substr_by_reference asserts: calling_start < region_start or calling_end >
 * region_end); a record or model out of bounds or not a nucleotide model of k; a job the forward scorer refuses.  The contig test
 * of get_event_subsequences (a variant on another contig asserts) is the caller's. */
typedef struct {
    int32_t  region_start;            /* AlignmentDB::m_region_start */
    int32_t  flank;                   /* min_flanking_sequence (variants: 30) */
    uint32_t alignment_flags;         /* NPH_HAF_* (variants: NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP) */
    uint32_t k;                       /* the reads' base-model k */
} nph_support_params;                 /* 16 bytes */
typedef struct {
    int32_t  ref_position;            /* Variant::ref_position */
    uint32_t ref_seq_len;             /* ref_seq.size() */
    uint64_t ref_seq_off;             /* first byte of ref_seq in ref_seqs[] */
} nph_support_variant;                /* 16 bytes */
typedef struct {
    double   support[4];              /* SupportFractionByBase for A, C, G, T */
    uint32_t n_reads;                 /* event sequences of the window (the divisor) */
    uint32_t applied;                 /* 1: apply_variant replaced ref_seq; 0: the four haplotypes are the window */
} nph_support_result;                 /* 40 bytes */
typedef struct {
    uint64_t n_variants, n_pairs;     /* variants; (variant, event sequence) pairs */
    uint64_t n_jobs;                  /* 4 per pair, one forward fill each */
    uint64_t n_dp_rows;               /* event rows over all jobs */
    double   host_ms;                 /* the host's exp, sums and divisions.  nph_last_kernel_ms after the call: the forward kernels
                                         (not the pair, scan, emit, scheduling or log-sum kernels) */
} nph_support_counts;                 /* 40 bytes */
int nph_all_support_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                          const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                          const char* ref_bases, size_t n_ref_bases,
                          const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                          const nph_meth_record* records, size_t n_records,
                          const nph_support_params* params, const char* ref_seqs, size_t n_seq_bytes,
                          const nph_support_variant* variants, size_t n_variants, double indel_bias,
                          nph_support_result* out, nph_support_counts* counts_out);

/* ---- variants: screen_variants_by_score on a candidate list (ref: src/nanopolish_call_variants.cpp:364-402) ------------------
 * Each candidate of the list on its own, in input order (the reference's semantics on one OpenMP thread):
 *   the window        calling_start = ref_position - flank, calling_end = ref_position + ref_seq_len + flank, narrowed to int; a
 *                     window with calling_start < region_start or calling_end > region_end is skipped (are_coordinates_valid):
 *                     status NPH_SCREEN_OUTSIDE, quality NaN.  The base haplotype is the ref_seq_len + 2 * flank + 1 bases
 *                     ref_bases[calling_start - region_start ..]
 *   the variant       apply_variant on a fresh window: when window[flank, flank + ref_seq_len) == ref_seq byte for byte
 *                     (case-sensitive; an empty ref_seq always matches) ref_seq is replaced by alt_seq.  Otherwise the haplotype is
 *                     the window and the quality is exactly 0.0: status NPH_SCREEN_NOT_APPLIED, nothing is scored
 *   the reads         get_event_subsequences(calling_start, calling_end): the records of nph_screen_edits_batch in record order,
 *                     bounded by _find_by_ref_bounds, event/bp ratio below 20
 *   the quality       total = 0.0, then per read: if (fabs(total) < score_threshold) total += set(variant) - set(base), each side
 *                     profile_hmm_score_set over the sequence and its -q alternatives (as nph_screen_load_methylation forms them)
 * screen_variants_by_score keeps the candidates whose quality is > 0.
 * Candidates with the same window (calling_start and ref_seq_len) share their reads and their base scores: the device scores the
 * base set once per (window, read) for all the window's candidates still inside the threshold, reads_per_round reads at a time.
 * Records: nph_meth_record in the compact form of nph_screen_edits_batch, model_id a nucleotide model of k = params->k.
 * meth (NULL: no types) and alt_model_ids: as nph_screen_load_methylation takes them, with exactly its checks.
 * NPH_ERR_INVALID: k outside 1..8; 2 * flank + 1 < k; reads_per_round == 0; alignment_flags other than NPH_HAF_*; an allele outside
 * alleles; ref_position + ref_seq_len + flank > INT32_MAX; a record or model out of range or not a nucleotide model of k; a job the
 * forward scorer refuses. */
#define NPH_SCREEN_SCREENED    0u     /* scored: quality = the thresholded total */
#define NPH_SCREEN_OUTSIDE     1u     /* the window leaves the region: the reference skips the candidate (quality NaN) */
#define NPH_SCREEN_NOT_APPLIED 2u     /* ref_seq is not the window's: the variant haplotype is the base, quality 0.0 */
typedef struct {
    int32_t  region_start;            /* AlignmentDB::m_region_start */
    int32_t  flank;                   /* opt::screen_flanking_sequence (10) */
    uint32_t score_threshold;         /* opt::screen_score_threshold (100; --faster: 25) */
    uint32_t alignment_flags;         /* NPH_HAF_* */
    uint32_t k;                       /* the reads' base-model k */
    uint32_t reads_per_round;         /* reads of a window scored between two early-exit tests (8) */
} nph_screen_list_params;             /* 24 bytes */
typedef struct {
    int64_t  ref_position;            /* Variant::ref_position (>= 0) */
    uint32_t ref_seq_len, alt_seq_len;
    uint64_t ref_seq_off, alt_seq_off;   /* first byte of each allele in alleles[] */
} nph_screen_candidate;               /* 32 bytes */
typedef struct {
    double   quality;                 /* Variant::quality after score_variant_thresholded (NaN: NPH_SCREEN_OUTSIDE) */
    uint32_t n_reads;                 /* event sequences of the window */
    uint32_t status;                  /* NPH_SCREEN_SCREENED, _OUTSIDE or _NOT_APPLIED */
} nph_screen_result;                  /* 16 bytes */
typedef struct {
    uint64_t n_candidates, n_windows; /* candidates; distinct windows among those inside the region */
    uint64_t n_rounds;                /* early-exit rounds */
    uint64_t n_jobs, n_dp_rows;       /* forward jobs run and their event rows */
    uint64_t n_jobs_without_exit;     /* jobs every read of every applied candidate would take: per window reads x (n(base) + sum n(c)) */
    uint64_t n_reference_rows;        /* the reference's DP rows: (n(base) + n(variant)) x E per (candidate, read) until its exit,
                                         n(s) = 1 + alternatives of s; candidates that do not apply count too (the reference scores them) */
    double   kernel_ms;               /* device time of the forward kernels of every round (not the pair, rank, emit or accumulate kernels) */
} nph_screen_list_counts;             /* 64 bytes */
int nph_screen_variants_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                              const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                              const char* ref_bases, size_t n_ref_bases,
                              const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                              const nph_meth_record* records, size_t n_records,
                              const nph_screen_list_params* params, const char* alleles, size_t n_allele_bytes,
                              const nph_screen_candidate* candidates, size_t n_candidates, double indel_bias,
                              const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                              nph_screen_result* out, nph_screen_list_counts* counts_out);

/* ---- variants: the haplotype scores and genotype choice of call_haplotype_from_candidates ------------------------------------
 * (ref: src/nanopolish_call_variants.cpp:782-880, score_variant_group and simple_call of src/common/nanopolish_variant.cpp:182-493)
 * The caller groups the candidates and builds each group's haplotypes: combination c of group g is haplotype hap_first + c, its
 * bases haplotype_bases[seq_off, seq_off + seq_len) and its variant ids (group-local, < n_variants) combination_variants[var_off, ..).
 * Combination 0 is the empty one (the base haplotype); every other combination names at least one variant.  Per group, on one OpenMP
 * thread's semantics:
 *   the reads     get_event_subsequences(calling_start, calling_end) in record order, as nph_screen_variants_batch walks them
 *   the keys      VariantGroup keys a read by "read_name:strand".  key_rank[read] is the rank of that string among the call's reads
 *                 (equal strings, equal ranks): a group's keys are its distinct ranks, ascending.  Per key, s[c][key] is the score
 *                 of its last record, read_sum[key] the add_logs chain over (record, combination) in order, is_rc the last record's
 *   the scores    s = profile_hmm_score_set(generate_methylated_alternatives(haplotype, -q types), record, alignment_flags), a float
 *   the sets      the multisets of ploidy combination ids in Combinations(n, ploidy, CO_WITH_REPLACEMENT) order (non-decreasing
 *                 tuples, lexicographic); set_score = sum over keys of add_logs(..., s - log(2)) chained from -inf; best = the first
 *                 set whose score exceeds the best so far (from -inf), base = set 0.  best - base < 20 keeps the base set
 *   per variant   the posterior exp(s - read_sum) summed per (key, variant) and per variant in simple_call's loop order, the strand
 *                 sums (1 - pp, pp) and the variant's count in the best set
 * The device runs the walk, K1, the key fold and the genotype search; exp and the sums run on the host with its libm (host_ms).
 * Records, meth and alt_model_ids: as nph_screen_variants_batch takes them.  NPH_ERR_INVALID: k outside 1..8; ploidy outside
 * 1..NPH_CALL_MAX_PLOIDY; alignment_flags other than NPH_HAF_*; a group with fewer than 2 haplotypes or fewer than ploidy (the
 * reference's Combinations asserts), a window outside the region or
 * calling_start > calling_end, a haplotype or variant range outside its array; a haplotype with fewer than k bases, its bases or
 * variant ids outside their arrays, a variant id >= the group's n_variants, a non-empty combination 0 or an empty later one; more
 * than 2^60 genotype sets in a group; a record, model or -q type the screening calls refuse; a job the forward scorer refuses. */
#define NPH_CALL_MAX_PLOIDY 8
#define NPH_CALL_CALLED    0u         /* best - base >= 20 (or a NaN difference): the best set stands */
#define NPH_CALL_BASE_KEPT 1u         /* best - base < 20: the base set is the call */
#define NPH_CALL_NO_BEST   2u         /* no set scored above -inf: no best set, every count is 0 */
typedef struct {
    int32_t  region_start;            /* AlignmentDB::m_region_start */
    uint32_t ploidy;                  /* opt::ploidy */
    uint32_t genotype_all;            /* opt::genotype_only: emit every variant, not only those with var_count > 0 */
    uint32_t alignment_flags;         /* NPH_HAF_* (variants: NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP) */
    uint32_t k;                       /* the reads' base-model k */
} nph_call_params;                    /* 20 bytes */
typedef struct {
    int32_t  calling_start, calling_end;   /* the group's window in reference coordinates */
    uint32_t hap_first, n_haplotypes;      /* haplotypes [hap_first, hap_first + n_haplotypes): one per combination */
    uint32_t var_first, n_variants;        /* results of variants [var_first, var_first + n_variants) go to variants_out */
} nph_call_group;                     /* 24 bytes */
typedef struct {
    uint64_t seq_off;                 /* first base in haplotype_bases[] */
    uint32_t seq_len;                 /* bases */
    uint32_t n_var;                   /* variant ids of its combination */
    uint64_t var_off;                 /* first id in combination_variants[] */
} nph_call_haplotype;                 /* 24 bytes */
typedef struct {
    uint32_t n_keys, n_combinations;  /* TotalReads; combinations (= n_haplotypes) */
    uint32_t status;                  /* NPH_CALL_* */
    uint32_t ploidy;                  /* entries of best_set written (0 with NPH_CALL_NO_BEST) */
    uint32_t best_set[NPH_CALL_MAX_PLOIDY];   /* the called set's combination ids (the base set's zeros after NPH_CALL_BASE_KEPT) */
    double   best_score, base_score;  /* the highest set score (-inf: none) and set 0's */
} nph_call_group_result;              /* 64 bytes */
typedef struct {
    uint32_t var_count;               /* AlleleCount: the variant's occurrences in the called set */
    uint32_t emit;                    /* genotype_all || var_count > 0: simple_call outputs it */
    double   support_sum;             /* read_variant_support: SupportFraction = support_sum / n_keys */
    double   strand[4];               /* ref_fwd, ref_rev, alt_fwd, alt_rev */
} nph_call_variant_result;            /* 48 bytes */
typedef struct {
    uint64_t n_groups, n_haplotypes;  /* groups; haplotypes over all groups */
    uint64_t n_pairs;                 /* (group, event sequence) pairs */
    uint64_t n_jobs, n_dp_rows;       /* forward jobs (one per pair, haplotype and alternative) and their event rows */
    uint64_t n_sets, n_set_terms;     /* genotype sets over all groups; sets x keys */
    double   forward_ms;              /* device time of the forward kernels */
    double   genotype_ms;             /* device time of the genotype kernels */
    double   host_ms;                 /* the host's exp and sums */
} nph_call_counts;                    /* 80 bytes */
int nph_call_variant_groups_batch(nph_ctx* ctx, const nph_read* reads, size_t n_reads,
                                  const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                  const char* ref_bases, size_t n_ref_bases,
                                  const int16_t* event_deltas, size_t n_deltas_total, const int32_t* first_event,
                                  const nph_meth_record* records, size_t n_records, const uint32_t* key_rank,
                                  const nph_call_params* params,
                                  const nph_call_group* groups, size_t n_groups,
                                  const nph_call_haplotype* haplotypes, size_t n_haplotypes,
                                  const char* haplotype_bases, size_t n_bases,
                                  const uint32_t* combination_variants, size_t n_combination_variants,
                                  size_t n_variants, double indel_bias,
                                  const nph_screen_methylation* meth, const uint32_t* alt_model_ids,
                                  nph_call_group_result* groups_out, nph_call_variant_result* variants_out,
                                  nph_call_counts* counts_out);

/* ---- variants: the basecall candidates of a region (AlignmentDB::get_variants_in_region) -------------------------------------
 * (ref: src/alignment/nanopolish_alignment_db.cpp:259-368)  The pile-up of the base-space alignments of a loaded region: every
 * mismatch or gap the reads show between reference positions start and stop, merged on (position, ref_seq, alt_seq), with its
 * instance count and the read depth at its position.  Per record, in record order, over aligned_bases (the record's
 * get_aligned_segments()[0]: (ref_pos, read_pos) pairs, both strictly increasing):
 *   the bounds    start_iter = lower_bound(start), stop_iter = lower_bound(stop) by ref_pos
 *   the depth     +1 over [max(start_iter->ref_pos, start), min(stop_iter == end ? back().ref_pos : stop_iter->ref_pos, stop)):
 *                 deleted reference bases count, the record's last aligned base does not
 *   the walk      from start_iter to stop_iter: is_gap = the next pair is not (ref + 1, read + 1) and is not stop_iter; on a gap,
 *                 next = the first later pair whose read base equals its reference base (byte compare), else stop_iter; without
 *                 one, next = the next pair.  (mismatch || gap) && next != stop_iter && next->ref_pos < stop - 1 is one instance:
 *                 ref_seq = region_ref[i.ref, next.ref), alt_seq = bases[i.read, next.read)
 * A record without a pair at or after start adds no depth and no instance (the reference dereferences end() there).
 * A record's alignment comes in the compact form of nph_methylation_batch_compact, read positions in place of event indices:
 * base_deltas[map_off + o] belongs to reference position ref_start_pos + o, NPH_METH_NO_PAIR where the record has no pair, else
 * its read position minus the previous pair's (first_read_pos for the first pair, whose own delta is then 0).  A read-position
 * step beyond int16 (an insertion of more than 32 767 bases) cannot be written in this form: the host mirror returns
 * NPH_ERR_UNSUPPORTED for it.
 * Out: one nph_region_candidate per distinct (ref_position, ref_seq, alt_seq), alt_seq = bases[alt_off, alt_off + alt_len) of one of
 * its instances; in ascending ref_position, otherwise in no documented order (the reference's std::map order and its filter are the
 * caller's: nph::get_variants_in_region).  count is exact; neither field depends on the order of the device's atomics.
 * out_cap too small: NPH_ERR_INVALID with *n_out set to the count needed.  NPH_ERR_INVALID also for stop < start (the reference
 * asserts), [start, stop] not inside [region_start, region_start + n_ref - 1], a record whose bases or alignment slice leave their
 * arrays, whose read positions leave its bases or do not strictly increase (a non-first delta below 1).
 * Counts: records, the pairs the walks visited, instances, distinct variants, and the device time of the call's kernels
 * (region_candidates.cu: cand_walk_kernel, cand_rep_kernel, cand_emit_kernel, the scans, the radix sort). */
typedef struct {
    uint64_t seq_off;                 /* first base of the record's read in bases[] (seq_nt16_str characters, '=' and 'N' included) */
    uint64_t map_off;                 /* first entry of its compact alignment in base_deltas[] */
    uint32_t seq_len;                 /* bases of the read */
    uint32_t map_len;                 /* reference positions its compact alignment covers (0: no pairs) */
    int32_t  ref_start_pos;           /* reference position of base_deltas[map_off] */
    int32_t  first_read_pos;          /* read position of the record's first pair */
} nph_seq_record;                     /* 32 bytes */
typedef struct {
    int32_t  ref_position;            /* Variant::ref_position */
    uint32_t ref_len;                 /* |ref_seq|: ref_seq = region_ref[ref_position - region_start, + ref_len) */
    uint32_t alt_len;                 /* |alt_seq| */
    uint32_t count;                   /* instances over all records */
    uint32_t depth;                   /* the depth at ref_position */
    uint32_t record;                  /* the record of the instance alt_off points into */
    uint64_t alt_off;                 /* alt_seq = bases[alt_off, alt_off + alt_len) */
} nph_region_candidate;               /* 32 bytes */
typedef struct {
    uint64_t n_records;               /* records of the call */
    uint64_t n_pairs;                 /* pairs in [start_iter, stop_iter) over all records */
    uint64_t n_instances;             /* mismatch or gap instances before the merge */
    uint64_t n_variants;              /* distinct variants */
    double   kernel_ms;               /* device time from the first kernel to the last (one read-back of the instance total between) */
} nph_candidate_counts;               /* 40 bytes */
int nph_region_candidates_batch(nph_ctx* ctx, const char* region_ref, size_t n_ref, int32_t region_start,
                                const char* bases, size_t n_bases, const int16_t* base_deltas, size_t n_deltas,
                                const nph_seq_record* records, size_t n_records, int32_t start, int32_t stop,
                                nph_region_candidate* out, size_t out_cap, uint64_t* n_out, nph_candidate_counts* counts_out);

/* ---- scorereads --train-transitions: forward scores and transition training counts of a job batch ----------------------------
 * `nanopolish scorereads --train-transitions` runs, for every segment model_score scores (src/nanopolish_scorereads.cpp:116-203),
 * profile_hmm_align(sequence, data) (K3, flags 0) after the forward score, and folds the path into
 * TransitionParameters::add_training_from_alignment (src/hmm/nanopolish_transition_parameters.cpp:294-368) of the segment's strand.
 * This call takes the batch of nph_hmm_score_batch_seq (reads, events, base codes, jobs) and returns both halves:
 *   scores_out[j]        == what nph_hmm_score_batch_seq gives for job j (K1, the same scheduler and kernels)
 *   counts_out[g]        the training counts of the jobs whose group (groups[j], NULL: all 0) is g, g < n_groups
 * Per job, over its path p of n states (nothing when n <= ignore_edge_length), prev_s = 'M', kmer_move = i == 0 ||
 * p[i-1].kmer_idx != p[i].kmer_idx:
 *   state_transitions[prev_s][2 * s + kmer_move] += 1 for every state, and once more for 5 < i < n - 5 (ignore_edge_length 5)
 *   in that interior, a state s != 'B' is one skip observation between k-mers from = p[i-1].kmer_idx and to = p[i].kmer_idx
 *   (to = from + 1 for 'K' after 'M'): the bin b = min(29, (size_t)(|l1 - l2| / 0.5)) of the two scaled means
 *   l = float(scale * level_mean[rank] + shift) (get_scaled_gaussian_from_pore_model_state) gets skip_total[b] += 1 and
 *   skip_count[b] += (s == 'K')
 *   n_matches += s == 'M', n_skips += s == 'K' (n_merges stays 0: an R9 path has no 'E' state)
 * Every count is an integer sum, so the records do not depend on the order the device visits the states in.  The reference counts
 * in uint32_t and this call in uint64_t: the two differ once a count passes 2^32.  TransitionParameters::train() needs, per bin,
 * exactly skip_count and skip_total (its observations add is_skip and 1 to the bin's doubles), so the records carry everything the
 * reference's observation vector does.
 * NPH_ERR_INVALID: a group >= n_groups, n_groups outside 1..256; a job nph_hmm_score_batch_seq refuses; and where the reference
 * asserts: a job profile_hmm_align finds no path for, a skip observation with to >= n_kmers, a state other than M, B, K; and a
 * skip observation whose scaled mean is not finite (the reference's bin is then undefined).  One more difference: the
 * reference's (size_t) of |l1 - l2| / 0.5 >= 2^64 (means beyond 2^62 pA) wraps to bin 0, this call clamps it to bin 29.
 * The Viterbi states stay on the device, in consecutive chunks of jobs under 1 GiB ((E_max + K_max) x 16 bytes per job), at most
 * max_chunk_jobs jobs each (0: no cap).  nph_last_kernel_ms after the call: the forward kernels, and K3, the state-offset kernel
 * and the observation kernel of every chunk (not the scheduler or the uploads); params->viterbi_ms_out and observe_ms_out split the
 * chunks' share. */
#define NPH_TT_BINS 30
#define NPH_TT_MAX_GROUPS 256
typedef struct {
    uint64_t state_transitions[3][6]; /* rows M, B, K (from); column 2 * to + kmer_move */
    uint64_t n_matches, n_merges, n_skips;
    uint64_t skip_total[NPH_TT_BINS]; /* skip observations per bin of |l1 - l2| (width 0.5, the last bin open) */
    uint64_t skip_count[NPH_TT_BINS]; /* of those, the ones whose state is 'K' */
} nph_transition_counts;              /* 648 bytes */
typedef struct {
    uint32_t n_groups;                /* counts records written: 2 (NUM_STRANDS) for scorereads */
    uint32_t ignore_edge_length;      /* add_training_from_alignment's default: 5 */
    uint32_t max_chunk_jobs;          /* jobs per chunk of Viterbi states: 0 = as many as fit the 1 GiB budget */
    uint32_t n_chunks_out;            /* written by the call: the chunks it ran */
    float    viterbi_ms_out;          /* written by the call: device ms of K3 and its state-offset kernel over all chunks */
    float    observe_ms_out;          /* written by the call: device ms of the observation kernel over all chunks */
} nph_tt_params;                      /* 24 bytes */
int nph_train_transitions_batch(nph_ctx* ctx,
                                const nph_read* reads, size_t n_reads,
                                const float* ev_mean, const double* ev_start_time, size_t n_events_total,
                                const uint8_t* seq_codes, size_t n_codes_total,
                                const nph_hmm_job* jobs, size_t n_jobs, const uint8_t* groups,
                                nph_tt_params* params, double indel_bias,
                                float* scores_out, nph_transition_counts* counts_out);

/* ---- measurement hooks (used by bench.py; not part of the reference surface) ------------- */
/* Device time in ms of the most recent nph_hmm_score / nph_abea_run kernel sequence, measured
 * with CUDA events on the context's stream (valid after a sync), and the number of kernel
 * launches it issued. */
int nph_last_kernel_ms(nph_ctx* ctx, float* ms_out, int* launches_out);
/* Pinned host memory helpers so callers can stage H2D/D2H at full PCIe speed. */
int nph_host_alloc(void** ptr_out, size_t bytes);
int nph_host_free(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* NPH_H */
