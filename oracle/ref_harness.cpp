// oracle/ref_harness.cpp — TEST INFRASTRUCTURE ONLY.
//
// A thin C-callable shell around the UNMODIFIED reference translation units of the
// hot path (compiled in place from /root/reference by oracle/Makefile into
// oracle/_ref/libnpref.so).  It lets tests/ and bench.py's cpu_baseline leg drive
//   profile_hmm_score                      (src/hmm/nanopolish_profile_hmm.cpp:23-30)
//   adaptive_banded_simple_event_align     (src/nanopolish_raw_loader.cpp:77-379)
//   estimate_scalings_using_mom            (src/nanopolish_raw_loader.cpp:17-60)
//   HMMInputSequence::get_kmer_rank        (src/hmm/nanopolish_hmm_input_sequence.h:76-91)
//   Alphabet::{reverse_complement,methylate,unmethylate,disambiguate}
// and (via --gc-sections, see oracle/Makefile) eventalign's align_read_to_ref + TSV writer, create_modbam_record,
// score_variant_thresholded and SquiggleRead's small members, on flat arrays.  Reads are assembled by hand exactly like the reference's own
// "scalings" unit test does (src/test/nanopolish_test.cpp:279-311): default-construct a
// SquiggleRead, set pore_type / base_model / scalings / events_per_base, push events.
//
// The product (nanopolish_b200/, include/) never links or loads this file.
#include <cstdint>
#include <cstring>
#include <cmath>
#include <limits>
#include <memory>
#include <sstream>
#include <string>
#include <vector>
#include <chrono>
#include <omp.h>

#include "nanopolish_common.h"
#include "nanopolish_squiggle_read.h"
#include "nanopolish_pore_model_set.h"
#include "nanopolish_profile_hmm.h"
#include "nanopolish_raw_loader.h"
#include "nanopolish_alphabet.h"
#include "nanopolish_emissions.h"
#include "logsum.h"
#include "nanopolish_eventalign.h"   // align_read_to_ref / emit_event_alignment_tsv (8f N1: segment chaining)
#include "nanopolish_anchor.h"
#include "nanopolish_basemods.h"     // create_modbam_record (the Mm / Ml tags of call-methylation --modbam-output)
#include "nanopolish_variant.h"      // score_variant_thresholded (8f N2)
#include "nanopolish_haplotype.h"
#include "nanopolish_variant_db.h"   // VariantGroup / Combinations (score_variant_group, 8f N2)
#include "nanopolish_methyltrain.h"  // recalibrate_model (8f N4: the calibration after ABEA); its Eigen solve comes from oracle/shim/Eigen/Dense
extern "C" {
#include "event_detection.h"   // src/thirdparty/scrappie (C99)
}
#include "ref_harness.h"

extern double hmm_indel_bias_factor;   // src/hmm/nanopolish_profile_hmm_r9.cpp:19

// nanopolish_squiggle_read.cpp itself is compiled in place and linked with --gc-sections (oracle/Makefile): its small
// members (SquiggleScalings::set4/set6, the destructor, get_closest_event_to, get_event_sample_idx,
// get_scaled_samples_for_event) are the reference's own; load_from_raw and the constructor that need HDF5, Eigen and the
// read databases are never referenced and are dropped by the linker.

// htslib is not built here; eventalign needs two of its calls.  Test doubles: the "FASTA index" is a contig held
// in memory, bam_endpos is pos + reference length of the CIGAR (what htslib computes for a mapped record).
extern "C" char* faidx_fetch_seq(const faidx_t* fai, const char* c_name, int p_beg_i, int p_end_i, int* len)
{
    const NprefContig* c = reinterpret_cast<const NprefContig*>(fai);
    if(c->name != c_name) { *len = -2; return NULL; }
    if(p_beg_i < 0) p_beg_i = 0;
    if(p_end_i >= (int)c->seq.size()) p_end_i = (int)c->seq.size() - 1;     // faidx clips to the contig, end inclusive
    int l = p_end_i >= p_beg_i ? p_end_i - p_beg_i + 1 : 0;
    char* out = (char*)malloc(l + 1);
    memcpy(out, c->seq.data() + p_beg_i, l);
    out[l] = 0;
    *len = l;
    return out;
}
extern "C" hts_pos_t bam_endpos(const bam1_t* b)
{
    hts_pos_t rlen = 0;
    const uint32_t* cigar = bam_get_cigar(b);
    for(uint32_t i = 0; i < b->core.n_cigar; ++i)
        if(bam_cigar_type(bam_cigar_op(cigar[i])) & 2) rlen += bam_cigar_oplen(cigar[i]);
    return b->core.pos + (rlen ? rlen : 1);
}
// Three more htslib calls, reached from create_modbam_record / SequenceAlignmentRecord: the 4-bit base table, a record
// copy, and the two aux-tag writers, which here just keep what the reference hands them.
extern "C" const char seq_nt16_str[] = "=ACMGRSVTWYHKDBN";
namespace { thread_local std::string g_mm_tag; thread_local std::vector<uint8_t> g_ml_tag; }
extern "C" bam1_t* bam_dup1(const bam1_t* b)
{
    bam1_t* c = (bam1_t*)calloc(1, sizeof(bam1_t));
    *c = *b;
    c->data = (uint8_t*)malloc(b->l_data > 0 ? b->l_data : 1);
    memcpy(c->data, b->data, b->l_data);
    c->m_data = b->l_data;
    return c;
}
extern "C" int bam_aux_update_str(bam1_t*, const char tag[2], int len, const char* data)
{
    if(tag[0] == 'M' && tag[1] == 'm') g_mm_tag.assign(data, len > 0 ? len - 1 : 0);
    return 0;
}
extern "C" int bam_aux_update_array(bam1_t*, const char tag[2], uint8_t type, uint32_t items, void* data)
{
    if(tag[0] == 'M' && tag[1] == 'l' && type == 'C') g_ml_tag.assign((uint8_t*)data, (uint8_t*)data + items);
    return 0;
}
// summarize_alignment (nanopolish_eventalign.cpp:486-537) returns a struct that the reference defines inside its .cpp
// (:131-153); the declaration below mirrors that layout so the function can be called.  It reads the record's NM tag
// through two more htslib calls, answered here with "no tag" / 0.
struct EventalignSummary {
    int num_events, num_steps, num_stays, num_skips;
    double sum_duration, sum_z_score;
    int alignment_edit_distance, reference_span;
};
EventalignSummary summarize_alignment(const SquiggleRead& sr, uint32_t strand_idx, const EventAlignmentParameters& params,
                                      const std::vector<EventAlignment>& alignments);
extern "C" uint8_t* bam_aux_get(const bam1_t*, const char[2]) { return NULL; }
extern "C" int64_t bam_aux2i(const uint8_t*) { return 0; }
std::vector<uint32_t> event_alignment_to_cigar(const std::vector<EventAlignment>& alignments);   // nanopolish_eventalign.cpp:256
void write_methylation_results_as_tsv(FILE* site_writer, const bam1_t* record, std::map<int, ScoredSite>& site_score_map);   // nanopolish_call_methylation.cpp:532
std::string cigar_ops_to_string(const std::vector<uint32_t>& ops);                                 // :246

namespace {
std::vector<const PoreModel*> g_models;
std::vector<std::unique_ptr<PoreModel>> g_owned_models;
std::vector<std::unique_ptr<SquiggleRead>> g_reads;
}

SquiggleRead* npref_read_of(int h) { return g_reads[h].get(); }

extern "C" {

int npref_model_builtin(const char* kit, const char* alphabet, const char* strand, int k)
{
    if(!PoreModelSet::has_model(kit, alphabet, strand, k)) return -1;
    const PoreModel* pm = PoreModelSet::get_model(kit, alphabet, strand, k);
    if(pm == NULL) return -1;
    g_models.push_back(pm);
    return (int)g_models.size() - 1;
}

// A hand-made model: level_log_stdv = log(level_stdv) as PoreModelStateParams::update_logs does
// (src/pore_model/nanopolish_poremodel.h:61-65).
int npref_model_custom(const char* alphabet, int k, uint32_t n_states, const double* mean, const double* stdv)
{
    std::unique_ptr<PoreModel> pm(new PoreModel(k));
    pm->pmalphabet = get_alphabet_by_name(alphabet);
    pm->states.resize(n_states);
    for(uint32_t i = 0; i < n_states; ++i)
        pm->states[i] = PoreModelStateParams(mean[i], stdv[i], 1.0, 1.0);
    g_models.push_back(pm.get());
    g_owned_models.push_back(std::move(pm));
    return (int)g_models.size() - 1;
}

int npref_model_info(int h, uint32_t* k, uint32_t* n_states, uint32_t* alphabet_size)
{
    const PoreModel* pm = g_models[h];
    *k = pm->k; *n_states = pm->states.size(); *alphabet_size = pm->pmalphabet->size();
    return 0;
}

int npref_model_dump(int h, double* mean, double* stdv, double* log_stdv)
{
    const PoreModel* pm = g_models[h];
    for(size_t i = 0; i < pm->states.size(); ++i) {
        mean[i] = pm->states[i].level_mean;
        stdv[i] = pm->states[i].level_stdv;
        log_stdv[i] = pm->states[i].level_log_stdv;
    }
    return 0;
}

int npref_read_create(uint32_t n_events, const float* mean, const double* start_time,
                      double shift, double scale, double drift, double var,
                      double events_per_base, int base_model)
{
    std::unique_ptr<SquiggleRead> sr(new SquiggleRead());
    sr->pore_type = PORETYPE_R9;
    sr->read_type = SRT_TEMPLATE;
    sr->nucleotide_type = SRNT_DNA;
    sr->base_model[0] = g_models[base_model];
    sr->base_model[1] = NULL;
    sr->scalings[0].set4(shift, scale, drift, var);
    sr->events_per_base[0] = events_per_base;
    sr->events[0].resize(n_events);
    for(uint32_t i = 0; i < n_events; ++i) {
        SquiggleEvent& e = sr->events[0][i];
        e.mean = mean[i];
        e.stdv = 1.0f;
        e.start_time = start_time[i];
        e.duration = 0.0f;
        e.log_stdv = 0.0f;
    }
    g_reads.push_back(std::move(sr));
    return (int)g_reads.size() - 1;
}

void npref_read_set_scalings(int h, double shift, double scale, double drift, double var, double events_per_base)
{
    g_reads[h]->scalings[0].set4(shift, scale, drift, var);
    g_reads[h]->events_per_base[0] = events_per_base;
}

void npref_reads_clear(void) { g_reads.clear(); }

// profile_hmm_score over a batch of jobs; OpenMP over jobs the way the reference parallelises
// over reads (src/common/nanopolish_bam_processor.cpp:99).  Returns elapsed seconds of the scoring loop.
double npref_score_batch(size_t n_jobs, const int32_t* read_h, const int32_t* model_h,
                         const uint32_t* e_start, const uint32_t* e_stop, const uint8_t* rc,
                         const uint32_t* flags, const char* seq_buf, const uint64_t* seq_off,
                         double indel_bias, int threads, float* out)
{
    hmm_indel_bias_factor = indel_bias;
    if(threads < 1) threads = 1;
    auto t0 = std::chrono::steady_clock::now();
    #pragma omp parallel for schedule(dynamic) num_threads(threads)
    for(size_t j = 0; j < n_jobs; ++j) {
        const PoreModel* pm = g_models[model_h[j]];
        std::string seq(seq_buf + seq_off[j], seq_buf + seq_off[j + 1]);
        HMMInputSequence hseq(seq, pm->pmalphabet);
        HMMInputData data;
        data.read = g_reads[read_h[j]].get();
        data.pore_model = pm;
        data.event_start_idx = e_start[j];
        data.event_stop_idx = e_stop[j];
        data.strand = 0;
        data.rc = rc[j];
        data.event_stride = rc[j] ? -1 : 1;
        out[j] = profile_hmm_score(hseq, data, flags[j]);
    }
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count();
}

// profile_hmm_align on one job; out = (event_idx, kmer_idx) u32 pairs, l_fm floats, state chars.
// Guards nothing: the reference is built with its asserts on, so a job with fewer than two events or a path that enters a
// -inf cell aborts the calling process (tests/test_viterbi_edges_oracle.py runs such jobs in a forked child).
int npref_align(int read_h, int model_h, const char* seq, uint32_t e_start, uint32_t e_stop, int rc, uint32_t flags,
                double indel_bias, uint32_t* ev_kmer_out, float* lfm_out, char* state_out, uint32_t cap)
{
    hmm_indel_bias_factor = indel_bias;
    const PoreModel* pm = g_models[model_h];
    HMMInputSequence hseq(std::string(seq), pm->pmalphabet);
    HMMInputData data;
    data.read = g_reads[read_h].get();
    data.pore_model = pm;
    data.event_start_idx = e_start;
    data.event_stop_idx = e_stop;
    data.strand = 0;
    data.rc = rc;
    data.event_stride = rc ? -1 : 1;
    std::vector<HMMAlignmentState> a = profile_hmm_align(hseq, data, flags);
    if (a.size() > cap) return -1;
    for (size_t i = 0; i < a.size(); ++i) {
        ev_kmer_out[2 * i] = a[i].event_idx; ev_kmer_out[2 * i + 1] = a[i].kmer_idx;
        lfm_out[i] = (float)a[i].l_fm; state_out[i] = a[i].state;
    }
    return (int)a.size();
}

int npref_kmer_ranks(int model_h, const char* seq, int rc, uint32_t* out)
{
    const PoreModel* pm = g_models[model_h];
    HMMInputSequence hseq(std::string(seq), pm->pmalphabet);
    uint32_t k = pm->k;
    if(hseq.length() < k) return 0;
    uint32_t n = hseq.length() - k + 1;
    for(uint32_t i = 0; i < n; ++i) out[i] = hseq.get_kmer_rank(i, k, rc != 0);
    return (int)n;
}

// op: 0 reverse_complement, 1 methylate, 2 unmethylate, 3 disambiguate
int npref_alphabet_op(const char* alphabet, int op, const char* in, char* out)
{
    const Alphabet* a = get_alphabet_by_name(alphabet);
    std::string s(in), r;
    switch(op) {
        case 0: r = a->reverse_complement(s); break;
        case 1: r = a->methylate(s); break;
        case 2: r = a->unmethylate(s); break;
        case 3: r = a->disambiguate(s); break;
        default: return -1;
    }
    memcpy(out, r.c_str(), r.size() + 1);
    return (int)r.size();
}

uint32_t npref_kmer_rank(const char* alphabet, const char* kmer, uint32_t k)
{
    return get_alphabet_by_name(alphabet)->kmer_rank(kmer, k);
}

// adaptive_banded_simple_event_align on one read; pairs_out = (ref_pos, read_pos) interleaved.
// Returns the number of pairs (0 == the reference's "failed QC" empty vector), or -1 if cap too small.
int64_t npref_abea(int read_h, int model_h, const char* seq, int32_t* pairs_out, size_t cap)
{
    std::vector<AlignedPair> p =
        adaptive_banded_simple_event_align(*g_reads[read_h], *g_models[model_h], std::string(seq));
    if(p.size() > cap) return -1;
    for(size_t i = 0; i < p.size(); ++i) {
        pairs_out[2 * i] = p[i].ref_pos;
        pairs_out[2 * i + 1] = p[i].read_pos;
    }
    return (int64_t)p.size();
}

// ABEA over many reads, OpenMP over reads; returns elapsed seconds. n_pairs_out[i] = pairs of read i.
double npref_abea_batch(size_t n_reads, const int32_t* read_h, int model_h, const char* seq_buf,
                        const uint64_t* seq_off, int threads, int32_t* pairs_out,
                        const uint64_t* pairs_off, int64_t* n_pairs_out)
{
    if(threads < 1) threads = 1;
    auto t0 = std::chrono::steady_clock::now();
    #pragma omp parallel for schedule(dynamic) num_threads(threads)
    for(size_t r = 0; r < n_reads; ++r) {
        std::string seq(seq_buf + seq_off[r], seq_buf + seq_off[r + 1]);
        std::vector<AlignedPair> p =
            adaptive_banded_simple_event_align(*g_reads[read_h[r]], *g_models[model_h], seq);
        size_t cap = pairs_off[r + 1] - pairs_off[r];
        if(p.size() > cap) { n_pairs_out[r] = -1; continue; }
        int32_t* o = pairs_out + 2 * pairs_off[r];
        for(size_t i = 0; i < p.size(); ++i) { o[2 * i] = p[i].ref_pos; o[2 * i + 1] = p[i].read_pos; }
        n_pairs_out[r] = (int64_t)p.size();
    }
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count();
}

// estimate_scalings_using_mom on the events of a read; out = {shift, scale, drift, var}
void npref_mom(int read_h, int model_h, const char* seq, double* out)
{
    SquiggleRead& sr = *g_reads[read_h];
    std::vector<event_t> ev(sr.events[0].size());
    for(size_t i = 0; i < ev.size(); ++i) { ev[i].mean = sr.events[0][i].mean; ev[i].start = 0; ev[i].length = 0; ev[i].stdv = 1; ev[i].pos = 0; ev[i].state = 0; }
    event_table et; et.n = ev.size(); et.start = 0; et.end = ev.size(); et.event = ev.data();
    SquiggleScalings s = estimate_scalings_using_mom(std::string(seq), *g_models[model_h], et);
    out[0] = s.shift; out[1] = s.scale; out[2] = s.drift; out[3] = s.var;
}

void npref_logsum_table(float* out) { p7_FLogsumInit(); extern float flogsum_lookup[]; memcpy(out, flogsum_lookup, sizeof(float) * p7_LOGSUM_TBL); }
float npref_add_logs(float a, float b) { return add_logs(a, b); }
float npref_log_probability_match_r9(int read_h, int model_h, uint32_t rank, uint32_t event_idx)
{
    return log_probability_match_r9(*g_reads[read_h], *g_models[model_h], rank, event_idx, 0);
}
float npref_log_normal_pdf(float x, float mean, float stdv)
{
    GaussianParameters g(mean, stdv);
    return log_normal_pdf(x, g);
}
// detect_events (src/thirdparty/scrappie/event_detection.c:268-319) on one raw signal, the way load_from_raw
// calls it (src/nanopolish_squiggle_read.cpp:229-235: the trimmed table is discarded, the whole array is segmented).
long long npref_detect_events(const float* raw, size_t n, int rna, uint64_t* start, float* length, float* mean, float* stdv, size_t cap)
{
    raw_table rt;
    rt.n = n; rt.start = 0; rt.end = n; rt.raw = const_cast<float*>(raw);
    event_table et = detect_events(rt, rna ? event_detection_rna : event_detection_defaults);
    if (et.event == NULL) return -2;
    long long ne = (long long)et.n;
    if (et.n <= cap) {
        for (size_t i = 0; i < et.n; ++i) { start[i] = et.event[i].start; length[i] = et.event[i].length; mean[i] = et.event[i].mean; stdv[i] = et.event[i].stdv; }
    } else ne = -1;
    free(et.event);
    return ne;
}

// The same with any detector_param: windows, thresholds and peak height as given.  The signal must have at least one
// boundary (create_events reads peaks[-1] otherwise).
long long npref_detect_events_params(const float* raw, size_t n, uint32_t window_length1, uint32_t window_length2, float threshold1,
                                     float threshold2, float peak_height, uint64_t* start, float* length, float* mean, float* stdv, size_t cap)
{
    raw_table rt;
    rt.n = n; rt.start = 0; rt.end = n; rt.raw = const_cast<float*>(raw);
    detector_param prm = event_detection_defaults;
    prm.window_length1 = window_length1; prm.window_length2 = window_length2;
    prm.threshold1 = threshold1; prm.threshold2 = threshold2; prm.peak_height = peak_height;
    event_table et = detect_events(rt, prm);
    if (et.event == NULL) return -2;
    long long ne = (long long)et.n;
    if (et.n <= cap) {
        for (size_t i = 0; i < et.n; ++i) { start[i] = et.event[i].start; length[i] = et.event[i].length; mean[i] = et.event[i].mean; stdv[i] = et.event[i].stdv; }
    } else ne = -1;
    free(et.event);
    return ne;
}

// trim_and_segment_raw (src/thirdparty/scrappie/scrappie_common.c:122-138) on a table covering the whole signal.
// The function frees rt.raw when nothing survives, so it gets its own copy.  Signals for which the reference would
// trip its own assert (fewer samples than a chunk, no chunk above the threshold) must not be passed.
int npref_trim_raw(const float* raw, size_t n, int trim_start, int trim_end, int varseg_chunk, float varseg_thresh,
                   uint32_t* start_out, uint32_t* end_out)
{
    raw_table rt;
    rt.n = n; rt.start = 0; rt.end = n;
    rt.raw = (float*)malloc(n * sizeof(float));
    memcpy(rt.raw, raw, n * sizeof(float));
    rt = trim_and_segment_raw(rt, trim_start, trim_end, varseg_chunk, varseg_thresh);
    if (rt.raw == NULL) { *start_out = 0; *end_out = 0; return 0; }
    *start_out = (uint32_t)rt.start; *end_out = (uint32_t)rt.end;
    free(rt.raw);
    return 1;
}

// What trim_raw_by_mad computes before it trims (scrappie_common.c:156-172): scrappie's own madf on every chunk of the signal
// into mad_out[n / varseg_chunk] and its own quantilef of those MADs at varseg_thresh, returned.  Both are external functions of
// scrappie_common.c that its header does not declare.  The signal must hold at least one chunk.
float madf(const float* x, size_t n, const float* med);
void quantilef(const float* x, size_t nx, float* p, size_t np);
float npref_trim_mads(const float* raw, size_t n, int varseg_chunk, float varseg_thresh, float* mad_out)
{
    const size_t nchunk = n / (size_t)varseg_chunk;
    for (size_t i = 0; i < nchunk; ++i) mad_out[i] = madf(raw + i * (size_t)varseg_chunk, (size_t)varseg_chunk, NULL);
    float p = varseg_thresh;
    quantilef(mad_out, nchunk, &p, 1);
    return p;
}

int npref_max_threads(void) { return omp_get_max_threads(); }
// process-wide settings for callers that drive several harness calls from their own threads: the entry points below save / set /
// restore hmm_indel_bias_factor and the OpenMP thread count around each call, which is only safe concurrently when every call sets
// the values that are already in place
void npref_set_globals(double indel_bias, int omp_threads) { hmm_indel_bias_factor = indel_bias; omp_set_num_threads(omp_threads); }

// ---- variants: score_variant_thresholded (src/common/nanopolish_variant.cpp:765-799) for each candidate, one OpenMP thread
// so that its early exit (stop adding reads once |sum| >= threshold) follows read order deterministically.
// Reads: whole-read windows [e_start, e_stop] with the given rc flag, base model = the read's.  methylation: 0 = none, 1 = {"cpg"}.
int npref_score_variants_thresholded(int n_reads, const int32_t* read_h, const uint32_t* e_start, const uint32_t* e_stop, const uint8_t* rc,
                                     const char* ref_seq, size_t ref_position, int n_var, const size_t* var_pos, const char** var_ref,
                                     const char** var_alt, uint32_t alignment_flags, uint32_t score_threshold, int methylation,
                                     double indel_bias, double* quality_out)
{
    const double saved_bias = hmm_indel_bias_factor;
    hmm_indel_bias_factor = indel_bias;
    const int saved_threads = omp_get_max_threads();
    omp_set_num_threads(1);
    std::vector<HMMInputData> input(n_reads);
    for(int j = 0; j < n_reads; ++j) {
        HMMInputData& d = input[j];
        d.read = g_reads[read_h[j]].get();
        d.pore_model = d.read->get_base_model(0);
        d.strand = 0;
        d.event_start_idx = e_start[j];
        d.event_stop_idx = e_stop[j];
        d.rc = rc[j];
        d.event_stride = d.event_start_idx <= d.event_stop_idx ? 1 : -1;
    }
    std::vector<std::string> methylation_types;
    if(methylation) methylation_types.push_back("cpg");
    Haplotype base("contig", ref_position, ref_seq);
    for(int v = 0; v < n_var; ++v) {
        Variant var;
        var.ref_name = "contig";
        var.ref_position = var_pos[v];
        var.ref_seq = var_ref[v];
        var.alt_seq = var_alt[v];
        var.quality = 0.0;
        quality_out[v] = score_variant_thresholded(var, base, input, alignment_flags, score_threshold, methylation_types).quality;
    }
    omp_set_num_threads(saved_threads);
    hmm_indel_bias_factor = saved_bias;
    return 0;
}

// ---- modBAM tags: create_modbam_record (src/basemods/nanopolish_basemods.cpp:107-177) on a hand-built record ----
// seq = SEQ as stored in the BAM; calls = (start_position, site sequence, strand-0 log-likelihoods) of each ScoredSite.
// Returns the number of Ml entries; mm_out receives the Mm string.
long long npref_modbam(const char* seq, int ref_pos, int flag, const uint32_t* cigar, int n_cigar, int n_calls, const int32_t* start_pos,
                       const char** site_seqs, const double* ll_m0, const double* ll_u0, char* mm_out, size_t mm_cap,
                       uint8_t* ml_out, size_t ml_cap)
{
    const size_t l_qseq = strlen(seq);
    std::vector<uint8_t> data(4 + 4 * (size_t)n_cigar + (l_qseq + 1) / 2 + l_qseq);
    memcpy(data.data(), "r\0\0\0", 4);
    memcpy(data.data() + 4, cigar, 4 * (size_t)n_cigar);
    uint8_t* pseq = data.data() + 4 + 4 * (size_t)n_cigar;
    for(size_t i = 0; i < l_qseq; ++i) {
        const char* at = strchr(seq_nt16_str, seq[i]);
        const uint8_t code = at ? (uint8_t)(at - seq_nt16_str) : 15;
        pseq[i >> 1] |= code << ((~i & 1) << 2);
    }
    bam1_t rec;
    memset(&rec, 0, sizeof(rec));
    rec.core.pos = ref_pos; rec.core.tid = 0; rec.core.flag = (uint16_t)flag; rec.core.l_qname = 4; rec.core.l_extranul = 2;
    rec.core.n_cigar = n_cigar; rec.core.l_qseq = (int32_t)l_qseq; rec.core.mtid = -1; rec.core.mpos = -1;
    rec.data = data.data(); rec.l_data = (int)data.size(); rec.m_data = (uint32_t)data.size();

    std::map<int, ScoredSite> calls;
    for(int i = 0; i < n_calls; ++i) {
        ScoredSite ss;
        ss.start_position = start_pos[i];
        ss.end_position = start_pos[i];
        ss.n_motif = 1;
        ss.sequence = site_seqs[i];
        ss.ll_methylated[0] = ll_m0[i];
        ss.ll_unmethylated[0] = ll_u0[i];
        calls[start_pos[i]] = ss;
    }
    MethylationCallingParameters params;
    params.alphabet = get_alphabet_by_name(params.methylation_type);
    g_mm_tag.clear(); g_ml_tag.clear();
    bam1_t* out = create_modbam_record(&rec, calls, params);
    free(out->data); free(out);
    if(g_mm_tag.size() + 1 > mm_cap || g_ml_tag.size() > ml_cap) return -1;
    memcpy(mm_out, g_mm_tag.c_str(), g_mm_tag.size() + 1);
    memcpy(ml_out, g_ml_tag.data(), g_ml_tag.size());
    return (long long)g_ml_tag.size();
}

// ---- eventalign: segment chaining + TSV (src/alignment/nanopolish_eventalign.cpp:612-827, :398-484, :256-325) ----
// What SquiggleRead carries beyond the events once load_from_raw has run: the basecalled sequence, the
// base-to-event map (one [start, stop] per k-mer, -1 where none), event stdv / duration, the read name.
void npref_read_set_eventalign(int h, const char* read_name, const char* read_sequence, const int32_t* map_start,
                               const int32_t* map_stop, size_t n_map, const float* stdv, const float* duration)
{
    SquiggleRead& sr = *g_reads[h];
    sr.read_name = read_name;
    sr.read_sequence = read_sequence;
    sr.base_to_event_map.resize(n_map);
    for(size_t i = 0; i < n_map; ++i) {
        sr.base_to_event_map[i].indices[0].start = map_start[i];
        sr.base_to_event_map[i].indices[0].stop = map_stop[i];
    }
    for(size_t i = 0; i < sr.events[0].size(); ++i) {
        sr.events[0][i].stdv = stdv[i];
        sr.events[0][i].duration = duration[i];
    }
}

// the trimmed raw samples load_from_raw keeps with SRF_LOAD_RAW_SAMPLES (src/nanopolish_squiggle_read.cpp:251-258)
void npref_read_set_samples(int h, const float* samples, size_t n, double sample_rate)
{
    SquiggleRead& sr = *g_reads[h];
    sr.samples.assign(samples, samples + n);
    sr.sample_start_time = 0;
    sr.sample_rate = sample_rate;
}
// SquiggleRead::get_event_sample_idx and ::get_scaled_samples_for_event (:399-428) of one event: what eventalign's
// --signal-index / --samples columns print.  Returns the number of samples.
long long npref_event_samples(int h, size_t event_idx, uint64_t* idx2_out, float* samples_out, size_t cap)
{
    const SquiggleRead& sr = *g_reads[h];
    const std::pair<size_t, size_t> si = sr.get_event_sample_idx(0, event_idx);
    idx2_out[0] = si.first; idx2_out[1] = si.second;
    const std::vector<float> v = sr.get_scaled_samples_for_event(0, event_idx);
    if(v.size() > cap) return -1;
    memcpy(samples_out, v.data(), sizeof(float) * v.size());
    return (long long)v.size();
}

namespace { thread_local EventalignSummary g_last_summary; }
// align_read_to_ref on a hand-built BAM record (pos, flag, CIGAR), then emit_event_alignment_tsv (default options)
// into tsv_out and the event CIGAR of the SAM output into cigar_out.  Returns the number of EventAlignments, or -1
// when tsv_cap is too small.  ea_out (optional) gets (ref_position, event_idx, hmm_state) triples.
long long npref_eventalign(int read_h, const char* contig_name, const char* contig_seq, int ref_pos, int flag,
                           const uint32_t* cigar, int n_cigar, int read_idx, int region_start, int region_end,
                           char* tsv_out, size_t tsv_cap, char* cigar_out, size_t cigar_cap, int32_t* ea_out, size_t ea_cap)
{
    NprefContig contig{contig_name, contig_seq};
    bam_hdr_t hdr;
    memset(&hdr, 0, sizeof(hdr));
    char* names[1] = { const_cast<char*>(contig.name.c_str()) };
    uint32_t lens[1] = { (uint32_t)contig.seq.size() };
    hdr.n_targets = 1; hdr.target_name = names; hdr.target_len = lens;
    bam1_t rec;
    memset(&rec, 0, sizeof(rec));
    std::vector<uint8_t> data(4 + 4 * (size_t)n_cigar);
    memcpy(data.data(), "r\0\0\0", 4);
    memcpy(data.data() + 4, cigar, 4 * (size_t)n_cigar);
    rec.core.pos = ref_pos; rec.core.tid = 0; rec.core.flag = (uint16_t)flag; rec.core.l_qname = 4; rec.core.l_extranul = 2;
    rec.core.n_cigar = n_cigar; rec.core.mtid = -1; rec.core.mpos = -1;
    rec.data = data.data(); rec.l_data = (int)data.size(); rec.m_data = (uint32_t)data.size();

    EventAlignmentParameters params;
    params.sr = g_reads[read_h].get();
    params.fai = reinterpret_cast<const faidx_t*>(&contig);
    params.hdr = &hdr;
    params.record = &rec;
    params.strand_idx = 0;
    params.read_idx = read_idx;
    params.region_start = region_start;
    params.region_end = region_end;
    std::vector<EventAlignment> alignment = align_read_to_ref(params);

    char* buf = NULL; size_t len = 0;
    FILE* fp = open_memstream(&buf, &len);
    emit_event_alignment_tsv(fp, *params.sr, 0, params, alignment);
    fclose(fp);
    bool ok = len < tsv_cap;
    if(ok) { memcpy(tsv_out, buf, len); tsv_out[len] = 0; }
    free(buf);
    if(!ok) return -1;
    // (event_alignment_to_cigar asserts on the event jump between two BAM segments: callers skip it for records with an N)
    std::string cs = (alignment.empty() || cigar_cap == 0) ? std::string() : cigar_ops_to_string(event_alignment_to_cigar(alignment));
    if(cigar_cap == 0) {} else if(cs.size() < cigar_cap) strcpy(cigar_out, cs.c_str()); else cigar_out[0] = 0;
    for(size_t i = 0; i < alignment.size() && 3 * i + 2 < ea_cap; ++i) {
        ea_out[3 * i] = alignment[i].ref_position; ea_out[3 * i + 1] = alignment[i].event_idx; ea_out[3 * i + 2] = alignment[i].hmm_state;
    }
    g_last_summary = summarize_alignment(*params.sr, 0, params, alignment);
    return (long long)alignment.size();
}

// the EventalignSummary of the most recent npref_eventalign call on this thread: {events, steps, stays, skips, span} and
// {sum_duration, sum_z_score}
void npref_eventalign_summary(int32_t* ints5, double* doubles2)
{
    ints5[0] = g_last_summary.num_events; ints5[1] = g_last_summary.num_steps; ints5[2] = g_last_summary.num_stays;
    ints5[3] = g_last_summary.num_skips; ints5[4] = g_last_summary.reference_span;
    doubles2[0] = g_last_summary.sum_duration; doubles2[1] = g_last_summary.sum_z_score;
}

// ---- call-methylation: calculate_methylation_for_read (src/basemods/nanopolish_basemods.cpp:238-457) followed by
// write_methylation_results_as_tsv (src/nanopolish_call_methylation.cpp:532-550) on a hand-built BAM record ----
// The read carries what load_from_raw leaves (events, scalings, read_sequence, base_to_event_map: npref_read_create +
// npref_read_set_eventalign); the reference comes from the in-memory contig through the faidx test double.  Returns the
// number of ScoredSites; sites_out gets (start, end, n_motif, strands_scored) and ll_out (ll_unmethylated[0],
// ll_methylated[0]) per site; tsv_out the rows the reference prints.  -1: a buffer is too small.
long long npref_call_methylation(int read_h, const char* read_name, const char* contig_name, const char* contig_seq, int ref_pos, int flag,
                                 const uint32_t* cigar, int n_cigar, const char* methylation_type, int region_start, int region_end,
                                 double indel_bias, char* tsv_out, size_t tsv_cap, int32_t* sites_out, double* ll_out, size_t site_cap)
{
    NprefContig contig{contig_name, contig_seq};
    bam_hdr_t hdr;
    memset(&hdr, 0, sizeof(hdr));
    char* names[1] = { const_cast<char*>(contig.name.c_str()) };
    uint32_t lens[1] = { (uint32_t)contig.seq.size() };
    hdr.n_targets = 1; hdr.target_name = names; hdr.target_len = lens;
    // record data: qname (NUL-terminated, padded to a multiple of four), CIGAR; no SEQ / QUAL (l_qseq = 0)
    const size_t nl = strlen(read_name) + 1, l_qname = (nl + 3) / 4 * 4;
    std::vector<uint8_t> data(l_qname + 4 * (size_t)n_cigar, 0);
    memcpy(data.data(), read_name, nl);
    memcpy(data.data() + l_qname, cigar, 4 * (size_t)n_cigar);
    bam1_t rec;
    memset(&rec, 0, sizeof(rec));
    rec.core.pos = ref_pos; rec.core.tid = 0; rec.core.flag = (uint16_t)flag; rec.core.l_qname = (uint16_t)l_qname;
    rec.core.l_extranul = (uint8_t)(l_qname - nl); rec.core.n_cigar = n_cigar; rec.core.mtid = -1; rec.core.mpos = -1;
    rec.data = data.data(); rec.l_data = (int)data.size(); rec.m_data = (uint32_t)data.size();

    MethylationCallingParameters params;
    params.methylation_type = methylation_type;
    params.alphabet = get_alphabet_by_name(params.methylation_type);
    OutputHandles handles;
    MethylationCallingResult result;
    const double saved_bias = hmm_indel_bias_factor;
    hmm_indel_bias_factor = indel_bias;
    calculate_methylation_for_read(handles, result, *g_reads[read_h], params, reinterpret_cast<const faidx_t*>(&contig), &hdr, &rec, 0,
                                   region_start, region_end);
    hmm_indel_bias_factor = saved_bias;
    std::map<int, ScoredSite>& sites = result[&rec];
    char* buf = NULL; size_t len = 0;
    FILE* fp = open_memstream(&buf, &len);
    write_methylation_results_as_tsv(fp, &rec, sites);
    fclose(fp);
    const bool ok = len < tsv_cap && sites.size() <= site_cap;
    if(ok) {
        memcpy(tsv_out, buf, len); tsv_out[len] = 0;
        size_t i = 0;
        for(const auto& kv : sites) {
            const ScoredSite& ss = kv.second;
            sites_out[4 * i] = ss.start_position; sites_out[4 * i + 1] = ss.end_position; sites_out[4 * i + 2] = ss.n_motif;
            sites_out[4 * i + 3] = ss.strands_scored;
            ll_out[2 * i] = ss.ll_unmethylated[0]; ll_out[2 * i + 1] = ss.ll_methylated[0];
            ++i;
        }
    }
    free(buf);
    return ok ? (long long)sites.size() : -1;
}

// ---- calibration after ABEA: the tail of SquiggleRead::load_from_raw (src/nanopolish_squiggle_read.cpp:272-336) ----
// load_from_raw itself needs fast5/slow5 input and cannot be called; what it does with the ABEA result is (a) the
// base-to-event map loop (:272-300), transcribed below because it is inline in that function, (b) the reference's own
// SquiggleRead::get_eventalignment_for_1d_basecalls (:340-391) and (c) the reference's own recalibrate_model
// (src/nanopolish_methyltrain.cpp:204-307), both compiled unmodified — recalibrate_model's FullPivLU solve through the
// restated header oracle/shim/Eigen/Dense (Eigen is not vendored and absent here).
// pairs = (k-mer, event) AlignedPairs as adaptive_banded_simple_event_align returns them.  out6 = shift, scale, drift, var,
// events_per_base, calibrated (0/1); returns the number of 'M' events, or -1 for an empty alignment.
long long npref_calibrate(int read_h, int model_h, const char* read_sequence, const int32_t* pairs, size_t n_pairs, double* out6)
{
    SquiggleRead& sr = *g_reads[read_h];
    const PoreModel& model = *g_models[model_h];
    const size_t strand_idx = 0;
    sr.read_sequence = read_sequence;
    if(n_pairs == 0) return -1;
    const size_t n_kmers = sr.read_sequence.size() - model.k + 1;
    sr.base_to_event_map.clear();
    sr.base_to_event_map.resize(n_kmers);
    size_t max_event = 0;
    size_t min_event = std::numeric_limits<size_t>::max();
    size_t prev_event_idx = -1;
    for(size_t i = 0; i < n_pairs; ++i) {
        size_t k_idx = pairs[2 * i];
        size_t event_idx = pairs[2 * i + 1];
        IndexPair& elem = sr.base_to_event_map[k_idx].indices[strand_idx];
        if(event_idx != prev_event_idx) {
            if(elem.start == -1) elem.start = event_idx;
            elem.stop = event_idx;
        }
        max_event = std::max(max_event, event_idx);
        min_event = std::min(min_event, event_idx);
        prev_event_idx = event_idx;
    }
    const double events_per_base = (double)(max_event - min_event) / n_kmers;
    std::vector<EventAlignment> alignment =
        sr.get_eventalignment_for_1d_basecalls(sr.read_sequence, "nucleotide", sr.base_to_event_map, model.k, strand_idx, 0);
    long long n_m = 0;
    for(const EventAlignment& ea : alignment) n_m += ea.hmm_state == 'M';
    const bool calibrated = recalibrate_model(sr, model, strand_idx, alignment, true, false);
    const SquiggleScalings& s = sr.scalings[strand_idx];
    out6[0] = s.shift; out6[1] = s.scale; out6[2] = s.drift; out6[3] = s.var; out6[4] = events_per_base; out6[5] = calibrated ? 1.0 : 0.0;
    return n_m;
}

// ---- variants: score_variant_group (src/common/nanopolish_variant.cpp:182-262): every combination of up to max_r of the group's
// variants applied to the base haplotype, each scored against every read with profile_hmm_score_set.  combos_out[c] = bitmask of
// the variant ids of combination c (c = VariantGroup's combination index), scores_out[c * n_reads + r] = its score for read r.
// Returns the number of combinations (-1: cap_comb too small).
long long npref_score_variant_group(int n_reads, const int32_t* read_h, const uint32_t* e_start, const uint32_t* e_stop, const uint8_t* rc,
                                    const char* ref_seq, size_t ref_position, int n_var, const size_t* var_pos, const char** var_ref,
                                    const char** var_alt, int max_haplotypes, uint32_t alignment_flags, int methylation, double indel_bias,
                                    uint32_t* combos_out, double* scores_out, size_t cap_comb)
{
    const double saved_bias = hmm_indel_bias_factor;
    hmm_indel_bias_factor = indel_bias;
    std::vector<HMMInputData> input(n_reads);
    for(int j = 0; j < n_reads; ++j) {
        HMMInputData& d = input[j];
        d.read = g_reads[read_h[j]].get();
        d.read->read_name = "r" + std::to_string(read_h[j]);       // read ids of the group's score table must be distinct
        d.pore_model = d.read->get_base_model(0);
        d.strand = 0;
        d.event_start_idx = e_start[j];
        d.event_stop_idx = e_stop[j];
        d.rc = rc[j];
        d.event_stride = d.event_start_idx <= d.event_stop_idx ? 1 : -1;
    }
    std::vector<std::string> methylation_types;
    if(methylation) methylation_types.push_back("cpg");
    std::vector<Variant> vars(n_var);
    for(int v = 0; v < n_var; ++v) {
        vars[v].ref_name = "contig"; vars[v].ref_position = var_pos[v]; vars[v].ref_seq = var_ref[v]; vars[v].alt_seq = var_alt[v];
        vars[v].quality = 0.0;
    }
    VariantGroup group(0, vars);
    Haplotype base("contig", ref_position, ref_seq);
    score_variant_group(group, base, input, max_haplotypes, 1, false, alignment_flags, methylation_types);
    hmm_indel_bias_factor = saved_bias;
    const size_t nc = group.get_num_combinations();
    if(nc > cap_comb) return -1;
    for(size_t c = 0; c < nc; ++c) {
        const VariantCombination& vc = group.get_combination(c);
        uint32_t mask = 0;
        for(size_t i = 0; i < vc.get_num_variants(); ++i) mask |= 1u << vc.get_variant_id(i);
        combos_out[c] = mask;
        for(int r = 0; r < n_reads; ++r)
        {
            // the read id score_variant_group forms (:236-238): operator<< of the uint8_t strand writes the CHARACTER with that code
            std::stringstream ss;
            ss << input[r].read->read_name << ":" << input[r].strand;
            scores_out[c * (size_t)n_reads + r] = group.get_combination_read_score(c, ss.str());
        }
    }
    return (long long)nc;
}

} // extern "C"
