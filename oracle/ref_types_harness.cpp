// oracle/ref_types_harness.cpp — TEST INFRASTRUCTURE ONLY.
//
// score_variant_thresholded (src/common/nanopolish_variant.cpp:765-799) with any opt::methylation_types list, for the tests of
// methylation-aware candidate screening (`variants -q cpg`, `-q dam,dcm`).  Linked by oracle/ref_types.mk into
// oracle/_ref/libnpref_types.so together with the same UNMODIFIED reference objects oracle/Makefile compiles for libnpref.so.
// Reads are assembled like npref_read_create does (ref_harness.cpp), with the built-in r9.4_450bps template nucleotide model as base
// model: SquiggleRead::get_model(strand, type) then finds the built-in model of each methylation type.
//
// The product (nanopolish_b200/, include/) never links or loads this file.
#include <cstdint>
#include <memory>
#include <string>
#include <vector>
#include <omp.h>

#include "nanopolish_common.h"
#include "nanopolish_squiggle_read.h"
#include "nanopolish_pore_model_set.h"
#include "nanopolish_profile_hmm.h"
#include "nanopolish_variant.h"
#include "nanopolish_haplotype.h"

extern double hmm_indel_bias_factor;   // src/hmm/nanopolish_profile_hmm_r9.cpp:19

namespace {
std::vector<std::unique_ptr<SquiggleRead>> g_type_reads;
}

extern "C" {

int npref_types_read_create(uint32_t n_events, const float* mean, const double* start_time,
                            double shift, double scale, double drift, double var, double events_per_base)
{
    std::unique_ptr<SquiggleRead> sr(new SquiggleRead());
    sr->pore_type = PORETYPE_R9;
    sr->read_type = SRT_TEMPLATE;
    sr->nucleotide_type = SRNT_DNA;
    sr->base_model[0] = PoreModelSet::get_model("r9.4_450bps", "nucleotide", "template", 6);
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
    g_type_reads.push_back(std::move(sr));
    return (int)g_type_reads.size() - 1;
}

void npref_types_reads_clear(void) { g_type_reads.clear(); }

// score_variant_thresholded for each variant, one OpenMP thread (its early exit then follows read order).  Reads: windows
// [e_start, e_stop] with the given rc flag, base model = the read's.  types_csv: opt::methylation_types as a comma-separated list in
// -q order ("" = none).
int npref_types_score_variants_thresholded(int n_reads, const int32_t* read_h, const uint32_t* e_start, const uint32_t* e_stop, const uint8_t* rc,
                                           const char* ref_seq, size_t ref_position, int n_var, const size_t* var_pos, const char** var_ref,
                                           const char** var_alt, uint32_t alignment_flags, uint32_t score_threshold, const char* types_csv,
                                           double indel_bias, double* quality_out)
{
    const double saved_bias = hmm_indel_bias_factor;
    hmm_indel_bias_factor = indel_bias;
    const int saved_threads = omp_get_max_threads();
    omp_set_num_threads(1);
    std::vector<HMMInputData> input(n_reads);
    for(int j = 0; j < n_reads; ++j) {
        HMMInputData& d = input[j];
        d.read = g_type_reads[read_h[j]].get();
        d.pore_model = d.read->get_base_model(0);
        d.strand = 0;
        d.event_start_idx = e_start[j];
        d.event_stop_idx = e_stop[j];
        d.rc = rc[j];
        d.event_stride = d.event_start_idx <= d.event_stop_idx ? 1 : -1;
    }
    std::vector<std::string> methylation_types;
    for(std::string s = types_csv; !s.empty(); ) {
        const size_t c = s.find(',');
        methylation_types.push_back(s.substr(0, c));
        s = c == std::string::npos ? std::string() : s.substr(c + 1);
    }
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

} // extern "C"
