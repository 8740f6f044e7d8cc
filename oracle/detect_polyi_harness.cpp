// detect_polyi_harness.cpp — TEST INFRASTRUCTURE ONLY.  Drives the reference's own detect-polyi code
// (src/nanopolish_detect_polyi.cpp, compiled here in place through the #include below, found on the reference's include path:
// DPISegmentationHMM and BernoulliHMM are local to that file) on a SquiggleRead assembled by hand the way polya_harness.cpp
// assembles one: samples, sample rate, scalings, event durations, base-to-event map and a basecalled sequence of the right
// length are set directly.
//
// dpi_estimate_polya_for_single_read itself needs a ReadDB and a fast5 file to build its SquiggleRead, so the harness runs the
// steps it runs after loading (:1061-1095): dpi_pre_segmentation_qc, DPISegmentationHMM(...).segment_squiggle,
// dpi_post_segmentation_qc, dpi_estimate_unaligned_duration_profile, dpi_estimate_polya_length, dpi_post_estimation_qc,
// BernoulliHMM(...).segmentation and post_boolhmm_detetection_qc, then prints the row with the reference's format string
// (:1105-1108).  The QC priority (:1079-1088) is the only restated logic.  Nothing of the reference is copied.
#include "nanopolish_detect_polyi.cpp"

#include <chrono>

namespace {
PoreModel g_polyi_model(5);   // only k is read (dpi_estimate_unaligned_duration_profile, :820)

void build_read(SquiggleRead& sr, const float* samples, size_t n, double sample_rate, double scale, double shift, double var,
                const float* duration, size_t n_events, const int32_t* map_start, const int32_t* map_stop, size_t n_kmers)
{
    sr.base_model[0] = &g_polyi_model;
    sr.base_model[1] = NULL;
    sr.scalings[0].set4(shift, scale, 0.0, var);
    sr.samples.assign(samples, samples + n);
    sr.sample_rate = sample_rate;
    sr.sample_start_time = 0;
    sr.read_sequence.assign(n_kmers + g_polyi_model.k - 1, 'A');
    sr.base_to_event_map.resize(n_kmers);
    for (size_t i = 0; i < n_kmers; ++i) {
        sr.base_to_event_map[i].indices[0].start = map_start[i];
        sr.base_to_event_map[i].indices[0].stop = map_stop[i];
    }
    sr.events[0].resize(n_events);
    for (size_t i = 0; i < n_events; ++i) sr.events[0][i].duration = duration[i];
}

int tag_code(const std::string& tag)   // NPH_POLYI_*
{
    return tag == "NONE" ? 0 : tag == "POLYA-ONLY" ? 1 : tag == "POLYI-ONLY" ? 2 : 3;
}
} // namespace

extern "C" {

// One loaded read.  seg_out: start, leader, adapter, polya, cliffs; rate_len_out: read_rate, polya_length; *qc_out: 0 PASS,
// 1 NOREGION, 2 ADAPTER, 3 SUFFCLIP; bern_out: BernoulliSegmentation {polyi, polya}; *detected_out: 0 NONE, 1 POLYA-ONLY,
// 2 POLYI-ONLY, 3 A+I.  The row (with its newline) goes to row_out; returns its length, -1 if cap is too small.
long long npref_polyi_read(const char* read_name, const char* ref_name, int pos, uint32_t suffix_clip,
                           const float* samples, size_t n, double sample_rate, double scale, double shift, double var,
                           const float* duration, size_t n_events, const int32_t* map_start, const int32_t* map_stop, size_t n_kmers,
                           uint64_t* seg_out, double* rate_len_out, int* qc_out, int32_t* bern_out, int* detected_out,
                           char* row_out, size_t cap)
{
    SquiggleRead sr;
    build_read(sr, samples, n, sample_rate, scale, shift, var, duration, n_events, map_start, map_stop, n_kmers);
    std::string pre_segmentation_qc_flag = dpi_pre_segmentation_qc(suffix_clip, 0, sr.read_sequence.length(), sr);
    DPISegmentationHMM hmm(static_cast<float>(sr.scalings[0].scale),
                           static_cast<float>(sr.scalings[0].shift),
                           static_cast<float>(sr.scalings[0].var));
    DPISegmentation region_indices = hmm.segment_squiggle(sr);
    std::string post_segmentation_qc_flag = dpi_post_segmentation_qc(region_indices, sr);
    double read_rate = dpi_estimate_unaligned_duration_profile(sr, NULL, NULL, NULL, 0, 0);
    double polya_length = dpi_estimate_polya_length(sr, region_indices, read_rate);
    std::string post_estimation_qc_flag = dpi_post_estimation_qc(region_indices, sr, read_rate, polya_length);
    std::string qc_tag;
    if (post_segmentation_qc_flag.compare("PASS") != 0) qc_tag = post_segmentation_qc_flag;
    else if (post_estimation_qc_flag.compare("PASS") != 0) qc_tag = post_estimation_qc_flag;
    else if (pre_segmentation_qc_flag.compare("PASS") != 0) qc_tag = pre_segmentation_qc_flag;
    else qc_tag = "PASS";
    BernoulliHMM boolhmm(static_cast<float>(sr.scalings[0].scale),
                         static_cast<float>(sr.scalings[0].shift),
                         static_cast<float>(sr.scalings[0].var));
    BernoulliSegmentation poly_segmentation = boolhmm.segmentation(sr, region_indices.adapter+1, region_indices.polya);
    std::string poly_detect_tag = post_boolhmm_detetection_qc(poly_segmentation, (region_indices.polya-(region_indices.adapter+1)));

    seg_out[0] = region_indices.start; seg_out[1] = region_indices.leader; seg_out[2] = region_indices.adapter;
    seg_out[3] = region_indices.polya; seg_out[4] = region_indices.cliffs;
    rate_len_out[0] = read_rate; rate_len_out[1] = polya_length;
    *qc_out = qc_tag == "PASS" ? 0 : qc_tag == "NOREGION" ? 1 : qc_tag == "ADAPTER" ? 2 : 3;
    bern_out[0] = poly_segmentation.polyi; bern_out[1] = poly_segmentation.polya;
    *detected_out = tag_code(poly_detect_tag);

    double leader_sample_start = region_indices.start+1;
    double adapter_sample_start = region_indices.leader+1;
    double polya_sample_start = region_indices.adapter+1;
    double transcr_sample_start = region_indices.polya+1;
    const int len = snprintf(row_out, cap, "%s\t%s\t%d\t%.1lf\t%.1lf\t%.1lf\t%.1lf\t%.2lf\t%.2lf\t%s\t%s\n",
                             read_name, ref_name, pos, leader_sample_start, adapter_sample_start, polya_sample_start,
                             transcr_sample_start, read_rate, polya_length, poly_detect_tag.c_str(), qc_tag.c_str());
    return (len < 0 || (size_t)len >= cap) ? -1 : len;
}

// the row of a read that failed to load (:1040-1041)
long long npref_polyi_failed_row(const char* read_name, const char* ref_name, int pos, char* row_out, size_t cap)
{
    const int len = snprintf(row_out, cap, "%s\t%s\t%d\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n", read_name, ref_name, pos);
    return (len < 0 || (size_t)len >= cap) ? -1 : len;
}

// wall time in seconds of segment_squiggle + dpi_estimate_unaligned_duration_profile + the Bernoulli segmentation for one read
// (CPU cost of the hot part)
double npref_polyi_time(const float* samples, size_t n, double sample_rate, double scale, double shift, double var,
                        const float* duration, size_t n_events, const int32_t* map_start, const int32_t* map_stop, size_t n_kmers)
{
    SquiggleRead sr;
    build_read(sr, samples, n, sample_rate, scale, shift, var, duration, n_events, map_start, map_stop, n_kmers);
    const auto t0 = std::chrono::steady_clock::now();
    DPISegmentationHMM hmm(static_cast<float>(sr.scalings[0].scale), static_cast<float>(sr.scalings[0].shift),
                           static_cast<float>(sr.scalings[0].var));
    DPISegmentation region_indices = hmm.segment_squiggle(sr);
    volatile double rate = dpi_estimate_unaligned_duration_profile(sr, NULL, NULL, NULL, 0, 0);
    BernoulliHMM boolhmm(static_cast<float>(sr.scalings[0].scale), static_cast<float>(sr.scalings[0].shift),
                         static_cast<float>(sr.scalings[0].var));
    volatile int polyi = boolhmm.segmentation(sr, region_indices.adapter+1, region_indices.polya).polyi;
    (void)rate; (void)polyi;
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

} // extern "C"
