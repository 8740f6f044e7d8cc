// nph_variants.hpp — SURVEY.md section 8(f) row N2: the variant-scoring callers of profile_hmm_score_set,
// re-expressed as job generators over the batched forward kernel.
//
//   Variant (the fields scoring touches)        ref: src/common/nanopolish_variant.h:21-110
//   Haplotype::apply_variant(s)                  ref: src/nanopolish_haplotype.cpp:30-85
//   generate_methylated_alternatives             ref: src/common/nanopolish_variant.cpp:158-178
//   score_variant_thresholded                    ref: src/common/nanopolish_variant.cpp:765-799
//   the scoring loop of score_variant_group      ref: src/common/nanopolish_variant.cpp:242-258
//   fix_homopolymers                             ref: src/nanopolish_call_variants.cpp:541-780 (its likelihoods on the device,
//                                                nph_homopolymer_likelihoods_batch)
//   annotate_variants_with_all_support           ref: src/common/nanopolish_variant.cpp:801-859 (its scores on the device,
//                                                nph_all_support_batch)
//   screen_variants_by_score                     ref: src/nanopolish_call_variants.cpp:364-402 (on the device,
//                                                nph_screen_variants_batch)
//   expand_variants                              ref: src/nanopolish_call_variants.cpp:406-450 (host only)
//   call_haplotype_from_candidates               ref: src/nanopolish_call_variants.cpp:782-880 (its scores and genotype choice on
//                                                the device, nph_call_variant_groups_batch), with simple_call's output
//                                                (src/common/nanopolish_variant.cpp:279-493)
//
// The reference scores one (read, sequence) pair per profile_hmm_score call inside an OpenMP loop.  Here every
// (read, haplotype, alphabet alternative) triple of a whole candidate set becomes one job of ONE launch; the base
// haplotype is scored once per read instead of once per candidate; the reference's host arithmetic on the returned
// floats (profile_hmm_score_set's table logsum in double, the early-exit accumulation of score_variant_thresholded
// in read order) is applied afterwards, unchanged.
#pragma once
#include "nph_host.hpp"
#include "nph_methylation.hpp"

namespace nph {

struct Variant {
    std::string ref_name;
    size_t ref_position = 0;
    std::string ref_seq;
    std::string alt_seq;
    double quality = 0.0;
    std::string info, genotype, filter;
    std::string key() const { return ref_name + ":" + std::to_string(ref_position) + ":" + ref_seq + ":" + alt_seq; }
    // Variant::add_info (ref: src/common/nanopolish_variant.h:82-92): key=value, ';'-separated
    template <typename T> void add_info(const std::string& k, T value)
    {
        const std::string kv = k + "=" + std::to_string(value);
        info = info.empty() ? kv : info + ";" + kv;
    }
    void add_info(const std::string& k, const std::string& value)
    {
        const std::string kv = k + "=" + value;
        info = info.empty() ? kv : info + ";" + kv;
    }
};

class Haplotype {
public:
    static const size_t INSERTED_POSITION;
    Haplotype(const std::string& ref_name, size_t ref_position, const std::string& ref_sequence);
    bool apply_variant(const Variant& v);                       // false (and no change) if incompatible
    bool apply_variants(const std::vector<Variant>& variants);
    const std::string& get_sequence() const { return m_sequence; }
    const std::string& get_reference() const { return m_reference; }
    size_t get_reference_position() const { return m_ref_position; }
    size_t get_reference_position_for_haplotype_base(size_t i) const;
    const std::vector<Variant>& get_variants() const { return m_variants; }
    const std::string& get_reference_name() const { return m_ref_name; }
    size_t get_reference_end() const { return m_ref_position + m_reference.length(); }
    // the reference positions of the haplotype's bases (INSERTED_POSITION for an inserted base)
    const std::vector<size_t>& coordinate_map() const { return m_coordinate_map; }
    // the haplotype over reference [start, end] (ref: src/nanopolish_haplotype.cpp:88-140): its first base is the last one at or
    // before start that has a reference position; throws Error(NPH_ERR_INVALID) where the reference asserts
    Haplotype substr_by_reference(size_t start, size_t end) const;
    // ref: src/nanopolish_haplotype.cpp:141-158.  Moves hap_lower down and hap_upper up over inserted bases and returns their
    // reference positions; all four npos when hap_lower reaches 0 or hap_upper the end
    void get_enclosing_reference_range_for_haplotype_range(size_t& hap_lower, size_t& hap_upper, size_t& ref_lower, size_t& ref_upper) const;

private:
    size_t find_derived_index_by_ref_lower_bound(size_t ref_index) const;
    std::string m_ref_name;
    size_t m_ref_position;
    std::string m_reference, m_sequence;
    std::vector<size_t> m_coordinate_map;
    std::vector<Variant> m_variants;
};

// {sequence} plus one methylated version per alphabet in methylation_types that changes the sequence
std::vector<HMMInputSequence> generate_methylated_alternatives(const HMMInputSequence& sequence,
                                                               const std::vector<std::string>& methylation_types);

// scores[read][haplotype] = profile_hmm_score_set(generate_methylated_alternatives(haplotype), input[read], flags)
// — the scoring loop of score_variant_group — as one batch.
std::vector<std::vector<double>> score_haplotypes(const std::vector<Haplotype>& haplotypes, const std::vector<HMMInputData>& input,
                                                  uint32_t alignment_flags, const std::vector<std::string>& methylation_types,
                                                  Engine& engine, double indel_bias = hmm_indel_bias_factor);

// The combinations of score_variant_group (ref: src/common/nanopolish_variant.cpp:193-232): max_r is the largest r for which the
// haplotype count stays below max_haplotypes; for r = 0..max_r the r-subsets of the group's variants in the order of the reference's
// Combinations generator (prev_permutation on a bool mask: ascending ids, lexicographic), each kept with its haplotype when
// apply_variants succeeds on base_haplotype.  Combination 0 is the empty one.
struct VariantCombinations {
    std::vector<std::vector<size_t>> combinations;
    std::vector<Haplotype> haplotypes;
    size_t max_r = 0;
};
VariantCombinations variant_combinations(const std::vector<Variant>& variants, const Haplotype& base_haplotype, int max_haplotypes);

// score_variant_group (ref: src/common/nanopolish_variant.cpp:182-262): every combination of variant_combinations scored against
// every read with profile_hmm_score_set, all as ONE batch.  combinations[c] lists the variant ids of combination c, scores[c][read]
// is what VariantGroup::set_combination_read_score receives.
struct VariantGroupScores {
    std::vector<std::vector<size_t>> combinations;
    std::vector<std::vector<double>> scores;
    size_t max_r = 0;
};
size_t nChoosek(size_t n, size_t k);                           // ref: src/common/nanopolish_common.cpp:93-105 (int arithmetic inside)
VariantGroupScores score_variant_group(const std::vector<Variant>& variants, const Haplotype& base_haplotype,
                                       const std::vector<HMMInputData>& input, int max_haplotypes, uint32_t alignment_flags,
                                       const std::vector<std::string>& methylation_types, Engine& engine,
                                       double indel_bias = hmm_indel_bias_factor);

// score_variant_thresholded for a whole candidate list: quality_i = sum over reads, in input order, of
// (variant_score - base_score), where a read is skipped once |running total| >= score_threshold — exactly the
// single-thread behaviour of the reference loop (its OpenMP version makes the skip set racy; the result here is
// the deterministic one).  Candidates that do not apply to the base haplotype keep quality 0.
std::vector<Variant> score_variants_thresholded(const std::vector<Variant>& input_variants, const Haplotype& base_haplotype,
                                                const std::vector<HMMInputData>& input, uint32_t alignment_flags,
                                                uint32_t score_threshold, const std::vector<std::string>& methylation_types,
                                                Engine& engine, double indel_bias = hmm_indel_bias_factor);

// the reference's single-candidate signature
Variant score_variant_thresholded(const Variant& input_variant, Haplotype base_haplotype, const std::vector<HMMInputData>& input,
                                  uint32_t alignment_flags, uint32_t score_threshold, const std::vector<std::string>& methylation_types);

// One SequenceAlignmentRecord of AlignmentDB (ref: src/alignment/nanopolish_alignment_db.h): the read's name and strand, its bases as
// stored in the BAM (seq_nt16_str characters, '=' and 'N' included) and aligned_bases = get_aligned_segments(record)[0]
struct SequenceAlignedRead {
    std::string read_name;
    bool rc = false;
    std::string sequence;
    std::vector<AlignedPair> aligned_bases;
};

// The AlignmentDB fix_homopolymers reads: the region [region_start, region_start + reference.size() - 1] of one contig and its event
// alignment records in AlignmentDB's order, each strand 0 of its read (read->events[0] with durations; rc[0], aligned_events[0]).
// sequence_records: the base-space records (get_variants_in_region reads them; the event-space calls do not).
struct HomopolymerRegion {
    std::string contig;
    int region_start = 0;
    std::string reference;
    std::vector<EventAlignedRead> records;
    std::vector<SequenceAlignedRead> sequence_records;
};

// One homopolymer fix_homopolymers scores, in scan order: the run, its calling window and the nph_hp_window it becomes.
struct HomopolymerWindow {
    size_t hp_start, hp_end;        // [hp_start, hp_end) in the input haplotype
    std::string calling;            // substr_by_reference(ref_calling_start, ref_calling_end)
    nph_hp_window dev;
};
// the scan of :552-616: every run of 3..9 bases (the last run never) that passes the flank, enclosing-range and region tests
std::vector<HomopolymerWindow> homopolymer_windows(const Haplotype& haplotype, int region_start, int region_end, int min_flanking_sequence);

// The call of one window (ref: src/nanopolish_call_variants.cpp:686-727): the first strict maximum of d_lik + e_lik from -inf (call
// stays npos when nothing beats it), quality = max - score[hp_length], kept unless quality < 10 (a NaN is kept), and
// size_diff = int(call - hp_length) (npos: a deletion).
struct HomopolymerCall { size_t call; double quality; int size_diff; bool kept; };
HomopolymerCall homopolymer_call(const nph_hp_likelihoods& lik, size_t hp_length);

// fix_homopolymers (ref: src/nanopolish_call_variants.cpp:541-780): the scan and its skip tests here, every window's likelihood
// vectors in one nph_homopolymer_likelihoods_batch, then the call (strict argmax from -inf, quality max - score[hp_length], kept
// unless < 10) and its 1-base insertion or deletion, tried at each base of the run until apply_variant accepts one, window by
// window.  counts_out (optional): the device call's counters.
Haplotype fix_homopolymers(const Haplotype& input, const HomopolymerRegion& region, int min_flanking_sequence, Engine& engine,
                           double indel_bias = hmm_indel_bias_factor, nph_hp_counts* counts_out = nullptr);

// The AlignmentDB of annotate_variants_with_all_support: the same view of a region and its records as fix_homopolymers reads
typedef HomopolymerRegion RegionAlignments;

// annotate_variants_with_all_support (ref: src/common/nanopolish_variant.cpp:801-859): per variant, the window [ref_position -
// min_flanking_sequence, ref_position + min_flanking_sequence] of the region's reference with its ref_seq replaced by A, C, G and T
// (apply_variant, or the window where it does not apply) scored against every event sequence of the window, all variants in one
// nph_all_support_batch; then INFO gets SupportFractionByBase=a,c,g,t, each "%.3f" (std::fixed, precision 3) of the mean over the
// reads of exp(score - log-sum of the four), in input order.  Throws Error(NPH_ERR_INVALID) where the reference asserts: a window
// outside the region, a variant on another contig; also for a ref_position beyond int32 (the reference narrows the window's ends to
// int).  The variants call it with alignment_flags NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP.  counts_out (optional): the
// device call's counters.
void annotate_variants_with_all_support(std::vector<Variant>& input, const RegionAlignments& alignments, int min_flanking_sequence,
                                        uint32_t alignment_flags, Engine& engine, double indel_bias = hmm_indel_bias_factor,
                                        nph_support_counts* counts_out = nullptr);

// screen_variants_by_score (ref: src/nanopolish_call_variants.cpp:364-402) with opt::screen_flanking_sequence = flank,
// opt::screen_score_threshold = score_threshold and opt::methylation_types = methylation_types: every candidate in its own window
// [ref_position - flank, ref_position + |ref_seq| + flank], scored by score_variant_thresholded against the window's event
// sequences, all candidates in one nph_screen_variants_batch.  Returns the candidates whose quality is > 0, in input order, with
// their quality and INFO cleared; a window outside the region skips its candidate.  Like the reference, the contig of a candidate is
// not checked.  Throws Error(NPH_ERR_INVALID) for a ref_position + |ref_seq| + flank beyond int32 (the reference narrows the window's
// ends to int).  counts_out (optional): the device call's counters.
std::vector<Variant> screen_variants_by_score(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants,
                                              uint32_t alignment_flags, int flank, uint32_t score_threshold,
                                              const std::vector<std::string>& methylation_types, Engine& engine,
                                              double indel_bias = hmm_indel_bias_factor, nph_screen_list_counts* counts_out = nullptr);

// expand_variants (ref: src/nanopolish_call_variants.cpp:406-450): each candidate, then for every one that is not a single-base
// substitution its deletion extended by one reference base (only if [ref_position, ref_position + |ref_seq|] lies in the region on
// the candidate's contig and region_end - (ref_position + |ref_seq|) > min_flanking_sequence) and its four insertions alt_seq + b,
// b in ACGT.  Throws Error(NPH_ERR_INVALID) where the reference asserts: an extended deletion whose first |ref_seq| bases are not
// ref_seq.
std::vector<Variant> expand_variants(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants, int min_flanking_sequence);

// The two-sided p-value of Fisher's exact test on the 2x2 table {{n11, n12}, {n21, n22}} as simple_call's kt_fisher_exact computes
// it (ref: src/thirdparty/fet.c): 1 when the table's margins allow one table only; otherwise the probabilities of the tables from
// each end inwards while they stay below 0.99999999 times the observed table's, plus the one that stops each walk when it is below
// 1.00000001 times it, capped at 1.  Each probability is exp of log-binomials (lgamma) or, between multiples of 11, the previous
// one times the hypergeometric ratio, so the result is the reference's bit for bit.
double fisher_exact_two_sided(int n11, int n12, int n21, int n22);
// ref: src/common/nanopolish_variant.cpp:264-277 (GATK's StrandOddsRatio)
double calculate_sor(double ref_fwd, double ref_rev, double alt_fwd, double alt_rev);
// ref: src/common/nanopolish_variant.cpp:148-158: ploidy alleles, the reference ones first, '/'-separated
std::string make_genotype(size_t alt_alleles, size_t ploidy);

// call_haplotype_from_candidates (ref: src/nanopolish_call_variants.cpp:782-880) with opt::min_flanking_sequence = flank,
// opt::min_distance_between_variants = min_distance, opt::max_haplotypes, opt::ploidy, opt::genotype_only, opt::methylation_types
// and opt::calculate_all_support as given, on one OpenMP thread:
//   the groups      the candidates in the given order (unsorted lists included) while ref_position minus the previous one's is at
//                   most min_distance; window [first - flank, last + |last.ref_seq| + flank], cut from the unedited region; a window
//                   wider than 200 is not called
//   the haplotypes  variant_combinations of each group; a group with one combination is not called
//   the call        every group's scores and genotype search in one nph_call_variant_groups_batch (the reads keyed by
//                   "read_name:0" as VariantGroup keys them); then per group simple_call's output: quality best - base (0 for a
//                   variant outside the called set), INFO TotalReads, AlleleCount, SupportFraction, SupportFractionByStrand,
//                   StrandSupport, StrandFisherTest, SOR, and the genotype ("." without reads); with calculate_all_support, one
//                   annotate_variants_with_all_support over every called variant appends SupportFractionByBase
//   the result      the region's haplotype with every group's called variants applied in order (apply_variant's refusals ignored)
// Throws Error(NPH_ERR_INVALID) where the reference asserts (a window outside the region, a called group with fewer combinations
// than the ploidy) and for a ref_position beyond int32.  counts_out (optional): the device call's counters.
Haplotype call_haplotype_from_candidates(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants,
                                         uint32_t alignment_flags, int flank, int min_distance, int max_haplotypes, int ploidy,
                                         bool genotype_only, const std::vector<std::string>& methylation_types, bool calculate_all_support,
                                         Engine& engine, double indel_bias = hmm_indel_bias_factor, nph_call_counts* counts_out = nullptr);

// std::stringstream << v with the stream's defaults (precision 6: 0.333333, 1, 5e-05), as the reference's Variant::add_info writes a double
std::string format_double(double v);

// AlignmentDB::get_variants_in_region(contig, start, stop, min_frequency, min_depth) (ref: src/alignment/nanopolish_alignment_db.cpp:
// 259-368) over alignments.sequence_records: the pile-up and merge in one nph_region_candidates_batch, then the reference's order on the
// host: the distinct variants in std::map order of their keys "contig:pos:ref:alt" (bytewise: "1000:..." < "100:..."), kept when
// (double)count / depth >= min_frequency && depth >= min_depth, INFO BaseCalledReadsWithVariant=count;BaseCalledFraction=f
// (format_double), then std::sort by position (not stable: the order among variants at one position is std::sort's, which reaches
// the VCF through call_haplotype_from_candidates' grouping).  Throws Error(NPH_ERR_INVALID) for stop < start, [start, stop] outside
// the region, a record whose pairs do not strictly increase or leave its bases; Error(NPH_ERR_UNSUPPORTED) for a read-position step
// beyond int16 (an insertion of more than 32 767 bases).  counts_out (optional): the device call's counters.
std::vector<Variant> get_variants_in_region(const RegionAlignments& alignments, int start, int stop, double min_frequency, int min_depth,
                                            Engine& engine, nph_candidate_counts* counts_out = nullptr);

// read_variants_for_region (ref: src/common/nanopolish_variant.cpp:81-108): the VCF lines of `text` (headers skipped) parsed as
// Variant::read_vcf parses them, kept when on `contig` with (int)ref_position in [region_start, region_end], INFO cleared.  Throws
// Error(NPH_ERR_INVALID) where read_vcf asserts: an empty contig, REF or ALT, a negative quality (an empty line included).
std::vector<Variant> read_variants_for_region(const std::string& text, const std::string& contig, int region_start, int region_end);

// The options of `nanopolish variants` that its default (non-consensus) mode reads, with the reference's defaults
// (ref: src/nanopolish_call_variants.cpp:115-140).  min_candidate_frequency is the float literal 0.2f widened to double.
struct CallVariantsOptions {
    int min_flanking_sequence = 30;
    int min_distance_between_variants = 10;
    int max_haplotypes = 1000;
    int ploidy = 0;                             // -p: required by the reference
    bool genotype_only = false;
    bool calculate_all_support = false;
    bool snps_only = false;
    double min_candidate_frequency = 0.2f;
    int min_candidate_depth = 20;
    std::vector<std::string> methylation_types;
    bool use_candidates = false;                // --candidates: candidates_vcf holds the file's text
    std::string candidates_vcf;
};

// call_variants_for_region (ref: src/nanopolish_call_variants.cpp:882-1011) in its default mode, with main's window checks
// (:1131-1170): start_base and end_base as main has them (end clamped to contig_length - 1).  BUFFER = min_flanking_sequence + 10,
// region_start = max(start_base, BUFFER); `alignments` is the region loaded over [region_start - BUFFER, min(end_base + BUFFER,
// contig_length - 1)], region_end = its last base - BUFFER.  Candidates: get_variants_in_region(region_start, region_end,
// min_candidate_frequency, min_candidate_depth), or read_variants_for_region over candidates_vcf; then call_haplotype_from_candidates
// with NPH_HAF_ALLOW_PRE_CLIP | NPH_HAF_ALLOW_POST_CLIP.  Throws Error(NPH_ERR_INVALID) for start_base > end_base, contig_length -
// start_base < 40, and a region not loaded at region_start - BUFFER.
Haplotype call_variants_for_region(const RegionAlignments& alignments, int start_base, int end_base, int contig_length,
                                   const CallVariantsOptions& options, Engine& engine, double indel_bias = hmm_indel_bias_factor);

// The VCF call_variants_main writes (ref: src/nanopolish_call_variants.cpp:1172-1278): the header (##fileformat, ##nanopolish_window=
// contig:start_base-end_base, the INFO and FORMAT tag lines in the reference's order, SupportFractionByBase only with
// calculate_all_support, the #CHROM line), then per variant of `called` (SNPs only with snps_only) INFO RefContext = the reference
// over [max(pos - 5, 0), min(pos + |ref| + 4, contig_length - 1)], taken from `alignments`, and Variant::write_vcf's line.  Throws
// Error(NPH_ERR_INVALID) for a context outside the loaded region.
std::string write_variants_vcf(const RegionAlignments& alignments, int start_base, int end_base, int contig_length,
                               const CallVariantsOptions& options, const Haplotype& called);

} // namespace nph
