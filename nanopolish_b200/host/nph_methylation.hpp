// nph_methylation.hpp — SURVEY.md section 8(f) row N3: call-methylation's per-read logic split into
// staging / one batched launch / scatter, plus the TSV writer.
//
//   calculate_methylation_for_read      ref: src/basemods/nanopolish_basemods.cpp:238-457
//   ScoredSite, MethylationCallingParameters   ref: src/basemods/nanopolish_basemods.h:45-77
//   AlignmentDB::_find_by_ref_bounds    ref: src/alignment/nanopolish_alignment_db.cpp:688-731
//   write_methylation_results_as_tsv    ref: src/nanopolish_call_methylation.cpp:532-550
//   create_modbam_record / create_reference_modbam_record (the Mm / Ml tags of --modbam-output)
//                                       ref: src/basemods/nanopolish_basemods.cpp:35-177, 179-238
//
// The reference scores two sequences per CpG group with two profile_hmm_score calls inside the per-read OpenMP
// loop.  Here add_read() only stages what the reference pulls out of the BAM record and the FASTA — the reference
// substring and the (ref_pos, event_idx) pairs of EventAlignmentRecord (src/alignment/nanopolish_alignment_db.cpp:50-91)
// — into page-locked buffers; run() hands the whole BamProcessor batch to nph_methylation_batch, where the motif scan,
// the grouping, the window / event-bound tests, the methylated / unmethylated k-mer ranks and the two scores per group
// all happen on the device (csrc/methylation.cu); what comes back is one 24-byte record per scored group, from which
// the ScoredSites and the TSV rows (write_methylation_results_as_tsv) are formed.
#pragma once
#include <cstdio>
#include "nph_host.hpp"

namespace nph {

struct ScoredSite {
    ScoredSite() { ll_unmethylated[0] = ll_unmethylated[1] = ll_methylated[0] = ll_methylated[1] = 0; strands_scored = 0; }
    std::string chromosome;
    int start_position = 0;
    int end_position = 0;
    int n_motif = 0;
    std::string sequence;
    double ll_unmethylated[2];
    double ll_methylated[2];
    int strands_scored;
};

struct MethylationCallingParameters {
    int min_separation = 10;
    int min_flank = 10;
    std::string methylation_type = "cpg";
    const Alphabet* alphabet = nullptr;      // get_alphabet_by_name(methylation_type)
};

// What the reference derives from the BAM record, the FASTA and the SquiggleRead before the group loop.
struct EventAlignedRead {
    SquiggleRead* read = nullptr;
    std::string read_name;                   // bam_get_qname
    bool is_reverse = false;                 // bam_is_rev: the "+"/"-" column
    std::string contig;
    int ref_start_pos = 0;                   // record->core.pos
    std::string ref_seq;                     // reference over [ref_start_pos, bam_endpos], already gDNAAlphabet.disambiguate()d
    // per strand: EventAlignmentRecord::aligned_events (ref_pos ascending, read_pos = event index) and ::rc
    std::vector<AlignedPair> aligned_events[2];
    bool rc[2] = {false, false};
};

// The compact event alignment of one record (include/nph.h, nph_methylation_batch_compact): deltas[0, ref_len) and *first_event from
// aligned_events over a reference substring starting at ref_start_pos.  false: a reference position outside the substring or out of
// order, or an event-index step beyond int16 (the caller then needs the pair form).
bool compact_event_alignment(const std::vector<AlignedPair>& aligned_events, int ref_start_pos, size_t ref_len, int16_t* deltas, int32_t* first_event);

// ---- modBAM tags (SAM specification: Mm = delta-encoded positions of the modified base, Ml = probabilities 0..255) ----
struct ModbamTags {
    std::string mm;                // e.g. "C+m?,3,0,12;"
    std::vector<uint8_t> ml;       // one entry per position listed in mm
};
// the unmodified base that the alphabet's methylated symbol replaces ('C' for cpg); the reference asserts one recognition site
char unmodified_symbol_of(const Alphabet* alphabet);
// reference position and probability code of every called site (strand-0 likelihoods, like the reference)
void calculate_call_vectors(const std::map<int, ScoredSite>& calls, const Alphabet* alphabet,
                            std::vector<size_t>& call_reference_positions, std::vector<uint8_t>& call_probabilities);
std::string generate_mm_tag(char unmodified_symbol, const std::string& sequence, const std::vector<size_t>& call_seq_indices);
// create_modbam_record: tags for the read's own BAM record.  bam_seq = SEQ as stored (reference orientation),
// aligned_bases = get_aligned_segments(record)[0] (nph_eventalign.hpp), is_reverse = bam_is_rev(record).
ModbamTags modbam_tags(const std::string& bam_seq, const std::vector<AlignedPair>& aligned_bases, bool is_reverse,
                       const std::map<int, ScoredSite>& calls, const MethylationCallingParameters& params);
// create_reference_modbam_record: tags against the (disambiguated) reference over the record's span
ModbamTags reference_modbam_tags(const std::string& ref_seq, int ref_start_pos, const std::map<int, ScoredSite>& calls,
                                 const MethylationCallingParameters& params);

// nph_meth_params (include/nph.h) for these calling parameters, model k-mer size and output window
nph_meth_params make_meth_params(const MethylationCallingParameters& params, uint32_t k, int region_start, int region_end);

// page-locked, growable host array (nph_host_alloc): what the batch hands to the C ABI is written once, in place
template <typename T>
class PinnedArray {
public:
    PinnedArray() {}
    ~PinnedArray() { if (m_p) nph_host_free(m_p); }
    PinnedArray(const PinnedArray&) = delete;
    PinnedArray& operator=(const PinnedArray&) = delete;
    T* data() { return m_p; }
    const T* data() const { return m_p; }
    size_t size() const { return m_n; }
    void clear() { m_n = 0; }
    void resize(size_t n);             // keeps the first min(n, size()) elements; new elements are uninitialised
private:
    T* m_p = nullptr;
    size_t m_n = 0, m_cap = 0;
};

// A BamProcessor batch in the flat layout nph_methylation_batch takes (one record = one read, one strand), plus what the
// TSV rows need per record.  records[].read / .model_id are already resolved (nph_read index, Engine::model_id).
struct FlatMethylationBatch {
    const nph_read* reads = nullptr; size_t n_reads = 0;
    const float* ev_mean = nullptr; const double* ev_start_time = nullptr; size_t n_events = 0;
    const char* ref_bases = nullptr; size_t n_ref = 0;
    const nph_aligned_pair* aligned_events = nullptr; size_t n_pairs = 0;
    // or the compact form (include/nph.h, nph_methylation_batch_compact): int16 event-index deltas parallel to ref_bases + the first
    // event index of every record; used instead of aligned_events when event_deltas != nullptr
    const int16_t* event_deltas = nullptr; const int32_t* first_event = nullptr;
    const nph_meth_record* records = nullptr; size_t n_records = 0;
    const char* const* read_names = nullptr;      // per record
    const uint8_t* is_reverse = nullptr;          // per record: bam_is_rev
    const char* contig = nullptr;
    int region_start = -1, region_end = -1;
};
struct FlatMethylationStats { uint64_t n_sites = 0, scored_events = 0; double device_seconds = 0, tsv_seconds = 0; };
// returns the TSV's byte count (rows are written only if it fits cap)
size_t call_methylation_flat(Engine& engine, const FlatMethylationBatch& batch, const MethylationCallingParameters& params, uint32_t k,
                             double indel_bias, char* tsv_out, size_t cap, FlatMethylationStats* stats = nullptr);

class MethylationCaller {
public:
    explicit MethylationCaller(const MethylationCallingParameters& params);
    // stage the read's reference substring and event alignments for run(); returns the read's index in this batch.
    // region_start/region_end = -1 for no window restriction (the reference's -w option).
    size_t add_read(const EventAlignedRead& r, int region_start = -1, int region_end = -1);
    // The same for a whole BamProcessor batch, staged by host_threads() workers.  Returns the index of the first read.
    size_t add_reads(const std::vector<EventAlignedRead>& reads, int region_start = -1, int region_end = -1);
    void run(Engine& engine, double indel_bias = hmm_indel_bias_factor);       // one device call for every staged read
    const std::map<int, ScoredSite>& sites(size_t read_idx) const;            // (built from the site records on first use)
    size_t num_reads() const { return m_reads.size(); }
    // forward jobs scored by the last run(): two per group
    size_t num_jobs() const { return (size_t)(2 * m_n_sites); }
    uint64_t scored_events() const { return m_scored_events; }                // after run()
    // every read's rows back to back in one buffer (formatted straight from the site records by host_threads() workers);
    // returns the byte count, or the required size when cap is too small
    size_t tsv_all(char* out, size_t cap) const;
    void write_tsv(FILE* fp, size_t read_idx) const;
    std::string tsv(size_t read_idx) const;
    std::vector<std::string> tsv_batch() const;            // every read's rows, formatted by host_threads() workers
    // the Mm / Ml tags of --modbam-output for one read of the batch (after run()): bam_seq and aligned_bases as in
    // nph::modbam_tags
    ModbamTags modbam(size_t read_idx, const std::string& bam_seq, const std::vector<AlignedPair>& aligned_bases) const
    {
        return modbam_tags(bam_seq, aligned_bases, m_reads[read_idx].is_reverse, sites(read_idx), m_params);
    }
    void clear();

private:
    struct ReadEntry {
        std::string name; bool is_reverse = false;
        mutable std::map<int, ScoredSite> sites; mutable bool sites_built = false;
        std::string contig; size_t ref_off = 0, ref_len = 0; int ref_start_pos = 0; uint32_t k = 0;
        size_t first_record = 0, n_records = 0;
    };
    struct Record { const SquiggleRead* read; const PoreModel* model; uint8_t strand; };
    void stage(const EventAlignedRead* const* reads, size_t n, int region_start, int region_end);
    void build_sites(size_t read_idx) const;
    void append_rows(std::string& out, size_t read_idx) const;
    void put_rows(void* row_buffer, size_t read_idx) const;          // the same into the writer's growing character buffer
    MethylationCallingParameters m_params;
    std::vector<ReadEntry> m_reads;
    // the flat batch (page-locked) and its results
    PinnedArray<char> m_ref;
    PinnedArray<nph_aligned_pair> m_pairs;
    PinnedArray<int16_t> m_deltas;            // compact event alignments, parallel to m_ref (built next to m_pairs; used unless a step overflowed)
    std::vector<int32_t> m_first_event;
    bool m_compact_ok = true;
    PinnedArray<nph_meth_site> m_sites;
    std::vector<nph_meth_record> m_records;
    std::vector<Record> m_record_meta;
    std::vector<uint64_t> m_site_off;
    uint64_t m_n_sites = 0, m_scored_events = 0;
    int m_region_start = -1, m_region_end = -1;
    bool m_region_set = false, m_ran = false;
};

} // namespace nph
