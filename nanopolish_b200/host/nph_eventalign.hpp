// nph_eventalign.hpp — SURVEY.md section 8(f) row N1, host half: eventalign's per-read segment chaining around the
// Viterbi kernel, and its writers.
//
//   HMMAlignmentState, profile_hmm_align      ref: src/common/nanopolish_common.h:65-73, src/hmm/nanopolish_profile_hmm.h:27-28
//   EventAlignment, EventAlignmentParameters  ref: src/alignment/nanopolish_eventalign.h:21-71
//   align_read_to_ref                         ref: src/alignment/nanopolish_eventalign.cpp:612-827
//   get_aligned_segments                      ref: src/alignment/nanopolish_anchor.cpp:20-87
//   trim_aligned_pairs_to_kmer / _to_ref_region / get_end_pair   ref: src/alignment/nanopolish_eventalign.cpp:166-207
//   emit_event_alignment_tsv / emit_tsv_header                   ref: :227-244, :398-484
//   event_alignment_to_cigar / emit_event_alignment_sam          ref: :256-325, :327-396
//   summarize_alignment + the summary row                        ref: :486-537, :600-607
//
// The reference walks a read in ~100-base reference windows: each profile_hmm_align call starts at the event where
// the previous window's output stopped, so the windows of ONE read are sequential, while different reads are
// independent (its OpenMP loop is over reads).  EventAligner::run hands every (read, BAM segment) chain to the chain
// kernel (nph_eventalign_chain: one warp walks one chain start to end on the device, ONE launch per batch of reads)
// and gets back 12-byte records; the strings of an EventAlignment are only built when a writer or alignment() asks.
// run_rounds() is the same computation driven from the host — one cursor per read, a round collects the next window
// of every unfinished read into one AlignBatch (one Viterbi launch, events resident in HBM since the first round) —
// kept for windows the chain kernel's scratch cannot hold and as the cross-check of the device cursor logic.
//
// BAM/FASTA access stays with the caller, which hands over what the reference pulls out of the record and the index:
// position, flag, mapping quality, the packed CIGAR and the reference substring.
#pragma once
#include <cstdio>
#include "nph_host.hpp"

namespace nph {

struct HMMAlignmentState {
    uint32_t event_idx;
    uint32_t kmer_idx;
    double l_posterior;                  // -INFINITY: "not computed", as in the reference (profile_hmm_r9.cpp:139-141)
    double l_fm;
    double log_transition_probability;   // -INFINITY
    char state;                          // 'M', 'B' (bad event), 'K' (k-mer skip)
};

// A batch of profile_hmm_align calls.  The read table survives clear_jobs() so that consecutive rounds over the same
// reads can leave the events resident on the device (run(..., reads_resident = true)).
class AlignBatch {
public:
    size_t add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags = 0);
    size_t size() const { return m_jobs.size(); }
    void clear_jobs();
    void clear();
    // reads_resident: the previous run() of THIS batch on THIS engine uploaded the same read table and nothing else
    // has used the engine since; skips the upload.  New reads added since then force an upload.
    std::vector<std::vector<HMMAlignmentState>> run(Engine& engine, double indel_bias = hmm_indel_bias_factor, bool reads_resident = false);
    // the flat job list, for callers that drive the rounds themselves
    const std::vector<nph_hmm_job>& jobs() const { return m_jobs; }
    const std::vector<uint32_t>& ranks() const { return m_ranks; }
    const SquiggleRead* job_read(size_t j) const { return m_reads.reads()[m_jobs[j].read].first; }

private:
    detail::ReadTable m_reads;
    std::vector<const PoreModel*> m_job_models;
    std::vector<nph_hmm_job> m_jobs;
    std::vector<uint32_t> m_ranks;
    size_t m_reads_uploaded = 0;
};

std::vector<HMMAlignmentState> profile_hmm_align(const HMMInputSequence& sequence, const HMMInputData& data, const uint32_t flags = 0);

// ---------------------------------------------------------------------------------------------
// eventalign
// ---------------------------------------------------------------------------------------------
typedef std::vector<AlignedPair> AlignedSegment;

enum { NPH_BAM_FUNMAP = 4, NPH_BAM_FREVERSE = 16 };
// packed BAM CIGAR operations (len << 4 | op), op codes of the SAM specification
enum { NPH_CIGAR_M = 0, NPH_CIGAR_I = 1, NPH_CIGAR_D = 2, NPH_CIGAR_N = 3, NPH_CIGAR_S = 4, NPH_CIGAR_H = 5, NPH_CIGAR_P = 6, NPH_CIGAR_EQ = 7, NPH_CIGAR_X = 8 };

std::vector<AlignedSegment> get_aligned_segments(int ref_pos, const std::vector<uint32_t>& cigar, int read_stride = 1);
void trim_aligned_pairs_to_kmer(std::vector<AlignedPair>& aligned_pairs, int max_kmer_idx);
void trim_aligned_pairs_to_ref_region(std::vector<AlignedPair>& aligned_pairs, int ref_start, int ref_end);
int get_end_pair(const std::vector<AlignedPair>& aligned_pairs, int ref_pos_max, int pair_idx);

struct EventAlignmentParameters {
    SquiggleRead* sr = nullptr;
    size_t strand_idx = 0;
    // from the BAM record and header
    std::string ref_name;                // hdr->target_name[record->core.tid]
    int ref_pos = 0;                     // record->core.pos
    uint16_t flag = 0;                   // record->core.flag (unmapped, reverse)
    uint8_t mapq = 0;                    // record->core.qual (SAM output only)
    int edit_distance = 0;               // the NM tag (summary only)
    std::vector<uint32_t> cigar;
    // from the FASTA index: the reference over [ref_pos, bam_endpos(record)], as faidx_fetch_seq returns it
    std::string ref_seq;
    // optional
    std::string alphabet;                // "" = the read's base model
    int read_idx = -1;
    int region_start = -1, region_end = -1;

    const PoreModel* get_model() const { return alphabet.empty() ? sr->get_base_model((uint32_t)strand_idx) : sr->get_model((uint32_t)strand_idx, alphabet); }
};

struct EventAlignment {
    std::string ref_name;
    std::string ref_kmer;
    int ref_position = 0;
    size_t read_idx = 0;
    int strand_idx = 0;
    int event_idx = 0;
    bool rc = false;
    std::string model_kmer;
    char hmm_state = 0;
};

struct EventalignSummary {
    int num_events = 0, num_steps = 0, num_stays = 0, num_skips = 0;
    double sum_duration = 0, sum_z_score = 0;
    int alignment_edit_distance = 0, reference_span = 0;
};

struct EventalignOptions {               // the reference's command-line switches that change the output
    bool print_read_names = false;       // -n
    bool scale_events = false;           // --scale-events
    bool write_signal_index = false;     // --signal-index: the event's [start, end) raw sample indices
    bool write_samples = false;          // --samples: the event's scaled raw samples (both need SquiggleRead::samples)
};

// What run_tsv returns: the rows of every queued read in one buffer, read i's at [read_off[i], read_off[i + 1]).  When the device
// wrote every read the bytes are the engine's page-locked staging and stay valid until the next run_tsv on that engine.
class EventalignTsv {
public:
    const char* data() const { return m_view ? m_view : m_owned.data(); }
    size_t size() const { return m_size; }
    std::vector<uint64_t> read_off;      // num_reads() + 1
    std::vector<uint8_t> on_host;        // per read: 1 = formatted by tsv() (refused by the device writer, or aligned by run_rounds)
    size_t batches = 0;                  // kernel batches issued, as run() counts them

private:
    friend class EventAligner;
    const char* m_view = nullptr;
    size_t m_size = 0;
    std::string m_owned;
};

class EventAligner {
public:
    // queue one read strand; returns its index in this batch
    size_t add_read(const EventAlignmentParameters& params);
    size_t num_reads() const { return m_reads.size(); }

    // Align every queued read: one launch of the chain kernel; reads with a window too large for its scratch are
    // re-run through run_rounds().  Returns the number of kernel batches issued (1 + fallback rounds).
    size_t run(Engine& engine, double indel_bias = hmm_indel_bias_factor);
    // run() with the TSV rows written on the device (nph_eventalign_tsv) from the records where the chain kernel left them: the
    // bytes of tsv_batch(opt) joined, without the records crossing PCIe.  Reads the device writer refuses and reads re-run
    // through run_rounds() take tsv().  Afterwards alignment(), sam(), summarize() and tsv() fetch the records on first use,
    // which must come before the engine runs another alignment.  Throws what tsv() throws for a read without raw samples.
    EventalignTsv run_tsv(Engine& engine, double indel_bias = hmm_indel_bias_factor, const EventalignOptions& opt = EventalignOptions());
    // The host-driven form: rounds of (collect next windows -> one Viterbi launch -> advance cursors) until no read has a
    // window left.  Returns the number of rounds (= the longest read's window count).
    size_t run_rounds(Engine& engine, double indel_bias = hmm_indel_bias_factor);

    // The two halves of a round, for callers that want to interleave their own work (and for the host-logic tests):
    // next_round() fills `batch` with one job per unfinished read (false = all reads are done); consume() takes the
    // paths of exactly those jobs, in order.
    bool next_round(AlignBatch& batch);
    void consume(const std::vector<std::vector<HMMAlignmentState>>& paths);
    const std::vector<size_t>& round_reads() const { return m_round; }     // read index of each job of the open round

    std::vector<EventAlignment> alignment(size_t read_idx) const;          // materialised from the compact records
    size_t num_alignments(size_t read_idx) const { ensure_records(); return m_reads[read_idx].output.size(); }
    size_t num_segments(size_t read_idx) const { ensure_records(); return m_reads[read_idx].segments_aligned; }   // profile_hmm_align calls made

    static std::string tsv_header(const EventalignOptions& opt = EventalignOptions());
    std::string tsv(size_t read_idx, const EventalignOptions& opt = EventalignOptions()) const;
    std::vector<std::string> tsv_batch(const EventalignOptions& opt = EventalignOptions()) const;   // all reads, formatted in parallel
    // one SAM text line (the reference writes the same record through htslib), "" for an empty alignment
    std::string sam(size_t read_idx) const;
    std::string event_cigar(size_t read_idx) const;
    EventalignSummary summarize(size_t read_idx) const;
    // the row of --summary; "" when the alignment is empty (the reference skips those)
    std::string summary_row(size_t read_idx, const std::string& fast5_path = "") const;
    void clear();

private:
    struct Rec { int ref_position; int event_idx; char state; };    // an EventAlignment without its strings
    struct SegmentStart { int first_event, last_event, start_ref; };
    struct ReadState {
        EventAlignmentParameters params;
        const PoreModel* pore_model = nullptr;
        uint32_t k = 0;
        std::string ref_seq, rc_ref_seq;          // upper-cased, disambiguated
        std::vector<AlignedSegment> segments;
        bool do_base_rc = false;
        // cursor
        size_t segment_idx = 0;
        bool in_segment = false, done = false;
        int last_event = 0;
        bool forward = true;
        int curr_start_event = 0, curr_start_ref = 0, curr_pair_idx = 0;
        // the job issued this round
        bool pending = false;
        int end_pair_idx = 0;
        uint8_t job_rc = 0;
        std::string fwd_subseq, rc_subseq;
        // results
        std::vector<Rec> output;
        size_t segments_aligned = 0;
    };
    bool prepare(ReadState& rs, AlignBatch& batch);      // true if a job was queued
    bool enter_segment(ReadState& rs);                    // false = the whole read is finished
    bool setup_segment(ReadState& rs, size_t segment_idx, SegmentStart& out);   // trims + start/stop events; false = no pairs left
    EventAlignment materialize(const ReadState& rs, const Rec& r) const;
    static void kmers_at(const ReadState& rs, const Rec& r, char* ref_kmer, char* model_kmer);   // NUL-terminated, k+1 bytes each
    static void require_samples(const SquiggleRead& sr, const EventalignOptions& opt);
    size_t run_device(Engine& engine, double indel_bias, const EventalignOptions* tsv_opt, EventalignTsv* tsv_out);
    void scatter(const nph_ea_record* records, const std::vector<nph_ea_chain>& chains, const std::vector<nph_ea_result>& results,
                 const std::vector<uint64_t>& chain_first, const std::vector<char>& skip);
    const char* device_tsv(Engine& engine, const EventalignOptions& opt, const std::vector<uint64_t>& chain_first, const std::vector<size_t>& owner,
                           std::vector<uint64_t>& read_off, std::vector<uint8_t>& refused);
    // after run_tsv: the chain run whose records are still on the device
    struct Lazy {
        Engine* engine = nullptr;
        uint64_t records_total = 0;
        std::vector<nph_ea_chain> chains;
        std::vector<nph_ea_result> results;
        std::vector<uint64_t> chain_first;
    };
    void ensure_records() const;
    Lazy m_lazy;
    std::vector<ReadState> m_reads;
    std::vector<size_t> m_round;                          // reads with a pending job, in job order
    AlignBatch m_batch;
};

std::vector<uint32_t> event_alignment_to_cigar(const std::vector<EventAlignment>& alignments);
// (format_fixed, the exact %.Nlf replacement the writers use, and kmer_ranks, the rolling pass that builds the chains' rank
// tables, live in nph_host.hpp)
std::string cigar_ops_to_string(const std::vector<uint32_t>& ops);

} // namespace nph
