// nph_polya.hpp — nanopolish polya (src/nanopolish_polya_estimator.cpp) as a batch call: estimate_polya_for_single_read
// (:733-862) for every record of a BamProcessor batch, the numeric part in ONE device call (nph_polya_batch), the TSV of
// polya_main (:877 header, :765-766 and :823-826 rows) written on the host with the reference's format strings.
//
// Per record the host does what the reference does before the numbers: secondary alignments (BAM_FSECONDARY) produce no
// row (:743-745); the suffix clip is the length of the record's LAST CIGAR operation, whatever its type (:753-758); a read
// missing from the index or whose events load_from_raw cleared (:761-762) gives the READ_FAILED_LOAD row.  The samples are
// the read's WHOLE raw signal (SquiggleRead::samples with SRF_LOAD_RAW_SAMPLES, squiggle_read.cpp:251-258): RawRead::samples.
// The verbose modes (per-sample and per-k-mer dumps) are not provided.
//
// DetectPolyiBatch is nanopolish detect-polyi (src/nanopolish_detect_polyi.cpp) the same way: dpi_estimate_polya_for_single_read
// (:1008-1144) for every record, with the same per-record rules (:1018-1052) and one nph_detect_polyi_batch call, and
// detect_polyi_main's TSV (:1159 header, :1040-1041 and :1105-1108 rows).  Its verbose modes (-v: the per-sample and per-k-mer
// dumps) are not provided either.
#pragma once
#include "nph_raw.hpp"

namespace nph {

constexpr uint16_t BAM_FSECONDARY = 0x100;     // htslib sam.h

// What estimate_polya_for_single_read reads of one BAM record and its read.
struct PolyaRecord {
    std::string read_name;                // bam_get_qname
    std::string contig;                   // hdr->target_name[core.tid]
    int32_t pos = 0;                      // core.pos
    uint16_t flag = 0;                    // core.flag
    std::vector<uint32_t> cigar;          // bam_get_cigar words (op | len << 4); must not be empty
    const SquiggleRead* read = nullptr;   // nullptr: not in the read index
    const RawRead* raw = nullptr;         // the read's whole raw signal and sample rate (required when read is set)
};

// One tail caller over a batch of records.  Result selects the caller: nph_polya_result is polya (nph_polya_batch,
// polya_main's TSV), nph_polyi_result is detect-polyi (nph_detect_polyi_batch, detect_polyi_main's TSV).
template <class Result>
class TailBatch {
public:
    // Adds a record; returns false (no row) for a secondary alignment.  Throws Error(NPH_ERR_INVALID) for a record without a
    // CIGAR (the reference reads cigar[n_cigar - 1]).
    bool add(const PolyaRecord& rec);
    // One device call over the records added since the last run; their results replace the previous ones.
    void run(Engine& engine);
    const std::vector<Result>& results() const { return m_results; }
    // The rows of the last run in record order, preceded by the caller's header line if header is set.
    std::string tsv(bool header = true) const;
    void clear();

private:
    std::vector<PolyaRecord> m_records;
    std::vector<Result> m_results;
    std::vector<PolyaRecord> m_done;      // the records m_results belong to
};

using PolyaBatch = TailBatch<nph_polya_result>;
using DetectPolyiBatch = TailBatch<nph_polyi_result>;

} // namespace nph
