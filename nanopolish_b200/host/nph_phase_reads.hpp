// nph_phase_reads.hpp — `nanopolish phase-reads` (phase_single_read, ref: src/nanopolish_phase_reads.cpp:178-347) split into
// staging / one device call / SAM records.
//
// add_read() applies the reference's record-level rules — no record when lower_bound(variants, {contig, pos}) is the end of the
// list or the read has no events on strand 0; a record (the plain reference, every quality 30) when the range is merely empty —
// and stages the fetched reference and the strand-0 event alignment in the compact form MethylationCaller uses.  run() hands the
// batch to nph_phase_reads_batch; sam() writes the records the reference writes with sam_write1, in add order.
// VCF parsing, -w, threads and BAM output stay with the caller: the variant list comes sorted by position (sortByPosition) with
// the 0/0 genotypes removed, as phase_reads_main builds it.
#pragma once
#include "nph_host.hpp"
#include "nph_methylation.hpp"
#include "nph_variants.hpp"

namespace nph {

class PhaseReads {
public:
    explicit PhaseReads(const std::vector<Variant>& sorted_variants);
    // r: strand 0 of the read with its aligned_events and rc, ref_seq = the reference over [ref_start_pos, bam_endpos] through
    // std::toupper (not disambiguated).  Returns whether the read writes a SAM record.
    bool add_read(const EventAlignedRead& r, uint16_t flag, uint8_t mapq);
    void run(Engine& engine, double indel_bias = hmm_indel_bias_factor);     // one device call for every staged record
    std::vector<std::string> sam() const;                                    // one SAM line per record, in add order (after run())
    const std::vector<nph_phase_call>& calls() const { return m_calls; }
    size_t num_records() const { return m_entries.size(); }
    void clear();

private:
    struct Entry { std::string name, contig; uint16_t flag; uint8_t mapq; const SquiggleRead* read; const PoreModel* model; };
    std::vector<Variant> m_variants;
    std::vector<nph_phase_variant> m_dev_variants;
    std::vector<Entry> m_entries;
    std::vector<char> m_ref;
    std::vector<int16_t> m_deltas;
    std::vector<int32_t> m_first_event;
    std::vector<nph_meth_record> m_records;
    std::vector<uint32_t> m_range;
    std::vector<uint64_t> m_call_off;
    std::vector<nph_phase_call> m_calls;
    bool m_ran = false;
};

} // namespace nph
