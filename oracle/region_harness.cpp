// region_harness.cpp — TEST INFRASTRUCTURE ONLY.  The default (non-consensus) mode of `nanopolish variants` on one region, from the
// reference's own functions: AlignmentDB::get_variants_in_region (src/alignment/nanopolish_alignment_db.cpp:259-368) over a hand-built
// AlignmentDB whose base-space records (m_sequence_records) are built in place, read_variants_for_region
// (src/common/nanopolish_variant.cpp:81-108), call_haplotype_from_candidates through npref_call_haplotype (call_harness.cpp, which
// compiles src/nanopolish_call_variants.cpp in place and is linked into the same library), and the header and records
// call_variants_main writes (src/nanopolish_call_variants.cpp:1172-1278) through Variant::write_vcf_header and Variant::write_vcf into a
// memory FILE*, RefContext taken from the loaded region.  Nothing of the reference is copied.
#include "nanopolish_alignment_db.h"
#include "nanopolish_profile_hmm.h"
#include "nanopolish_variant.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <sstream>
#include <string>
#include <unistd.h>
#include <vector>

extern "C" long long npref_call_haplotype(const char* contig, int region_start, int region_end, const char* region_ref, int n_records,
                                          const int32_t* read_h, const char** read_names, const uint8_t* rc, const int8_t* stride,
                                          const uint64_t* pair_off, const uint32_t* n_pairs, const int32_t* pairs, int n_variants,
                                          const int32_t* var_pos, const char** var_ref, const char** var_alt, int flank, int min_distance,
                                          int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support,
                                          uint32_t alignment_flags, char* out, size_t cap);   // call_harness.cpp

namespace {

// pointer-to-member of a private member, through an explicit instantiation
template <typename Tag, typename Tag::type M>
struct Expose { friend typename Tag::type member(Tag) { return M; } };
#define NPREF_EXPOSE(TAG, TYPE, NAME)                                          \
    struct TAG { typedef TYPE AlignmentDB::*type; friend type member(TAG); };  \
    template struct Expose<TAG, &AlignmentDB::NAME>;
NPREF_EXPOSE(RgContig, std::string, m_region_contig)
NPREF_EXPOSE(RgStart, int, m_region_start)
NPREF_EXPOSE(RgEnd, int, m_region_end)
NPREF_EXPOSE(RgRef, std::string, m_region_ref_sequence)
NPREF_EXPOSE(RgSeqRecords, std::vector<SequenceAlignmentRecord>, m_sequence_records)

// the AlignmentDB of one call with its base-space records only, built in place and torn down by its destructor
struct SeqDbInPlace {
    alignas(AlignmentDB) unsigned char storage[sizeof(AlignmentDB)];
    AlignmentDB* db;
    std::string* contig;
    std::string* ref;
    std::vector<SequenceAlignmentRecord>* seq_records;
    // base-space record r: bases seq_bases[r], strand seq_rc[r], aligned_bases seq_pairs[2 * seq_pair_off[r] ..) up to
    // seq_pair_off[r + 1] (SequenceAlignmentRecord has no constructor but the one from a bam1_t: its members are built in place)
    SeqDbInPlace(const char* c, int region_start, int region_end, const char* region_ref, int n_seq, const char** seq_bases,
                 const uint8_t* seq_rc, const int32_t* seq_pairs, const uint64_t* seq_pair_off)
    {
        db = reinterpret_cast<AlignmentDB*>(storage);
        contig = new (&(db->*member(RgContig()))) std::string(c);
        ref = new (&(db->*member(RgRef()))) std::string(region_ref);
        seq_records = new (&(db->*member(RgSeqRecords()))) std::vector<SequenceAlignmentRecord>();
        db->*member(RgStart()) = region_start;
        db->*member(RgEnd()) = region_end;
        for (int r = 0; r < n_seq; ++r) {
            alignas(SequenceAlignmentRecord) unsigned char raw[sizeof(SequenceAlignmentRecord)];
            SequenceAlignmentRecord* sr = reinterpret_cast<SequenceAlignmentRecord*>(raw);
            new (&sr->read_name) std::string("seq" + std::to_string(r));
            new (&sr->sequence) std::string(seq_bases[r]);
            new (&sr->aligned_bases) std::vector<AlignedPair>();
            sr->rc = seq_rc[r];
            for (uint64_t i = seq_pair_off[r]; i < seq_pair_off[r + 1]; ++i) {
                AlignedPair ap;
                ap.ref_pos = seq_pairs[2 * i]; ap.read_pos = seq_pairs[2 * i + 1];
                sr->aligned_bases.push_back(ap);
            }
            seq_records->push_back(*sr);
            sr->aligned_bases.~vector(); sr->sequence.~basic_string(); sr->read_name.~basic_string();
        }
    }
    ~SeqDbInPlace() { seq_records->~vector(); ref->~basic_string(); contig->~basic_string(); }
};

long long write_out(const std::string& s, char* out, size_t cap)
{
    if (s.size() >= cap) return -1;
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

} // namespace

extern "C" {

// AlignmentDB::get_variants_in_region(contig, start, stop, min_frequency, min_depth) over the region [region_start, region_end] of
// `contig` and the base-space records of SeqDbInPlace.  out: one line per variant in the returned order, "ref_position \t ref_seq \t
// alt_seq \t info".  Returns the length written, -1 when cap is too small.
long long npref_variants_in_region(const char* contig, int region_start, int region_end, const char* region_ref, int n_seq, const char** seq_bases,
                                   const uint8_t* seq_rc, const int32_t* seq_pairs, const uint64_t* seq_pair_off, int start, int stop,
                                   double min_frequency, int min_depth, char* out, size_t cap)
{
    SeqDbInPlace d(contig, region_start, region_end, region_ref, n_seq, seq_bases, seq_rc, seq_pairs, seq_pair_off);
    std::string s;
    for (const Variant& v : d.db->get_variants_in_region(contig, start, stop, min_frequency, min_depth))
        s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\t" + v.info + "\n";
    return write_out(s, out, cap);
}

// The default mode of `nanopolish variants` on the window [start_base, end_base] of a contig of contig_length bases, over the region
// loaded at region_start (the caller's [start - BUFFER, min(end + BUFFER, contig_length - 1)]) with npref_call_haplotype's event records
// and npref_variants_in_region's base-space records.  call_variants_for_region's default branch (src/nanopolish_call_variants.cpp:
// 882-1011): BUFFER = flank + 10, region_start = max(start_base, BUFFER), region_end = the region's end - BUFFER, the candidates of
// get_variants_in_region (candidates_vcf NULL) or of read_variants_for_region over a temporary file holding candidates_vcf, then
// call_haplotype_from_candidates with HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP (npref_call_haplotype: the reference's own, its
// options set per call, one OpenMP thread).  Then call_variants_main's VCF.  Returns the length written, -1 when cap is too small,
// -2 when the temporary file cannot be written, -3 when npref_call_haplotype fails.
long long npref_call_region(const char* contig, int contig_length, int start_base, int end_base, int region_start, int region_end, const char* region_ref,
                            int n_records, const int32_t* read_h, const char** read_names, const uint8_t* rc, const int8_t* stride,
                            const uint64_t* pair_off, const uint32_t* n_pairs, const int32_t* pairs, int n_seq, const char** seq_bases,
                            const uint8_t* seq_rc, const int32_t* seq_pairs, const uint64_t* seq_pair_off, int flank, int min_distance,
                            int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support, int snps_only,
                            double min_frequency, int min_depth, const char* candidates_vcf, char* out, size_t cap)
{
    SeqDbInPlace d(contig, region_start, region_end, region_ref, n_seq, seq_bases, seq_rc, seq_pairs, seq_pair_off);
    const int BUFFER = flank + 10;
    const uint32_t alignment_flags = HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP;
    const int rs = start_base < BUFFER ? BUFFER : start_base;
    const int re = d.db->get_region_end() - BUFFER;
    std::vector<Variant> candidates;
    if (!candidates_vcf) {
        candidates = d.db->get_variants_in_region(contig, rs, re, min_frequency, min_depth);
    } else {
        char path[] = "/tmp/npref_candidates_XXXXXX";
        const int fd = mkstemp(path);
        FILE* f = fd >= 0 ? fdopen(fd, "w") : nullptr;
        const bool ok = f && std::fputs(candidates_vcf, f) >= 0;
        if (f) std::fclose(f);
        if (ok) candidates = read_variants_for_region(path, contig, rs, re);
        if (fd >= 0) std::remove(path);
        if (!ok) return -2;
    }
    // call_haplotype_from_candidates on the list: the derived sequence, then per called variant "ref_position \t ref_seq \t alt_seq \t
    // the quality's bits \t info \t genotype"
    std::vector<int32_t> pos;
    std::vector<const char*> vref, valt;
    for (const Variant& v : candidates) { pos.push_back((int32_t)v.ref_position); vref.push_back(v.ref_seq.c_str()); valt.push_back(v.alt_seq.c_str()); }
    pos.push_back(0); vref.push_back(""); valt.push_back("");
    std::vector<char> called(size_t(1) << 24);
    const long long n = npref_call_haplotype(contig, region_start, region_end, region_ref, n_records, read_h, read_names, rc, stride, pair_off, n_pairs,
                                             pairs, (int)candidates.size(), pos.data(), vref.data(), valt.data(), flank, min_distance, max_haplotypes,
                                             ploidy, genotype_only, types_csv, calculate_all_support, alignment_flags, called.data(), called.size());
    if (n < 0) return -3;
    std::vector<Variant> variants;
    std::istringstream lines(std::string(called.data(), (size_t)n));
    std::string line;
    std::getline(lines, line);                                   // the derived sequence
    while (std::getline(lines, line)) {
        std::vector<std::string> f;
        for (size_t a = 0, b; ; a = b + 1) {
            b = line.find('\t', a);
            f.push_back(line.substr(a, b == std::string::npos ? std::string::npos : b - a));
            if (b == std::string::npos) break;
        }
        Variant v;
        v.ref_name = contig;
        v.ref_position = std::stoull(f[0]);
        v.ref_seq = f[1]; v.alt_seq = f[2];
        const uint64_t bits = std::stoull(f[3], nullptr, 16);
        std::memcpy(&v.quality, &bits, sizeof(bits));
        v.genotype = f[5];
        // simple_call copies the candidate and appends its INFO to the candidate's (the basecall counts of get_variants_in_region);
        // npref_call_haplotype takes candidates without INFO, so the candidate's INFO goes back in front here.  Candidates with one
        // key share one INFO: get_variants_in_region's keys are distinct and read_variants_for_region clears INFO.
        std::string cand_info;
        for (const Variant& c : candidates)
            if (c.ref_position == v.ref_position && c.ref_seq == v.ref_seq && c.alt_seq == v.alt_seq) { cand_info = c.info; break; }
        v.info = cand_info.empty() ? f[4] : f[4].empty() ? cand_info : cand_info + ";" + f[4];
        variants.push_back(v);
    }
    std::vector<std::string> header_fields;
    std::stringstream polish_window;
    polish_window << contig << ":" << start_base << "-" << std::min(end_base, contig_length - 1);
    header_fields.push_back(Variant::make_vcf_header_key_value("nanopolish_window", polish_window.str()));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "TotalReads", 1, "Integer", "The number of event-space reads used to call the variant"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "SupportFraction", 1, "Float", "The fraction of event-space reads that support the variant"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "SupportFractionByStrand", 2, "Float", "Fraction of event-space reads that support the variant for each strand"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "BaseCalledReadsWithVariant", 1, "Integer", "The number of base-space reads that support the variant"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "BaseCalledFraction", 1, "Float", "The fraction of base-space reads that support the variant"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "AlleleCount", 1, "Integer", "The inferred number of copies of the allele"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "StrandSupport", 4, "Integer", "Number of reads supporting the REF and ALT allele, by strand"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "StrandFisherTest", 1, "Integer", "Strand bias fisher test"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "SOR", 1, "Float", "StrandOddsRatio test from GATK"));
    header_fields.push_back(Variant::make_vcf_tag_string("INFO", "RefContext", 1, "String", "The reference sequence context surrounding the variant call"));
    if (calculate_all_support)
        header_fields.push_back(Variant::make_vcf_tag_string("INFO", "SupportFractionByBase", 4, "Float", "The fraction of reads supporting A,C,G,T at this position"));
    header_fields.push_back(Variant::make_vcf_tag_string("FORMAT", "GT", 1, "String", "Genotype"));
    char* buf = nullptr;
    size_t len = 0;
    FILE* fp = open_memstream(&buf, &len);
    Variant::write_vcf_header(fp, header_fields);
    for (Variant& v : variants) {
        if (!snps_only || v.is_snp()) {
            int context_start_base = (int)v.ref_position - 5;
            if (context_start_base < 0) context_start_base = 0;
            int context_end_base = (int)(v.ref_position + v.ref_seq.length() + 4);
            if (context_end_base >= contig_length) context_end_base = contig_length - 1;
            v.add_info("RefContext", d.ref->substr(context_start_base - region_start, context_end_base - context_start_base + 1));
            v.write_vcf(fp);
        }
    }
    std::fclose(fp);
    const std::string s(buf, len);
    std::free(buf);
    return write_out(s, out, cap);
}

} // extern "C"
