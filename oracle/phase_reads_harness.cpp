// phase_reads_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own phase_single_read (src/nanopolish_phase_reads.cpp,
// compiled here in place through the #include below) unmodified, on one hand-built BAM record, and prints the SAM record it writes.
//
// What the function reaches outside its computation is answered by test doubles:
//   SquiggleRead(name, read_db)  the constructor that loads a read from a ReadDB is routed (-Wl,--wrap, oracle/phase.mk) to a copy
//                                of a read assembled by npref_read_create + npref_read_set_eventalign (ref_harness.cpp), found by
//                                its handle through npref_read_of
//   faidx_fetch_seq, bam_endpos  ref_harness.cpp's doubles (the contig held in memory)
//   bam_init1, bam_destroy1      calloc / free of a record
//   sam_write1                   keeps the record; npref_phase_read prints it as a SAM line (the mandatory fields of the SAM
//                                specification; no tags)
//   seq_nt16_table               the 4-bit base codes of the SAM/BAM specification ('=' and the IUPAC codes "=ACMGRSVTWYHKDBN",
//                                either case; every other byte is N)
// Nothing of the reference or of htslib is copied.
#include "nanopolish_phase_reads.cpp"
#include "ref_harness.h"

#include <cstdio>
#include <new>

extern double hmm_indel_bias_factor;                  // src/hmm/nanopolish_profile_hmm_r9.cpp:19

namespace {
thread_local int g_read_h = -1;                       // the handle whose read the wrapped constructor copies
thread_local std::string g_sam;                       // the last record sam_write1 received, as a SAM line
thread_local bool g_written = false;

} // namespace

// seq_nt16_table, computed from the specification's code string
constexpr unsigned char nt16(int c, int i = 0)
{
    return i == 16 ? (unsigned char)((c >= '0' && c <= '3') ? 1 << (c - '0') : 15)
                   : (c == "=ACMGRSVTWYHKDBN"[i] || c == "=acmgrsvtwyhkdbn"[i]) ? (unsigned char)i : nt16(c, i + 1);
}
#define NT16_4(c) nt16(c), nt16(c + 1), nt16(c + 2), nt16(c + 3)
#define NT16_16(c) NT16_4(c), NT16_4(c + 4), NT16_4(c + 8), NT16_4(c + 12)
#define NT16_64(c) NT16_16(c), NT16_16(c + 16), NT16_16(c + 32), NT16_16(c + 48)
extern "C" const unsigned char seq_nt16_table[256] = { NT16_64(0), NT16_64(64), NT16_64(128), NT16_64(192) };

// ---- the wrapped constructor (oracle/phase.mk links with --wrap=<its mangled name>) ----
extern "C" void __wrap__ZN12SquiggleReadC1ERKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEERK6ReadDBj(SquiggleRead* self, const std::string&,
                                                                                                         const ReadDB&, uint32_t)
{
    // what npref_read_create / npref_read_set_eventalign set, member by member (TransitionParameters owns raw buffers, so the
    // whole object is not assigned)
    SquiggleRead* sr = new (self) SquiggleRead();
    const SquiggleRead& src = *npref_read_of(g_read_h);
    sr->pore_type = src.pore_type; sr->read_type = src.read_type; sr->nucleotide_type = src.nucleotide_type;
    sr->read_name = src.read_name; sr->read_sequence = src.read_sequence;
    for (int s = 0; s < 2; ++s) {
        sr->base_model[s] = src.base_model[s]; sr->scalings[s] = src.scalings[s]; sr->events_per_base[s] = src.events_per_base[s];
        sr->events[s] = src.events[s];
    }
    sr->base_to_event_map = src.base_to_event_map;
}

extern "C" bam1_t* bam_init1(void) { return (bam1_t*)calloc(1, sizeof(bam1_t)); }
extern "C" void bam_destroy1(bam1_t* b) { if (b) { free(b->data); free(b); } }
extern "C" int sam_write1(samFile*, const bam_hdr_t* h, const bam1_t* b)
{
    std::string s = bam_get_qname(b);
    s += "\t" + std::to_string(b->core.flag) + "\t" + std::string(h->target_name[b->core.tid]) + "\t" + std::to_string(b->core.pos + 1) +
         "\t" + std::to_string(b->core.qual) + "\t";
    const uint32_t* cg = bam_get_cigar(b);
    for (uint32_t i = 0; i < b->core.n_cigar; ++i) s += std::to_string(bam_cigar_oplen(cg[i])) + bam_cigar_opchr(cg[i]);
    s += "\t*\t0\t0\t";
    const uint8_t* sq = bam_get_seq(b);
    for (int i = 0; i < b->core.l_qseq; ++i) s += "=ACMGRSVTWYHKDBN"[bam_seqi(sq, i)];
    s += "\t";
    const uint8_t* q = bam_get_qual(b);
    for (int i = 0; i < b->core.l_qseq; ++i) s += (char)(q[i] + 33);
    g_sam = s + "\n";
    g_written = true;
    return 0;
}

extern "C" {

// phase_single_read on one record: read_h from npref_read_create (+ npref_read_set_eventalign), the contig in memory, the record's
// pos / flag / mapq / CIGAR, and the sorted variant list (positions, REF and ALT strings).  The SAM line goes to sam_out; returns
// its length, 0 when the function wrote no record, -1 when cap is too small.
long long npref_phase_read(int read_h, const char* read_name, const char* contig_name, const char* contig_seq, int ref_pos, int flag, int mapq,
                           const uint32_t* cigar, int n_cigar, int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt,
                           double indel_bias, char* sam_out, size_t cap)
{
    g_read_h = read_h;
    NprefContig contig{contig_name, contig_seq};
    bam_hdr_t hdr;
    std::memset(&hdr, 0, sizeof(hdr));
    char* names[1] = { const_cast<char*>(contig.name.c_str()) };
    uint32_t lens[1] = { (uint32_t)contig.seq.size() };
    hdr.n_targets = 1; hdr.target_name = names; hdr.target_len = lens;
    const size_t nl = std::strlen(read_name) + 1, l_qname = (nl + 3) / 4 * 4;
    std::vector<uint8_t> data(l_qname + 4 * (size_t)n_cigar, 0);
    std::memcpy(data.data(), read_name, nl);
    std::memcpy(data.data() + l_qname, cigar, 4 * (size_t)n_cigar);
    bam1_t rec;
    std::memset(&rec, 0, sizeof(rec));
    rec.core.pos = ref_pos; rec.core.tid = 0; rec.core.flag = (uint16_t)flag; rec.core.qual = (uint8_t)mapq; rec.core.l_qname = (uint16_t)l_qname;
    rec.core.l_extranul = (uint8_t)(l_qname - nl); rec.core.n_cigar = n_cigar; rec.core.mtid = -1; rec.core.mpos = -1;
    rec.data = data.data(); rec.l_data = (int)data.size(); rec.m_data = (uint32_t)data.size();
    std::vector<Variant> variants((size_t)n_variants);
    for (int i = 0; i < n_variants; ++i) {
        variants[i].ref_name = contig_name; variants[i].ref_position = (size_t)var_pos[i];
        variants[i].ref_seq = var_ref[i]; variants[i].alt_seq = var_alt[i];
    }
    const double saved_bias = hmm_indel_bias_factor;
    hmm_indel_bias_factor = indel_bias;
    g_written = false;
    phase_single_read(*reinterpret_cast<const ReadDB*>(&contig), reinterpret_cast<const faidx_t*>(&contig), variants, nullptr, &hdr, &rec, 0, -1, -1);
    hmm_indel_bias_factor = saved_bias;
    if (!g_written) return 0;
    if (g_sam.size() >= cap) return -1;
    std::memcpy(sam_out, g_sam.c_str(), g_sam.size() + 1);
    return (long long)g_sam.size();
}

} // extern "C"
