// hp_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own fix_homopolymers (src/nanopolish_call_variants.cpp:541-780,
// compiled here in place through the #include below) unmodified on a hand-built haplotype and AlignmentDB, and returns the fixed
// haplotype.
//
// What the function reaches outside its computation:
//   opt::min_flanking_sequence  the TU's own option, set per call
//   AlignmentDB                 its constructor reads files and its members are private.  The harness never runs the constructor:
//                               it constructs, in storage of sizeof(AlignmentDB), the five members fix_homopolymers and
//                               get_event_subsequences read (region contig, start, end, reference, event records) and nothing
//                               else, and destroys exactly those.  The members are reached through pointers to members named in
//                               an explicit template instantiation (access checking does not apply to the names in one), so no
//                               reference source is compiled with any change, not even of access
//   EventAlignmentRecord::sr    the SquiggleRead of a handle of ref_harness.cpp (npref_read_create + npref_read_set_eventalign,
//                               which set durations; the reads are PORETYPE_R9), taken through npref_abea, whose call of
//                               adaptive_banded_simple_event_align is wrapped (-Wl,--wrap, oracle/hp.mk) as in phase_reads_harness.cpp
// Nothing of the reference is copied.
#include "nanopolish_call_variants.cpp"

#include <cstdio>
#include <new>

extern "C" long long npref_abea(int read_h, int model_h, const char* seq, int32_t* pairs_out, size_t cap);   // ref_harness.cpp

namespace {

// pointer-to-member of a private member, through an explicit instantiation
template <typename Tag, typename Tag::type M>
struct Expose { friend typename Tag::type member(Tag) { return M; } };
#define NPREF_EXPOSE(TAG, TYPE, NAME)                                          \
    struct TAG { typedef TYPE AlignmentDB::*type; friend type member(TAG); };  \
    template struct Expose<TAG, &AlignmentDB::NAME>;
NPREF_EXPOSE(DbContig, std::string, m_region_contig)
NPREF_EXPOSE(DbStart, int, m_region_start)
NPREF_EXPOSE(DbEnd, int, m_region_end)
NPREF_EXPOSE(DbRef, std::string, m_region_ref_sequence)
NPREF_EXPOSE(DbRecords, std::vector<EventAlignmentRecord>, m_event_records)

thread_local bool g_capture = false;
thread_local SquiggleRead* g_read = nullptr;

SquiggleRead* read_of(int h)
{
    g_capture = true;
    npref_abea(h, 0, "", nullptr, 0);
    g_capture = false;
    return g_read;
}

} // namespace

extern "C" std::vector<AlignedPair> __real__Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE(
    SquiggleRead&, const PoreModel&, const std::string&);
extern "C" std::vector<AlignedPair> __wrap__Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE(
    SquiggleRead& sr, const PoreModel& pm, const std::string& seq)
{
    if (g_capture) { g_read = &sr; return std::vector<AlignedPair>(); }
    return __real__Z34adaptive_banded_simple_event_alignR12SquiggleReadRK9PoreModelRKNSt7__cxx1112basic_stringIcSt11char_traitsIcESaIcEEE(sr, pm, seq);
}

extern "C" {

// fix_homopolymers(Haplotype(contig, hap_pos, hap_ref) + the variants applied in order, db) with opt::min_flanking_sequence =
// min_flank.  db: region [region_start, region_end] of `contig` with reference region_ref, and one EventAlignmentRecord per record
// (read handle, rc, stride, aligned_events as n_pairs (ref_pos, read_pos) pairs from pairs[pair_off]), strand 0.
// out: the fixed sequence, a newline, then one line per variant of the fixed haplotype:
//   ref_position \t ref_seq \t alt_seq \t quality as 16 hex digits of its bits \t info
// Returns the length written, -1 when cap is too small, -2 when a variant of the input does not apply.
long long npref_fix_homopolymers(const char* contig, int region_start, int region_end, const char* region_ref,
                                 int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                                 const uint32_t* n_pairs, const int32_t* pairs,
                                 int hap_pos, const char* hap_ref, int n_variants, const int32_t* var_pos, const char** var_ref,
                                 const char** var_alt, int min_flank, char* out, size_t cap)
{
    alignas(AlignmentDB) unsigned char storage[sizeof(AlignmentDB)];
    AlignmentDB* db = reinterpret_cast<AlignmentDB*>(storage);
    std::string* db_contig = new (&(db->*member(DbContig()))) std::string(contig);
    std::string* db_ref = new (&(db->*member(DbRef()))) std::string(region_ref);
    std::vector<EventAlignmentRecord>* db_records = new (&(db->*member(DbRecords()))) std::vector<EventAlignmentRecord>();
    db->*member(DbStart()) = region_start;
    db->*member(DbEnd()) = region_end;
    for (int r = 0; r < n_records; ++r) {
        EventAlignmentRecord er;
        er.sr = read_of(read_h[r]);
        er.rc = rc[r]; er.strand = 0; er.stride = stride[r];
        for (uint32_t i = 0; i < n_pairs[r]; ++i) {
            AlignedPair ap;
            ap.ref_pos = pairs[2 * (pair_off[r] + i)]; ap.read_pos = pairs[2 * (pair_off[r] + i) + 1];
            er.aligned_events.push_back(ap);
        }
        db_records->push_back(er);
    }
    Haplotype hap(contig, (size_t)hap_pos, hap_ref);
    bool applied = true;
    for (int i = 0; i < n_variants; ++i) {
        Variant v;
        v.ref_name = contig; v.ref_position = (size_t)var_pos[i]; v.ref_seq = var_ref[i]; v.alt_seq = var_alt[i];
        applied = applied && hap.apply_variant(v);
    }
    std::string s;
    if (applied) {
        const int saved = opt::min_flanking_sequence;
        opt::min_flanking_sequence = min_flank;
        const Haplotype fixed = fix_homopolymers(hap, *db);
        opt::min_flanking_sequence = saved;
        s = fixed.get_sequence() + "\n";
        for (const Variant& v : fixed.get_variants()) {
            uint64_t bits;
            std::memcpy(&bits, &v.quality, sizeof(bits));
            char q[32];
            std::snprintf(q, sizeof(q), "%016llx", (unsigned long long)bits);
            s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\t" + q + "\t" + v.info + "\n";
        }
    }
    db_records->~vector();
    db_ref->~basic_string();
    db_contig->~basic_string();
    if (!applied) return -2;
    if (s.size() >= cap) return -1;
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

// Haplotype::substr_by_reference(start, end) and get_enclosing_reference_range_for_haplotype_range(lo, hi) of
// Haplotype(contig, hap_pos, hap_ref) + the variants applied in order: out = the substring's sequence, range = {hap_lower, hap_upper,
// ref_lower, ref_upper} (npos as -1).  Returns the substring's reference position, -2 when a variant does not apply.  The reference's
// asserts are on: a range it refuses aborts the process.
long long npref_haplotype_ranges(int hap_pos, const char* hap_ref, int n_variants, const int32_t* var_pos, const char** var_ref,
                                 const char** var_alt, long long start, long long end, long long lo, long long hi, long long* range,
                                 char* out, size_t cap)
{
    Haplotype hap("ctg", (size_t)hap_pos, hap_ref);
    for (int i = 0; i < n_variants; ++i) {
        Variant v;
        v.ref_name = "ctg"; v.ref_position = (size_t)var_pos[i]; v.ref_seq = var_ref[i]; v.alt_seq = var_alt[i];
        if (!hap.apply_variant(v)) return -2;
    }
    size_t a = (size_t)lo, b = (size_t)hi, ra = 0, rb = 0;
    hap.get_enclosing_reference_range_for_haplotype_range(a, b, ra, rb);
    const size_t r4[4] = {a, b, ra, rb};
    for (int i = 0; i < 4; ++i) range[i] = r4[i] == std::string::npos ? -1 : (long long)r4[i];
    const Haplotype sub = hap.substr_by_reference((size_t)start, (size_t)end);
    if (sub.get_sequence().size() + 1 > cap) return -1;
    std::memcpy(out, sub.get_sequence().c_str(), sub.get_sequence().size() + 1);
    return (long long)sub.get_reference_position();
}

} // extern "C"
