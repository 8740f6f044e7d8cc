// support_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own annotate_variants_with_all_support
// (src/common/nanopolish_variant.cpp:801-859, linked from libnpref.so's objects) unmodified on a variant list and a hand-built
// AlignmentDB, and returns the variants' INFO.
//
// What the function reaches outside its computation:
//   AlignmentDB                 its constructor reads files and its members are private.  The harness never runs the constructor:
//                               it constructs, in storage of sizeof(AlignmentDB), the five members annotate_variants_with_all_support
//                               and get_event_subsequences read (region contig, start, end, reference, event records) and nothing
//                               else, and destroys exactly those — as hp_harness.cpp does for fix_homopolymers.  The members are
//                               reached through pointers to members named in an explicit template instantiation (access checking
//                               does not apply to the names in one), so no reference source is compiled with any change
//   EventAlignmentRecord::sr    the SquiggleRead of a handle of ref_harness.cpp (npref_read_create), taken through npref_abea, whose
//                               call of adaptive_banded_simple_event_align is wrapped (-Wl,--wrap, oracle/support.mk)
// Nothing of the reference is copied.
#include "nanopolish_alignment_db.h"
#include "nanopolish_variant.h"

#include <cstring>
#include <new>
#include <string>
#include <vector>

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

// annotate_variants_with_all_support(variants, db, min_flank, alignment_flags) on the variants {contig, var_pos[i], var_ref[i],
// var_alt[i]} in order.  db: region [region_start, region_end] of `contig` with reference region_ref, and one EventAlignmentRecord
// per record (read handle, rc, stride, aligned_events as n_pairs (ref_pos, read_pos) pairs from pairs[pair_off]), strand 0.
// out: one line per variant, its INFO after the call.  Returns the length written, -1 when cap is too small.  The reference's
// asserts are on: a window outside the region aborts the process.
long long npref_all_support(const char* contig, int region_start, int region_end, const char* region_ref,
                            int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                            const uint32_t* n_pairs, const int32_t* pairs,
                            int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt, int min_flank,
                            uint32_t alignment_flags, char* out, size_t cap)
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
    std::vector<Variant> variants(n_variants);
    for (int i = 0; i < n_variants; ++i) {
        variants[i].ref_name = contig; variants[i].ref_position = (size_t)var_pos[i];
        variants[i].ref_seq = var_ref[i]; variants[i].alt_seq = var_alt[i];
    }
    annotate_variants_with_all_support(variants, *db, min_flank, alignment_flags);
    std::string s;
    for (const Variant& v : variants) s += v.info + "\n";
    db_records->~vector();
    db_ref->~basic_string();
    db_contig->~basic_string();
    if (s.size() >= cap) return -1;
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

} // extern "C"
