// screen_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own screen_variants_by_score and expand_variants
// (src/nanopolish_call_variants.cpp:364-450, compiled here in place through the #include below) unmodified on a hand-built candidate
// list and AlignmentDB, and returns their output lists.
//
// What the functions reach outside their computation:
//   opt::screen_flanking_sequence, opt::screen_score_threshold, opt::methylation_types, opt::min_flanking_sequence
//                               the TU's own options, set per call and restored after it; one OpenMP thread, so that
//                               score_variant_thresholded's early exit follows read order
//   AlignmentDB                 built in place exactly as hp_harness.cpp does for fix_homopolymers: the five members the functions
//                               and get_event_subsequences read (region contig, start, end, reference, event records), reached
//                               through pointers to members named in an explicit template instantiation, constructed in storage of
//                               sizeof(AlignmentDB) and destroyed again.  No reference source is compiled with any change
//   EventAlignmentRecord::sr    the SquiggleRead of a handle of ref_harness.cpp (npref_read_create, with the built-in r9.4_450bps
//                               nucleotide model as base model, so that SquiggleRead::get_model(strand, type) finds the built-in
//                               model of each methylation type), taken through npref_abea, whose call of
//                               adaptive_banded_simple_event_align is wrapped (-Wl,--wrap, oracle/screen.mk)
// Nothing of the reference is copied.
#include "nanopolish_call_variants.cpp"

#include <omp.h>
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

// the AlignmentDB of one call, built in place and torn down by its destructor
struct DbInPlace {
    alignas(AlignmentDB) unsigned char storage[sizeof(AlignmentDB)];
    AlignmentDB* db;
    std::string* contig;
    std::string* ref;
    std::vector<EventAlignmentRecord>* records;
    DbInPlace(const char* c, int region_start, int region_end, const char* region_ref, int n_records, const int32_t* read_h, const uint8_t* rc,
              const int8_t* stride, const uint64_t* pair_off, const uint32_t* n_pairs, const int32_t* pairs)
    {
        db = reinterpret_cast<AlignmentDB*>(storage);
        contig = new (&(db->*member(DbContig()))) std::string(c);
        ref = new (&(db->*member(DbRef()))) std::string(region_ref);
        records = new (&(db->*member(DbRecords()))) std::vector<EventAlignmentRecord>();
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
            records->push_back(er);
        }
    }
    ~DbInPlace() { records->~vector(); ref->~basic_string(); contig->~basic_string(); }
};

static std::vector<Variant> candidates_of(const char* contig, int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt)
{
    std::vector<Variant> vs(n_variants);
    for (int i = 0; i < n_variants; ++i) {
        vs[i].ref_name = contig; vs[i].ref_position = (size_t)var_pos[i]; vs[i].ref_seq = var_ref[i]; vs[i].alt_seq = var_alt[i];
    }
    return vs;
}

static long long write_out(const std::string& s, char* out, size_t cap)
{
    if (s.size() >= cap) return -1;
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

// screen_variants_by_score(db, candidates, alignment_flags) with opt::screen_flanking_sequence = flank, opt::screen_score_threshold =
// threshold and opt::methylation_types = types_csv split at commas ("" = none), on one OpenMP thread.  db as npref_fix_homopolymers
// takes it.  out: one line per output variant, "ref_position \t ref_seq \t alt_seq \t the 16 hex digits of the quality's bits
// \t info".  Returns the length written, -1 when cap is too small.
long long npref_screen_variants(const char* contig, int region_start, int region_end, const char* region_ref,
                                int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                                const uint32_t* n_pairs, const int32_t* pairs, int n_variants, const int32_t* var_pos, const char** var_ref,
                                const char** var_alt, int flank, int threshold, const char* types_csv, uint32_t alignment_flags, char* out,
                                size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, n_records, read_h, rc, stride, pair_off, n_pairs, pairs);
    const std::vector<Variant> candidates = candidates_of(contig, n_variants, var_pos, var_ref, var_alt);
    const int saved_flank = opt::screen_flanking_sequence, saved_threshold = opt::screen_score_threshold;
    const std::vector<std::string> saved_types = opt::methylation_types;
    const int saved_threads = omp_get_max_threads();
    opt::screen_flanking_sequence = flank;
    opt::screen_score_threshold = threshold;
    opt::methylation_types.clear();
    for (std::string s = types_csv; !s.empty(); ) {
        const size_t c = s.find(',');
        opt::methylation_types.push_back(s.substr(0, c));
        s = c == std::string::npos ? std::string() : s.substr(c + 1);
    }
    omp_set_num_threads(1);
    const std::vector<Variant> kept = screen_variants_by_score(*d.db, candidates, alignment_flags);
    omp_set_num_threads(saved_threads);
    opt::screen_flanking_sequence = saved_flank;
    opt::screen_score_threshold = saved_threshold;
    opt::methylation_types = saved_types;
    std::string s;
    for (const Variant& v : kept) {
        uint64_t bits;
        std::memcpy(&bits, &v.quality, sizeof(bits));
        char q[32];
        std::snprintf(q, sizeof(q), "%016llx", (unsigned long long)bits);
        s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\t" + q + "\t" + v.info + "\n";
    }
    return write_out(s, out, cap);
}

// expand_variants(db, candidates, region_start, region_end, 0) with opt::min_flanking_sequence = min_flank, db without records.
// out: one line per output variant, "ref_position \t ref_seq \t alt_seq".  Returns the length written, -1 when cap is too small.
// The reference's asserts are on.
long long npref_expand_variants(const char* contig, int region_start, int region_end, const char* region_ref, int n_variants,
                                const int32_t* var_pos, const char** var_ref, const char** var_alt, int min_flank, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    const std::vector<Variant> candidates = candidates_of(contig, n_variants, var_pos, var_ref, var_alt);
    const int saved = opt::min_flanking_sequence;
    opt::min_flanking_sequence = min_flank;
    const std::vector<Variant> expanded = expand_variants(*d.db, candidates, region_start, region_end, 0);
    opt::min_flanking_sequence = saved;
    std::string s;
    for (const Variant& v : expanded) s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\n";
    return write_out(s, out, cap);
}

} // extern "C"
