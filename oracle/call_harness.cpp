// call_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own call_haplotype_from_candidates
// (src/nanopolish_call_variants.cpp:782-880, compiled here in place through the #include below) unmodified on a hand-built candidate
// list and AlignmentDB, and returns the derived haplotype and its variants.  Also exports the reference's kt_fisher_exact
// (src/thirdparty/fet.c) and its Combinations generator (src/nanopolish_variant_db.cpp), for the tests of the host mirror's own.
//
// What the function reaches outside its computation:
//   opt::min_flanking_sequence, opt::min_distance_between_variants, opt::max_haplotypes, opt::ploidy, opt::genotype_only,
//   opt::methylation_types, opt::calculate_all_support
//                               the TU's own options, set per call and restored after it; one OpenMP thread
//   AlignmentDB                 built in place as screen_harness.cpp builds it
//   EventAlignmentRecord::sr    the SquiggleRead of a handle of ref_harness.cpp, as screen_harness.cpp finds it; its read_name is
//                               set per record (VariantGroup keys reads by "read_name:strand")
// Nothing of the reference is copied.
#include "nanopolish_call_variants.cpp"

#include "fet.h"
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

static std::vector<std::string> split_csv(const char* csv)
{
    std::vector<std::string> out;
    for (std::string s = csv; !s.empty(); ) {
        const size_t c = s.find(',');
        out.push_back(s.substr(0, c));
        s = c == std::string::npos ? std::string() : s.substr(c + 1);
    }
    return out;
}

// call_haplotype_from_candidates(db, candidates, alignment_flags) with the options given, on one OpenMP thread; record r's read is
// named read_names[r].  out: the derived sequence, then one line per variant of the derived haplotype, "ref_position \t ref_seq \t
// alt_seq \t the 16 hex digits of the quality's bits \t info \t genotype".  Returns the length written, -1 when cap is too small.
long long npref_call_haplotype(const char* contig, int region_start, int region_end, const char* region_ref, int n_records, const int32_t* read_h,
                               const char** read_names, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off, const uint32_t* n_pairs,
                               const int32_t* pairs, int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt, int flank,
                               int min_distance, int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support,
                               uint32_t alignment_flags, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, n_records, read_h, rc, stride, pair_off, n_pairs, pairs);
    for (int r = 0; r < n_records; ++r) (*d.records)[r].sr->read_name = read_names[r];
    const std::vector<Variant> candidates = candidates_of(contig, n_variants, var_pos, var_ref, var_alt);
    const int s_flank = opt::min_flanking_sequence, s_dist = opt::min_distance_between_variants, s_maxh = opt::max_haplotypes;
    const int s_ploidy = opt::ploidy, s_gt = opt::genotype_only, s_all = opt::calculate_all_support;
    const std::vector<std::string> s_types = opt::methylation_types;
    const int saved_threads = omp_get_max_threads();
    opt::min_flanking_sequence = flank;
    opt::min_distance_between_variants = min_distance;
    opt::max_haplotypes = max_haplotypes;
    opt::ploidy = ploidy;
    opt::genotype_only = genotype_only;
    opt::calculate_all_support = calculate_all_support;
    opt::methylation_types = split_csv(types_csv);
    omp_set_num_threads(1);
    const Haplotype derived = call_haplotype_from_candidates(*d.db, candidates, alignment_flags);
    omp_set_num_threads(saved_threads);
    opt::min_flanking_sequence = s_flank; opt::min_distance_between_variants = s_dist; opt::max_haplotypes = s_maxh;
    opt::ploidy = s_ploidy; opt::genotype_only = s_gt; opt::calculate_all_support = s_all; opt::methylation_types = s_types;
    std::string s = derived.get_sequence() + "\n";
    for (const Variant& v : derived.get_variants()) {
        uint64_t bits;
        std::memcpy(&bits, &v.quality, sizeof(bits));
        char q[32];
        std::snprintf(q, sizeof(q), "%016llx", (unsigned long long)bits);
        s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\t" + q + "\t" + v.info + "\t" + v.genotype + "\n";
    }
    return write_out(s, out, cap);
}

// kt_fisher_exact's two-sided p-value
double npref_fisher_exact(int n11, int n12, int n21, int n22)
{
    double left, right, two;
    kt_fisher_exact(n11, n12, n21, n22, &left, &right, &two);
    return two;
}

// the sets Combinations(n, k, with_replacement ? CO_WITH_REPLACEMENT : CO_WITHOUT_REPLACEMENT) visits, k ids each, into out (room
// for cap ids).  Returns the number of sets, -1 when cap is too small.
long long npref_combinations(int n, int k, int with_replacement, uint32_t* out, size_t cap)
{
    Combinations c((size_t)n, (size_t)k, with_replacement ? CO_WITH_REPLACEMENT : CO_WITHOUT_REPLACEMENT);
    long long sets = 0;
    size_t at = 0;
    while (!c.done()) {
        const std::vector<size_t> ids = c.get();
        if (at + ids.size() > cap) return -1;
        for (size_t id : ids) out[at++] = (uint32_t)id;
        ++sets;
        c.next();
    }
    return sets;
}

} // extern "C"
