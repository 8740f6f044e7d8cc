// variants_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own variant calling unmodified on hand-built candidate lists,
// haplotypes and AlignmentDBs, and returns what it computed:
//   fix_homopolymers, screen_variants_by_score, expand_variants, call_haplotype_from_candidates and the header and records
//   call_variants_main writes (src/nanopolish_call_variants.cpp, compiled here in place through the #include below)
//   annotate_variants_with_all_support and read_variants_for_region (src/common/nanopolish_variant.cpp) and
//   AlignmentDB::get_variants_in_region (src/alignment/nanopolish_alignment_db.cpp), linked from libnpref.so's objects
//   Haplotype::substr_by_reference and get_enclosing_reference_range_for_haplotype_range, kt_fisher_exact (src/thirdparty/fet.c)
//   and the Combinations generator (src/nanopolish_variant_db.cpp), for the tests of the host mirror's own
//
// What the functions reach outside their computation:
//   opt::*                      the TU's own options: each entry point sets the ones its comment names and an OptGuard restores them,
//                               and the OpenMP thread count where it runs on one thread, when it returns
//   AlignmentDB                 its constructor reads files and its members are private.  The harness never runs the constructor:
//                               DbInPlace constructs, in storage of sizeof(AlignmentDB), the members the functions read (region
//                               contig, start, end, reference, event records, base-space records) and nothing else, and destroys
//                               exactly those.  The members are reached through pointers to members named in an explicit template
//                               instantiation (access checking does not apply to the names in one), so no reference source is
//                               compiled with any change, not even of access
//   EventAlignmentRecord::sr    the SquiggleRead of a handle of ref_harness.cpp (npref_read_of): npref_read_create with the built-in
//                               r9.4_450bps nucleotide model as base model, so that SquiggleRead::get_model(strand, type) finds the
//                               built-in model of each methylation type, and npref_read_set_eventalign for the event durations
// Nothing of the reference is copied.
#include "nanopolish_call_variants.cpp"
#include "ref_harness.h"

#include "fet.h"
#include <omp.h>
#include <cstdio>
#include <cstdlib>
#include <new>

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
NPREF_EXPOSE(DbSeqRecords, std::vector<SequenceAlignmentRecord>, m_sequence_records)

// event record r: read handle read_h[r], rc[r], stride[r], strand 0, aligned_events the n_pairs[r] (ref_pos, read_pos) pairs from
// pairs[2 * pair_off[r]]
struct EventRecords {
    int n;
    const int32_t* read_h; const uint8_t* rc; const int8_t* stride; const uint64_t* pair_off; const uint32_t* n_pairs; const int32_t* pairs;
};

// base-space record r: bases bases[r], strand rc[r], aligned_bases the pairs from pairs[2 * pair_off[r]] up to pairs[2 * pair_off[r + 1]]
struct SeqRecords {
    int n;
    const char** bases; const uint8_t* rc; const int32_t* pairs; const uint64_t* pair_off;
};

// the AlignmentDB of one call, built in place and torn down by its destructor
struct DbInPlace {
    alignas(AlignmentDB) unsigned char storage[sizeof(AlignmentDB)];
    AlignmentDB* db;
    std::string* contig;
    std::string* ref;
    std::vector<EventAlignmentRecord>* records;
    std::vector<SequenceAlignmentRecord>* seq_records;
    DbInPlace(const char* c, int region_start, int region_end, const char* region_ref, const EventRecords& ev, const SeqRecords& sq = SeqRecords())
    {
        db = reinterpret_cast<AlignmentDB*>(storage);
        contig = new (&(db->*member(DbContig()))) std::string(c);
        ref = new (&(db->*member(DbRef()))) std::string(region_ref);
        records = new (&(db->*member(DbRecords()))) std::vector<EventAlignmentRecord>();
        seq_records = new (&(db->*member(DbSeqRecords()))) std::vector<SequenceAlignmentRecord>();
        db->*member(DbStart()) = region_start;
        db->*member(DbEnd()) = region_end;
        for (int r = 0; r < ev.n; ++r) {
            EventAlignmentRecord er;
            er.sr = npref_read_of(ev.read_h[r]);
            er.rc = ev.rc[r]; er.strand = 0; er.stride = ev.stride[r];
            for (uint64_t i = ev.pair_off[r]; i < ev.pair_off[r] + ev.n_pairs[r]; ++i) {
                AlignedPair ap;
                ap.ref_pos = ev.pairs[2 * i]; ap.read_pos = ev.pairs[2 * i + 1];
                er.aligned_events.push_back(ap);
            }
            records->push_back(er);
        }
        // SequenceAlignmentRecord has no constructor but the one from a bam1_t: its members are built in place
        for (int r = 0; r < sq.n; ++r) {
            alignas(SequenceAlignmentRecord) unsigned char raw[sizeof(SequenceAlignmentRecord)];
            SequenceAlignmentRecord* sr = reinterpret_cast<SequenceAlignmentRecord*>(raw);
            new (&sr->read_name) std::string("seq" + std::to_string(r));
            new (&sr->sequence) std::string(sq.bases[r]);
            new (&sr->aligned_bases) std::vector<AlignedPair>();
            sr->rc = sq.rc[r];
            for (uint64_t i = sq.pair_off[r]; i < sq.pair_off[r + 1]; ++i) {
                AlignedPair ap;
                ap.ref_pos = sq.pairs[2 * i]; ap.read_pos = sq.pairs[2 * i + 1];
                sr->aligned_bases.push_back(ap);
            }
            seq_records->push_back(*sr);
            sr->aligned_bases.~vector(); sr->sequence.~basic_string(); sr->read_name.~basic_string();
        }
    }
    ~DbInPlace() { seq_records->~vector(); records->~vector(); ref->~basic_string(); contig->~basic_string(); }
};

// the opt:: values the entry points set, and with one_thread() the OpenMP thread count, restored when the guard goes out of scope
struct OptGuard {
    int* const ints[8] = {&opt::min_flanking_sequence, &opt::screen_flanking_sequence, &opt::screen_score_threshold,
                          &opt::min_distance_between_variants, &opt::max_haplotypes, &opt::ploidy, &opt::genotype_only,
                          &opt::calculate_all_support};
    int saved[8];
    const std::vector<std::string> types = opt::methylation_types;
    int threads = 0;
    OptGuard() { for (int i = 0; i < 8; ++i) saved[i] = *ints[i]; }
    void one_thread() { threads = omp_get_max_threads(); omp_set_num_threads(1); }
    ~OptGuard()
    {
        for (int i = 0; i < 8; ++i) *ints[i] = saved[i];
        opt::methylation_types = types;
        if (threads) omp_set_num_threads(threads);
    }
};

std::vector<Variant> candidates_of(const char* contig, int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt)
{
    std::vector<Variant> vs(n_variants);
    for (int i = 0; i < n_variants; ++i) {
        vs[i].ref_name = contig; vs[i].ref_position = (size_t)var_pos[i]; vs[i].ref_seq = var_ref[i]; vs[i].alt_seq = var_alt[i];
    }
    return vs;
}

// csv split at commas ("" = none)
std::vector<std::string> split_csv(const char* csv)
{
    std::vector<std::string> out;
    for (std::string s = csv; !s.empty(); ) {
        const size_t c = s.find(',');
        out.push_back(s.substr(0, c));
        s = c == std::string::npos ? std::string() : s.substr(c + 1);
    }
    return out;
}

// "ref_position \t ref_seq \t alt_seq \t the 16 hex digits of the quality's bits \t info", then "\t genotype" with_genotype, and a newline
std::string variant_line(const Variant& v, bool with_genotype = false)
{
    uint64_t bits;
    std::memcpy(&bits, &v.quality, sizeof(bits));
    char q[32];
    std::snprintf(q, sizeof(q), "%016llx", (unsigned long long)bits);
    return std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\t" + q + "\t" + v.info +
           (with_genotype ? "\t" + v.genotype : std::string()) + "\n";
}

long long write_out(const std::string& s, char* out, size_t cap)
{
    if (s.size() >= cap) return -1;
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

// call_haplotype_from_candidates(d.db, candidates, alignment_flags) with the options given, on one OpenMP thread; record r's read is
// named read_names[r]
Haplotype call_haplotype(const DbInPlace& d, const std::vector<Variant>& candidates, const char** read_names, int flank, int min_distance,
                         int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support,
                         uint32_t alignment_flags)
{
    for (size_t r = 0; r < d.records->size(); ++r) (*d.records)[r].sr->read_name = read_names[r];
    OptGuard g;
    opt::min_flanking_sequence = flank;
    opt::min_distance_between_variants = min_distance;
    opt::max_haplotypes = max_haplotypes;
    opt::ploidy = ploidy;
    opt::genotype_only = genotype_only;
    opt::calculate_all_support = calculate_all_support;
    opt::methylation_types = split_csv(types_csv);
    g.one_thread();
    return call_haplotype_from_candidates(*d.db, candidates, alignment_flags);
}

} // namespace

extern "C" {

// fix_homopolymers(Haplotype(contig, hap_pos, hap_ref) + the variants applied in order, db) with opt::min_flanking_sequence =
// min_flank.  db: region [region_start, region_end] of `contig` with reference region_ref, and the event records (EventRecords).
// out: the fixed sequence, a newline, then one line per variant of the fixed haplotype (variant_line).  Returns the length written,
// -1 when cap is too small, -2 when a variant of the input does not apply.
long long npref_fix_homopolymers(const char* contig, int region_start, int region_end, const char* region_ref,
                                 int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                                 const uint32_t* n_pairs, const int32_t* pairs,
                                 int hap_pos, const char* hap_ref, int n_variants, const int32_t* var_pos, const char** var_ref,
                                 const char** var_alt, int min_flank, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, {n_records, read_h, rc, stride, pair_off, n_pairs, pairs});
    Haplotype hap(contig, (size_t)hap_pos, hap_ref);
    for (const Variant& v : candidates_of(contig, n_variants, var_pos, var_ref, var_alt))
        if (!hap.apply_variant(v)) return -2;
    OptGuard g;
    opt::min_flanking_sequence = min_flank;
    const Haplotype fixed = fix_homopolymers(hap, *d.db);
    std::string s = fixed.get_sequence() + "\n";
    for (const Variant& v : fixed.get_variants()) s += variant_line(v);
    return write_out(s, out, cap);
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
    for (const Variant& v : candidates_of("ctg", n_variants, var_pos, var_ref, var_alt))
        if (!hap.apply_variant(v)) return -2;
    size_t a = (size_t)lo, b = (size_t)hi, ra = 0, rb = 0;
    hap.get_enclosing_reference_range_for_haplotype_range(a, b, ra, rb);
    const size_t r4[4] = {a, b, ra, rb};
    for (int i = 0; i < 4; ++i) range[i] = r4[i] == std::string::npos ? -1 : (long long)r4[i];
    const Haplotype sub = hap.substr_by_reference((size_t)start, (size_t)end);
    if (sub.get_sequence().size() + 1 > cap) return -1;
    std::memcpy(out, sub.get_sequence().c_str(), sub.get_sequence().size() + 1);
    return (long long)sub.get_reference_position();
}

// screen_variants_by_score(db, candidates, alignment_flags) with opt::screen_flanking_sequence = flank, opt::screen_score_threshold =
// threshold and opt::methylation_types = types_csv split at commas, on one OpenMP thread, so that score_variant_thresholded's early
// exit follows read order.  db as npref_fix_homopolymers takes it.  out: one line per output variant (variant_line).  Returns the
// length written, -1 when cap is too small.
long long npref_screen_variants(const char* contig, int region_start, int region_end, const char* region_ref,
                                int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                                const uint32_t* n_pairs, const int32_t* pairs, int n_variants, const int32_t* var_pos, const char** var_ref,
                                const char** var_alt, int flank, int threshold, const char* types_csv, uint32_t alignment_flags, char* out,
                                size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, {n_records, read_h, rc, stride, pair_off, n_pairs, pairs});
    OptGuard g;
    opt::screen_flanking_sequence = flank;
    opt::screen_score_threshold = threshold;
    opt::methylation_types = split_csv(types_csv);
    g.one_thread();
    std::string s;
    for (const Variant& v : screen_variants_by_score(*d.db, candidates_of(contig, n_variants, var_pos, var_ref, var_alt), alignment_flags))
        s += variant_line(v);
    return write_out(s, out, cap);
}

// expand_variants(db, candidates, region_start, region_end, 0) with opt::min_flanking_sequence = min_flank, db without records.
// out: one line per output variant, "ref_position \t ref_seq \t alt_seq".  Returns the length written, -1 when cap is too small.
// The reference's asserts are on.
long long npref_expand_variants(const char* contig, int region_start, int region_end, const char* region_ref, int n_variants,
                                const int32_t* var_pos, const char** var_ref, const char** var_alt, int min_flank, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, EventRecords());
    OptGuard g;
    opt::min_flanking_sequence = min_flank;
    std::string s;
    for (const Variant& v : expand_variants(*d.db, candidates_of(contig, n_variants, var_pos, var_ref, var_alt), region_start, region_end, 0))
        s += std::to_string(v.ref_position) + "\t" + v.ref_seq + "\t" + v.alt_seq + "\n";
    return write_out(s, out, cap);
}

// call_haplotype_from_candidates(db, candidates, alignment_flags) with opt::min_flanking_sequence = flank,
// opt::min_distance_between_variants, opt::max_haplotypes, opt::ploidy, opt::genotype_only, opt::calculate_all_support and
// opt::methylation_types = types_csv split at commas, on one OpenMP thread; db as npref_fix_homopolymers takes it, record r's read
// named read_names[r] (VariantGroup keys reads by "read_name:strand").  out: the derived sequence, then one line per variant of the
// derived haplotype (variant_line with its genotype).  Returns the length written, -1 when cap is too small.
long long npref_call_haplotype(const char* contig, int region_start, int region_end, const char* region_ref, int n_records, const int32_t* read_h,
                               const char** read_names, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off, const uint32_t* n_pairs,
                               const int32_t* pairs, int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt, int flank,
                               int min_distance, int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support,
                               uint32_t alignment_flags, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, {n_records, read_h, rc, stride, pair_off, n_pairs, pairs});
    const Haplotype derived = call_haplotype(d, candidates_of(contig, n_variants, var_pos, var_ref, var_alt), read_names, flank, min_distance,
                                             max_haplotypes, ploidy, genotype_only, types_csv, calculate_all_support, alignment_flags);
    std::string s = derived.get_sequence() + "\n";
    for (const Variant& v : derived.get_variants()) s += variant_line(v, true);
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

// annotate_variants_with_all_support(variants, db, min_flank, alignment_flags) on the variants {contig, var_pos[i], var_ref[i],
// var_alt[i]} in order; db as npref_fix_homopolymers takes it.  out: one line per variant, its INFO after the call.  Returns the
// length written, -1 when cap is too small.  The reference's asserts are on: a window outside the region aborts the process.
long long npref_all_support(const char* contig, int region_start, int region_end, const char* region_ref,
                            int n_records, const int32_t* read_h, const uint8_t* rc, const int8_t* stride, const uint64_t* pair_off,
                            const uint32_t* n_pairs, const int32_t* pairs,
                            int n_variants, const int32_t* var_pos, const char** var_ref, const char** var_alt, int min_flank,
                            uint32_t alignment_flags, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, {n_records, read_h, rc, stride, pair_off, n_pairs, pairs});
    std::vector<Variant> variants = candidates_of(contig, n_variants, var_pos, var_ref, var_alt);
    annotate_variants_with_all_support(variants, *d.db, min_flank, alignment_flags);
    std::string s;
    for (const Variant& v : variants) s += v.info + "\n";
    return write_out(s, out, cap);
}

// AlignmentDB::get_variants_in_region(contig, start, stop, min_frequency, min_depth) over the region [region_start, region_end] of
// `contig` and the base-space records (SeqRecords).  out: one line per variant in the returned order, "ref_position \t ref_seq \t
// alt_seq \t info".  Returns the length written, -1 when cap is too small.
long long npref_variants_in_region(const char* contig, int region_start, int region_end, const char* region_ref, int n_seq, const char** seq_bases,
                                   const uint8_t* seq_rc, const int32_t* seq_pairs, const uint64_t* seq_pair_off, int start, int stop,
                                   double min_frequency, int min_depth, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, EventRecords(), {n_seq, seq_bases, seq_rc, seq_pairs, seq_pair_off});
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
// call_haplotype_from_candidates with HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP, as npref_call_haplotype runs it.  Then
// call_variants_main's VCF.  Returns the length written, -1 when cap is too small, -2 when the temporary file cannot be written.
long long npref_call_region(const char* contig, int contig_length, int start_base, int end_base, int region_start, int region_end, const char* region_ref,
                            int n_records, const int32_t* read_h, const char** read_names, const uint8_t* rc, const int8_t* stride,
                            const uint64_t* pair_off, const uint32_t* n_pairs, const int32_t* pairs, int n_seq, const char** seq_bases,
                            const uint8_t* seq_rc, const int32_t* seq_pairs, const uint64_t* seq_pair_off, int flank, int min_distance,
                            int max_haplotypes, int ploidy, int genotype_only, const char* types_csv, int calculate_all_support, int snps_only,
                            double min_frequency, int min_depth, const char* candidates_vcf, char* out, size_t cap)
{
    DbInPlace d(contig, region_start, region_end, region_ref, {n_records, read_h, rc, stride, pair_off, n_pairs, pairs},
                {n_seq, seq_bases, seq_rc, seq_pairs, seq_pair_off});
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
    // call_haplotype_from_candidates on the candidates' positions and alleles alone, as npref_call_haplotype takes them
    std::vector<Variant> bare(candidates.size());
    for (size_t i = 0; i < candidates.size(); ++i) {
        bare[i].ref_name = contig; bare[i].ref_position = candidates[i].ref_position;
        bare[i].ref_seq = candidates[i].ref_seq; bare[i].alt_seq = candidates[i].alt_seq;
    }
    std::vector<Variant> variants = call_haplotype(d, bare, read_names, flank, min_distance, max_haplotypes, ploidy, genotype_only, types_csv,
                                                   calculate_all_support, alignment_flags).get_variants();
    for (Variant& v : variants) {
        // simple_call copies the candidate and appends its INFO to the candidate's (the basecall counts of get_variants_in_region);
        // the candidates above have no INFO, so the candidate's INFO goes back in front here.  Candidates with one key share one
        // INFO: get_variants_in_region's keys are distinct and read_variants_for_region clears INFO.
        std::string cand_info;
        for (const Variant& c : candidates)
            if (c.ref_position == v.ref_position && c.ref_seq == v.ref_seq && c.alt_seq == v.alt_seq) { cand_info = c.info; break; }
        v.info = cand_info.empty() ? v.info : v.info.empty() ? cand_info : cand_info + ";" + v.info;
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
