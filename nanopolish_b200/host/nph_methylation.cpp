// nph_methylation.cpp — see nph_methylation.hpp (SURVEY.md section 8f, row N3).
#include "nph_methylation.hpp"
#include "../csrc/tsv_format.cuh"

#include <algorithm>
#include <cmath>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>

namespace nph {

// ---------------------------------------------------------------------------------------------
// modBAM tags
// ---------------------------------------------------------------------------------------------
char unmodified_symbol_of(const Alphabet* alphabet)
{
    if (alphabet->num_recognition_sites() != 1) throw Error(NPH_ERR_UNSUPPORTED, "modBAM output needs an alphabet with one recognition site");
    char unmodified = 'N';
    const char* modified_motif = alphabet->get_recognition_site_methylated(0);
    for (size_t i = 0; i < alphabet->recognition_length(); ++i)
        if (modified_motif[i] == METHYLATED_SYMBOL) unmodified = alphabet->get_recognition_site(0)[i];
    if (unmodified == 'N') throw Error(NPH_ERR_INVALID, "alphabet without a methylated symbol");
    return unmodified;
}

void calculate_call_vectors(const std::map<int, ScoredSite>& calls, const Alphabet* alphabet,
                            std::vector<size_t>& call_reference_positions, std::vector<uint8_t>& call_probabilities)
{
    for (const auto& kv : calls) {
        const ScoredSite& call = kv.second;
        // the called positions are where methylate() puts the symbol; start_position is the first site of the group, so
        // the flank in front of it is subtracted
        const std::string m_seq = alphabet->methylate(call.sequence);
        const size_t flank_offset = m_seq.find_first_of(METHYLATED_SYMBOL);
        if (flank_offset == std::string::npos) throw Error(NPH_ERR_INVALID, "scored site without a motif");      // the reference asserts
        // shared by every motif of the group; strand 0 only, as in the reference
        const double methylation_probability = std::exp(call.ll_methylated[0]) / (std::exp(call.ll_methylated[0]) + std::exp(call.ll_unmethylated[0]));
        const uint8_t code = (uint8_t)std::min(255, (int)(methylation_probability * 255));
        for (size_t j = 0; j < m_seq.size(); j++) {
            if (m_seq[j] == METHYLATED_SYMBOL) {
                call_reference_positions.push_back((size_t)(call.start_position + (int)j - (int)flank_offset));
                call_probabilities.push_back(code);
            }
        }
    }
}

// The MM tag (SAM tags specification, base modifications): "<base>+m?" then, per listed call, how many unmodified <base>s of the
// sequence lie between the previous listed position and this one, comma separated, ';' at the end.  One walk over the sequence with a
// running count of the unmodified symbol; the listed indices ascend (modbam_tags orders them), and an index that steps backwards
// restarts the walk there, which is what counting "from the previous position + 1" means for it (nothing in between: 0).
std::string generate_mm_tag(char unmodified_symbol, const std::string& sequence, const std::vector<size_t>& call_seq_indices)
{
    std::string tag(1, unmodified_symbol);
    tag += "+m?";
    size_t cursor = 0;            // first base not yet accounted for
    for (const size_t at : call_seq_indices) {
        size_t skipped = 0;
        for (; cursor < at; ++cursor) skipped += sequence[cursor] == unmodified_symbol ? 1u : 0u;
        tag += ',';
        tag += std::to_string(skipped);
        cursor = at + 1;
    }
    tag += ';';
    return tag;
}

ModbamTags modbam_tags(const std::string& bam_seq, const std::vector<AlignedPair>& aligned_bases, bool is_reverse,
                       const std::map<int, ScoredSite>& calls, const MethylationCallingParameters& params)
{
    const Alphabet* alphabet = params.alphabet ? params.alphabet : get_alphabet_by_name(params.methylation_type);
    if (std::string(alphabet->get_name()) != "cpg") throw Error(NPH_ERR_UNSUPPORTED, "modBAM output supports the cpg alphabet only");   // the reference asserts
    const char unmodified_symbol = unmodified_symbol_of(alphabet);
    std::vector<size_t> call_reference_positions;
    std::vector<uint8_t> call_reference_probabilities;
    calculate_call_vectors(calls, alphabet, call_reference_positions, call_reference_probabilities);

    // reference position -> index into the read as sequenced
    const std::string original_sequence = !is_reverse ? bam_seq : gDNAAlphabet.reverse_complement(bam_seq);
    std::map<size_t, size_t> reference_to_read_map;
    for (const AlignedPair& ap : aligned_bases)
        reference_to_read_map[(size_t)ap.ref_pos] = !is_reverse ? (size_t)ap.read_pos : original_sequence.length() - (size_t)ap.read_pos - 1;
    // a CG read from the opposite strand has its C aligned to the reference G
    const size_t strand_offset = !is_reverse ? 0 : 1;
    ModbamTags out;
    std::vector<size_t> call_seq_indices;
    for (size_t i = 0; i < call_reference_positions.size(); ++i) {
        auto iter = reference_to_read_map.find(call_reference_positions[i] + strand_offset);
        if (iter == reference_to_read_map.end()) continue;
        const size_t read_index = iter->second;
        if (read_index < original_sequence.size() && original_sequence[read_index] == unmodified_symbol) {
            call_seq_indices.push_back(read_index);
            out.ml.push_back(call_reference_probabilities[i]);
        }
    }
    // SEQ is reverse complemented for reverse-strand records: list the calls in the original direction
    if (is_reverse) {
        std::reverse(call_seq_indices.begin(), call_seq_indices.end());
        std::reverse(out.ml.begin(), out.ml.end());
    }
    out.mm = generate_mm_tag(unmodified_symbol, original_sequence, call_seq_indices);
    return out;
}

ModbamTags reference_modbam_tags(const std::string& ref_seq, int ref_start_pos, const std::map<int, ScoredSite>& calls,
                                 const MethylationCallingParameters& params)
{
    const Alphabet* alphabet = params.alphabet ? params.alphabet : get_alphabet_by_name(params.methylation_type);
    const char unmodified_symbol = unmodified_symbol_of(alphabet);
    std::vector<size_t> call_reference_positions;
    ModbamTags out;
    calculate_call_vectors(calls, alphabet, call_reference_positions, out.ml);
    std::vector<size_t> indices;
    for (size_t pos : call_reference_positions) indices.push_back(pos - (size_t)ref_start_pos);
    out.mm = generate_mm_tag(unmodified_symbol, ref_seq, indices);
    return out;
}

template <typename T>
void PinnedArray<T>::resize(size_t n)
{
    if (n > m_cap) {
        const size_t want = std::max<size_t>(n + n / 2, 1024);
        void* np = nullptr;
        const int rc = nph_host_alloc(&np, want * sizeof(T));
        if (rc != NPH_OK) throw Error(rc, "nph_host_alloc (page-locked staging)");
        if (m_p) { std::memcpy(np, m_p, m_n * sizeof(T)); nph_host_free(m_p); }
        m_p = static_cast<T*>(np);
        m_cap = want;
    }
    m_n = n;
}
template class PinnedArray<char>;
template class PinnedArray<nph_aligned_pair>;
template class PinnedArray<nph_meth_site>;
template class PinnedArray<int16_t>;

nph_meth_params make_meth_params(const MethylationCallingParameters& params, uint32_t k, int region_start, int region_end)
{
    const Alphabet* a = params.alphabet ? params.alphabet : get_alphabet_by_name(params.methylation_type);
    nph_meth_params p;
    std::memset(&p, 0, sizeof(p));
    p.min_separation = params.min_separation;
    p.min_flank = params.min_flank;
    p.max_span = 200;                      // basemods.cpp:336
    p.min_event_span = 10;                 // basemods.cpp:363
    p.region_start = region_start;
    p.region_end = region_end;
    p.k = k;
    p.alphabet_size = a->size();
    if (a->size() > 7 || a->num_recognition_sites() > NPH_METH_MAX_SITES || a->recognition_length() >= NPH_METH_MAX_SITE_LEN || a->num_recognition_sites() == 0)
        throw Error(NPH_ERR_UNSUPPORTED, "alphabet outside nph_meth_params' limits");
    for (uint32_t i = 0; i < a->size(); ++i) { p.bases[i] = a->base((uint8_t)i); p.complements[i] = a->complement(a->base((uint8_t)i)); }
    p.n_sites = (uint32_t)a->num_recognition_sites();
    p.site_len = (uint32_t)a->recognition_length();
    for (uint32_t s = 0; s < p.n_sites; ++s) {
        std::memcpy(p.sites[s], a->get_recognition_site(s), p.site_len);
        std::memcpy(p.sites_methylated[s], a->get_recognition_site_methylated(s), p.site_len);
        std::memcpy(p.sites_methylated_complement[s], a->get_recognition_site_methylated_complement(s), p.site_len);
    }
    return p;
}

bool compact_event_alignment(const std::vector<AlignedPair>& ae, int ref_start_pos, size_t ref_len, int16_t* deltas, int32_t* first_event)
{
    const long long len = (long long)ref_len;
    for (long long o = 0; o < len; ++o) deltas[o] = (int16_t)NPH_METH_NO_PAIR;
    long long prev_off = -1;
    int prev_ev = ae.empty() ? 0 : ae[0].read_pos;
    *first_event = prev_ev;
    for (const AlignedPair& ap : ae) {
        const long long o = (long long)ap.ref_pos - ref_start_pos;
        const long long step = (long long)ap.read_pos - prev_ev;
        if (o <= prev_off || o >= len || step > 32767 || step < -32767) return false;
        deltas[o] = (int16_t)step;
        prev_off = o; prev_ev = ap.read_pos;
    }
    return true;
}

MethylationCaller::MethylationCaller(const MethylationCallingParameters& params) : m_params(params)
{
    if (!m_params.alphabet) m_params.alphabet = get_alphabet_by_name(m_params.methylation_type);
}

void MethylationCaller::clear()
{
    m_reads.clear();
    m_ref.clear(); m_pairs.clear(); m_sites.clear(); m_records.clear(); m_record_meta.clear(); m_site_off.clear();
    m_deltas.clear(); m_first_event.clear(); m_compact_ok = true;
    m_n_sites = 0; m_scored_events = 0; m_region_set = false; m_ran = false;
}

// Copy what the device enumeration reads — the reference substring once per read, the event alignment of each
// strand that has events and a motif model — into the page-locked batch buffers (parallel over reads), one
// nph_meth_record per (read, strand).
void MethylationCaller::stage(const EventAlignedRead* const* reads, size_t n, int region_start, int region_end)
{
    if (m_region_set && (region_start != m_region_start || region_end != m_region_end))
        throw Error(NPH_ERR_UNSUPPORTED, "one output window per batch: call run() before changing region_start / region_end");
    m_region_start = region_start; m_region_end = region_end; m_region_set = true;
    m_ran = false;
    struct Slot { size_t ref_off[2], pair_off[2], rec[2]; bool use[2]; };
    std::vector<Slot> slots(n);
    size_t ref_total = m_ref.size(), pair_total = m_pairs.size();
    const size_t first_read = m_reads.size();
    for (size_t i = 0; i < n; ++i) {
        const EventAlignedRead& r = *reads[i];
        ReadEntry re;
        re.name = r.read_name; re.is_reverse = r.is_reverse; re.contig = r.contig;
        re.ref_off = ref_total; re.ref_len = r.ref_seq.size(); re.ref_start_pos = r.ref_start_pos;
        re.first_record = m_records.size();
        bool ref_placed = false;
        for (size_t strand_idx = 0; strand_idx < 2; ++strand_idx) {
            slots[i].use[strand_idx] = false;
            if (r.ref_seq.empty() || !r.read->has_events_for_strand(strand_idx)) continue;
            const PoreModel* motif_model = r.read->get_model((uint32_t)strand_idx, m_params.methylation_type);
            if (!motif_model) continue;                                   // no model for this motif on this strand
            if (r.read->pore_type != PORETYPE_R9) throw Error(NPH_ERR_UNSUPPORTED, "only R9 reads are supported (load_from_raw always makes R9)");
            const uint32_t k = (uint32_t)r.read->get_model_k((uint32_t)strand_idx);
            if (re.k && re.k != k) throw Error(NPH_ERR_UNSUPPORTED, "strands with different k in one read");
            re.k = k;
            nph_meth_record rec;
            std::memset(&rec, 0, sizeof(rec));
            // every record carries its own copy of the reference substring: the compact event alignment runs parallel to it
            slots[i].ref_off[strand_idx] = ref_total; slots[i].rec[strand_idx] = m_records.size();
            if (!ref_placed) { re.ref_off = ref_total; ref_placed = true; }
            rec.ref_off = ref_total; rec.ref_len = (uint32_t)r.ref_seq.size();
            ref_total += r.ref_seq.size();
            rec.pair_off = pair_total; rec.n_pairs = (uint32_t)r.aligned_events[strand_idx].size();
            rec.ref_start_pos = r.ref_start_pos; rec.rc = r.rc[strand_idx] ? 1 : 0; rec.strand = (uint8_t)strand_idx;
            slots[i].use[strand_idx] = true; slots[i].pair_off[strand_idx] = pair_total;
            pair_total += rec.n_pairs;
            m_records.push_back(rec);
            m_record_meta.push_back(Record{r.read, motif_model, (uint8_t)strand_idx});
        }
        re.n_records = m_records.size() - re.first_record;
        m_reads.push_back(std::move(re));
    }
    (void)first_read;
    m_ref.resize(ref_total);
    m_pairs.resize(pair_total);
    m_deltas.resize(ref_total);
    m_first_event.resize(m_records.size(), 0);
    char* const ref = m_ref.data();
    nph_aligned_pair* const pairs = m_pairs.data();
    int16_t* const deltas = m_deltas.data();
    int compact_ok = m_compact_ok ? 1 : 0;
    static_assert(sizeof(AlignedPair) == sizeof(nph_aligned_pair), "AlignedPair layout");
#pragma omp parallel for schedule(dynamic, 16) num_threads(host_threads()) if (n > 64)
    for (long long ii = 0; ii < (long long)n; ++ii) {
        const EventAlignedRead& r = *reads[(size_t)ii];
        const Slot& s = slots[(size_t)ii];
        for (int st = 0; st < 2; ++st) {
            if (!s.use[st]) continue;
            std::memcpy(ref + s.ref_off[st], r.ref_seq.data(), r.ref_seq.size());
            const std::vector<AlignedPair>& ae = r.aligned_events[st];
            if (!ae.empty()) std::memcpy(pairs + s.pair_off[st], ae.data(), sizeof(AlignedPair) * ae.size());
            // compact form: event-index steps per reference base (nph.h); a step beyond int16, a reference position outside the
            // substring or out of order makes the whole batch fall back to the pair lists
            if (!compact_event_alignment(ae, r.ref_start_pos, r.ref_seq.size(), deltas + s.ref_off[st], &m_first_event[s.rec[st]])) {
#pragma omp atomic write
                compact_ok = 0;
            }
        }
    }
    m_compact_ok = compact_ok != 0;
}

size_t MethylationCaller::add_read(const EventAlignedRead& r, int region_start, int region_end)
{
    const size_t read_idx = m_reads.size();
    const EventAlignedRead* one = &r;
    stage(&one, 1, region_start, region_end);
    return read_idx;
}

size_t MethylationCaller::add_reads(const std::vector<EventAlignedRead>& reads, int region_start, int region_end)
{
    const size_t first = m_reads.size();
    std::vector<const EventAlignedRead*> ptrs(reads.size());
    for (size_t i = 0; i < reads.size(); ++i) ptrs[i] = &reads[i];
    stage(ptrs.data(), ptrs.size(), region_start, region_end);
    return first;
}

void MethylationCaller::run(Engine& engine, double indel_bias)
{
    m_site_off.assign(m_records.size() + 1, 0);
    m_n_sites = 0; m_scored_events = 0;
    for (ReadEntry& re : m_reads) { re.sites.clear(); re.sites_built = false; }
    m_ran = true;
    if (m_records.empty()) return;
    // one nph_read per distinct (SquiggleRead, strand)
    detail::ReadTable reads;
    uint32_t k = 0;
    for (size_t i = 0; i < m_records.size(); ++i) {
        const Record& rm = m_record_meta[i];
        m_records[i].read = reads.index(rm.read, rm.strand);
        m_records[i].model_id = engine.model_id(rm.model);
        if (k && rm.model->k != k) throw Error(NPH_ERR_UNSUPPORTED, "models with different k in one call-methylation batch");
        k = rm.model->k;
    }
    const detail::FlatReads fr = detail::flatten_reads(engine, reads);
    const nph_meth_params mp = make_meth_params(m_params, k, m_region_start, m_region_end);
    size_t cap = 0;
    for (const nph_meth_record& r : m_records) cap += r.ref_len / (size_t)(m_params.min_separation + 1) + 2;
    m_sites.resize(cap);
    if (m_compact_ok)
        engine.check(nph_methylation_batch_compact(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events,
                                                   m_ref.data(), m_deltas.data(), m_ref.size(), m_first_event.data(), m_records.data(), m_records.size(),
                                                   &mp, indel_bias, m_site_off.data(), m_sites.data(), cap, &m_scored_events),
                     "nph_methylation_batch_compact");
    else
        engine.check(nph_methylation_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events,
                                           m_ref.data(), m_ref.size(), m_pairs.data(), m_pairs.size(), m_records.data(), m_records.size(),
                                           &mp, indel_bias, m_site_off.data(), m_sites.data(), cap, &m_scored_events),
                     "nph_methylation_batch");
    m_n_sites = m_site_off.back();
}

// TSV rows (write_methylation_results_as_tsv, call_methylation.cpp:532-550) are written straight into a growing character
// buffer by csrc/tsv_format.cuh's put_meth_row, the writer the device uses too — no printf and no per-field string appends.
namespace {
struct RowBuffer {
    std::unique_ptr<char[]> p;
    size_t n = 0, cap = 0;
    char* room(size_t extra)           // at least `extra` writable bytes at the returned position
    {
        if (n + extra > cap) {
            const size_t want = std::max(cap * 2, n + extra + 4096);
            std::unique_ptr<char[]> q(new char[want]);
            if (n) std::memcpy(q.get(), p.get(), n);
            p.swap(q); cap = want;
        }
        return p.get() + n;
    }
};
const size_t kRowOverhead = 3 * 48 + 64;            // three %.2lf fields of float sums (printf: at most 44 bytes each), integers, tabs

// One row whose strands sum to sum_m and sum_u (row.diff, row.m, row.u hold their fixed_of<2>).  A number the exact formatter
// refuses (non-finite, >= 2^52) takes the reference's format string.
void append_row(RowBuffer& out, const nph_tsv::MethRow& row, double sum_m, double sum_u)
{
    const size_t room = row.contig_len + row.name_len + row.seq_len + kRowOverhead;
    char* const o = out.room(room);
    if (row.diff.ok && row.m.ok && row.u.ok) { out.n += (size_t)(nph_tsv::put_meth_row(o, row) - o); return; }
    out.n += (size_t)snprintf(o, room, "%.*s\t%c\t%d\t%d\t%.*s\t%.2lf\t%.2lf\t%.2lf\t%d\t%d\t%.*s\n", (int)row.contig_len, row.contig, row.strand,
                              row.start, row.end, (int)row.name_len, row.name, sum_m - sum_u, sum_m, sum_u, row.strands_scored, row.n_motif,
                              (int)row.seq_len, row.seq);
}

// The rows of a record that is its read's only scored strand: its site records are already the rows, in ascending position.
// ref_bases + rec.ref_off is the record's reference.
void append_record_rows(RowBuffer& out, const std::string& contig, bool is_reverse, const char* name, size_t name_len, const char* ref_bases,
                        const nph_meth_record& rec, uint32_t k, const nph_meth_site* sites, size_t n)
{
    for (size_t s = 0; s < n; ++s) {
        const nph_meth_site& ms = sites[s];
        const nph_tsv::RowNums r = nph_tsv::row_numbers(ms, rec, k);
        if (!r.seq_ok) throw Error(NPH_ERR_INVALID, nph_tsv::kSeqRefused);
        const nph_tsv::MethRow row{contig.data(), (uint32_t)contig.size(), is_reverse ? '-' : '+', ms.start_position, ms.end_position, name,
                                   (uint32_t)name_len, r.diff, r.m, r.u, 1, (int)ms.n_motif, ref_bases + rec.ref_off + r.seq_b, r.seq_len};
        // the other strand's 0.0 added, as row_numbers does
        append_row(out, row, (double)ms.ll_methylated + 0.0, (double)ms.ll_unmethylated + 0.0);
    }
}
} // namespace

// The ScoredSite map of one read from its site records (the strands of a read meet at start_position,
// exactly as the reference's find-or-insert does, basemods.cpp:403-425).
void MethylationCaller::build_sites(size_t read_idx) const
{
    const ReadEntry& re = m_reads[read_idx];
    if (re.sites_built) return;
    if (!m_ran) throw Error(NPH_ERR_STATE, "MethylationCaller::sites before run()");
    for (size_t rec = re.first_record; rec < re.first_record + re.n_records; ++rec) {
        const nph_meth_record& R = m_records[rec];
        const size_t strand = R.strand;
        for (uint64_t s = m_site_off[rec]; s < m_site_off[rec + 1]; ++s) {
            const nph_meth_site& ms = m_sites.data()[s];
            auto iter = re.sites.find(ms.start_position);
            if (iter == re.sites.end()) {
                ScoredSite ss;
                ss.chromosome = re.contig;
                ss.start_position = ms.start_position;
                ss.end_position = ms.end_position;
                ss.n_motif = (int)ms.n_motif;
                // the motif site(s) with a k-mer's worth of context either side (std::string::substr cuts at the end)
                const nph_tsv::RowNums r = nph_tsv::row_numbers(ms, R, re.k);
                if (!r.seq_ok) throw Error(NPH_ERR_INVALID, nph_tsv::kSeqRefused);
                ss.sequence.assign(m_ref.data() + R.ref_off + r.seq_b, r.seq_len);
                iter = re.sites.insert({ms.start_position, ss}).first;
            }
            iter->second.ll_unmethylated[strand] = ms.ll_unmethylated;      // float -> double, like `double s = profile_hmm_score(...)`
            iter->second.ll_methylated[strand] = ms.ll_methylated;
            iter->second.strands_scored += 1;
        }
    }
    re.sites_built = true;
}

const std::map<int, ScoredSite>& MethylationCaller::sites(size_t read_idx) const
{
    build_sites(read_idx);
    return m_reads[read_idx].sites;
}

void MethylationCaller::append_rows(std::string& out, size_t read_idx) const
{
    RowBuffer rb;
    put_rows(&rb, read_idx);
    out.append(rb.p.get(), rb.n);
}

void MethylationCaller::put_rows(void* row_buffer, size_t read_idx) const
{
    RowBuffer& out = *static_cast<RowBuffer*>(row_buffer);
    const ReadEntry& re = m_reads[read_idx];
    if (re.n_records == 1 && !re.sites_built) {
        if (!m_ran) throw Error(NPH_ERR_STATE, "MethylationCaller::tsv before run()");
        const size_t rec = re.first_record;
        append_record_rows(out, re.contig, re.is_reverse, re.name.data(), re.name.size(), m_ref.data(), m_records[rec], re.k,
                           m_sites.data() + m_site_off[rec], (size_t)(m_site_off[rec + 1] - m_site_off[rec]));
        return;
    }
    for (const auto& kv : sites(read_idx)) {
        const ScoredSite& ss = kv.second;
        const double sum_m = ss.ll_methylated[0] + ss.ll_methylated[1], sum_u = ss.ll_unmethylated[0] + ss.ll_unmethylated[1];
        const nph_tsv::MethRow row{ss.chromosome.data(), (uint32_t)ss.chromosome.size(), re.is_reverse ? '-' : '+', ss.start_position,
                                   ss.end_position, re.name.data(), (uint32_t)re.name.size(), nph_tsv::fixed_of<2>(sum_m - sum_u),
                                   nph_tsv::fixed_of<2>(sum_m), nph_tsv::fixed_of<2>(sum_u), ss.strands_scored, ss.n_motif,
                                   ss.sequence.data(), (uint32_t)ss.sequence.size()};
        append_row(out, row, sum_m, sum_u);
    }
}

std::string MethylationCaller::tsv(size_t read_idx) const
{
    std::string out;
    append_rows(out, read_idx);
    return out;
}

std::vector<std::string> MethylationCaller::tsv_batch() const
{
    std::vector<std::string> out(m_reads.size());
    parallel_for(m_reads.size(), m_reads.size() > 64 ? host_threads() : 1, 16, [&](size_t i) { out[i] = tsv(i); });
    return out;
}

size_t MethylationCaller::tsv_all(char* out, size_t cap) const
{
    // contiguous blocks of reads per worker: format into a private buffer, then copy to the block's offset
    const size_t n = m_reads.size();
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)host_threads(), (n + 63) / 64));
    std::vector<RowBuffer> parts((size_t)T);
    parallel_for((size_t)T, T, 1, [&](size_t t) {
        const size_t b = n * t / (size_t)T, e = n * (t + 1) / (size_t)T;
        parts[t].room((e - b) * 4096);
        for (size_t i = b; i < e; ++i) put_rows(&parts[t], i);
    });
    std::vector<size_t> off((size_t)T + 1, 0);
    for (int t = 0; t < T; ++t) off[t + 1] = off[t] + parts[t].n;
    if (off[T] > cap || !out) return off[T];
#pragma omp parallel for schedule(static, 1) num_threads(T) if (T > 1)
    for (int t = 0; t < T; ++t) if (parts[t].n) std::memcpy(out + off[t], parts[t].p.get(), parts[t].n);
    return off[T];
}

// The whole of call-methylation for a batch that already sits in flat host buffers (the layout of nph_methylation_batch):
// one device call that returns the TSV rows formatted on the device.  Pair lists, a value the device formatter refuses or
// $NPH_METH_HOST_TSV take the record path instead: one device call for the site records, whose rows host_threads() workers format.
namespace {
void format_records(const FlatMethylationBatch& b, uint32_t k, const uint64_t* site_off, const nph_meth_site* sites, std::vector<RowBuffer>& parts)
{
    const size_t n = b.n_records;
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)host_threads(), (n + 63) / 64));
    parts.clear();
    parts.resize((size_t)T);
    const std::string contig(b.contig ? b.contig : "");
    parallel_for((size_t)T, T, 1, [&](size_t t) {
        const size_t lo = n * t / (size_t)T, hi = n * (t + 1) / (size_t)T;
        RowBuffer& out = parts[t];
        out.room((size_t)(site_off[hi] - site_off[lo]) * 96 + 64);
        for (size_t r = lo; r < hi; ++r) {
            const char* name = b.read_names[r];
            append_record_rows(out, contig, b.is_reverse[r] != 0, name, std::strlen(name), b.ref_bases, b.records[r], k, sites + site_off[r],
                               (size_t)(site_off[r + 1] - site_off[r]));
        }
    });
}
} // namespace

size_t call_methylation_flat(Engine& engine, const FlatMethylationBatch& b, const MethylationCallingParameters& params, uint32_t k,
                             double indel_bias, char* tsv_out, size_t cap, FlatMethylationStats* stats)
{
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    const nph_meth_params mp = make_meth_params(params, k, b.region_start, b.region_end);
    const size_t n = b.n_records;
    // Rows formatted on the device (nph_methylation_batch_compact_tsv): the site records never leave it and the host's share of the call
    // is the name table.  Needs the compact event alignment and a destination; $NPH_METH_HOST_TSV keeps the host formatter (A/B, tests).
    static const bool host_tsv = std::getenv("NPH_METH_HOST_TSV") != nullptr;
    if (b.event_deltas && tsv_out && !host_tsv && n > 0) {
        std::vector<uint32_t> name_off(n + 1, 0);
        for (size_t r = 0; r < n; ++r) name_off[r + 1] = name_off[r] + (uint32_t)std::strlen(b.read_names[r]);
        std::string names((size_t)name_off[n], '\0');
        for (size_t r = 0; r < n; ++r) std::memcpy(&names[name_off[r]], b.read_names[r], name_off[r + 1] - name_off[r]);
        uint64_t n_bytes = 0, n_sites = 0, scored = 0;
        const double td = now();
        const int rc = nph_methylation_batch_compact_tsv(engine.ctx(), b.reads, b.n_reads, b.ev_mean, b.ev_start_time, b.n_events, b.ref_bases,
                                                         b.event_deltas, b.n_ref, b.first_event, b.records, n, &mp, indel_bias,
                                                         b.contig ? b.contig : "", names.data(), name_off.data(), b.is_reverse,
                                                         tsv_out, cap, &n_bytes, &n_sites, &scored);
        if (rc == NPH_OK || (rc == NPH_ERR_INVALID && n_bytes > cap)) {          // too small a destination: report the size, like the host path
            if (stats) { stats->n_sites = n_sites; stats->scored_events = scored; stats->device_seconds = now() - td; stats->tsv_seconds = (now() - t0) - stats->device_seconds; }
            return (size_t)n_bytes;
        }
        if (rc != NPH_ERR_UNSUPPORTED) engine.check(rc, "nph_methylation_batch_compact_tsv");
        // a value the device formatter refuses (not finite, beyond 2^52): score again through the record path and format here
    }
    size_t site_cap = 0;
    for (size_t r = 0; r < n; ++r) site_cap += b.records[r].ref_len / (size_t)(params.min_separation + 1) + 2;
    nph_meth_site* sites =
        static_cast<nph_meth_site*>(engine.pinned(Engine::Staging::MethylationSites, sizeof(nph_meth_site) * std::max<size_t>(site_cap, 1)));
    std::vector<uint64_t> site_off(n + 1, 0);
    uint64_t scored = 0;
    const double td = now();
    const int rc = b.event_deltas
        ? nph_methylation_batch_compact(engine.ctx(), b.reads, b.n_reads, b.ev_mean, b.ev_start_time, b.n_events, b.ref_bases, b.event_deltas,
                                        b.n_ref, b.first_event, b.records, n, &mp, indel_bias, site_off.data(), sites, site_cap, &scored)
        : nph_methylation_batch(engine.ctx(), b.reads, b.n_reads, b.ev_mean, b.ev_start_time, b.n_events, b.ref_bases, b.n_ref,
                                b.aligned_events, b.n_pairs, b.records, n, &mp, indel_bias, site_off.data(), sites, site_cap, &scored);
    const double device_s = now() - td;
    engine.check(rc, b.event_deltas ? "nph_methylation_batch_compact" : "nph_methylation_batch");
    std::vector<RowBuffer> parts;
    format_records(b, k, site_off.data(), sites, parts);
    std::vector<size_t> off(parts.size() + 1, 0);
    for (size_t t = 0; t < parts.size(); ++t) off[t + 1] = off[t] + parts[t].n;
    const size_t total = off.back();
    if (tsv_out && total <= cap) {
#pragma omp parallel for schedule(static, 1) num_threads(host_threads()) if (parts.size() > 1)
        for (long long t = 0; t < (long long)parts.size(); ++t)
            if (parts[(size_t)t].n) std::memcpy(tsv_out + off[(size_t)t], parts[(size_t)t].p.get(), parts[(size_t)t].n);
    }
    // device_seconds: time inside the device call; tsv_seconds: what the formatting and the copy added on top
    if (stats) { stats->n_sites = site_off[n]; stats->scored_events = scored; stats->device_seconds = device_s; stats->tsv_seconds = (now() - t0) - device_s; }
    return total;
}

void MethylationCaller::write_tsv(FILE* fp, size_t read_idx) const
{
    const std::string s = tsv(read_idx);
    fwrite(s.data(), 1, s.size(), fp);
}

} // namespace nph
