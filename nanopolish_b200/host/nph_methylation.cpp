// nph_methylation.cpp — see nph_methylation.hpp (SURVEY.md section 8f, row N3).
#include "nph_methylation.hpp"

#include <algorithm>
#include <cmath>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>

namespace nph {

static const int MAX_EVENT_TO_BP_RATIO = 20;       // ref: src/alignment/nanopolish_alignment_db.h:18

// lower_bound on ref_pos for both ends; bounded only if an aligned base sits at or outside each boundary.
// (The right-hand test compares the successor with ref_START, as the reference does.)
bool find_by_ref_bounds(const std::vector<AlignedPair>& pairs, int ref_start, int ref_stop, int& read_start, int& read_stop)
{
    auto lb = [](const AlignedPair& o, int v) { return o.ref_pos < v; };
    auto start_iter = std::lower_bound(pairs.begin(), pairs.end(), ref_start, lb);
    auto stop_iter = std::lower_bound(pairs.begin(), pairs.end(), ref_stop, lb);
    if (start_iter == pairs.end() || stop_iter == pairs.end()) return false;
    bool left_bounded = start_iter->ref_pos <= ref_start || (start_iter != pairs.begin() && (start_iter - 1)->ref_pos <= ref_start);
    bool right_bounded = stop_iter->ref_pos >= ref_stop || ((stop_iter + 1) != pairs.end() && (stop_iter + 1)->ref_pos >= ref_start);
    if (!(left_bounded && right_bounded)) return false;
    read_start = start_iter->read_pos;
    read_stop = stop_iter->read_pos;
    return true;
}

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

MethylationCaller::MethylationCaller(const MethylationCallingParameters& params, Mode mode) : m_mode(mode), m_params(params)
{
    if (!m_params.alphabet) m_params.alphabet = get_alphabet_by_name(m_params.methylation_type);
}

void MethylationCaller::clear()
{
    m_batch.clear(); m_pending.clear(); m_reads.clear();
    m_ref.clear(); m_pairs.clear(); m_sites.clear(); m_records.clear(); m_record_meta.clear(); m_site_off.clear();
    m_deltas.clear(); m_first_event.clear(); m_compact_ok = true;
    m_n_sites = 0; m_scored_events = 0; m_region_set = false; m_ran = false;
}

// Device mode: copy what the enumeration reads — the reference substring once per read, the event alignment of each
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
            int16_t* d = deltas + s.ref_off[st];
            const long long len = (long long)r.ref_seq.size();
            for (long long o = 0; o < len; ++o) d[o] = (int16_t)NPH_METH_NO_PAIR;
            long long prev_off = -1;
            int prev_ev = ae.empty() ? 0 : ae[0].read_pos;
            m_first_event[s.rec[st]] = prev_ev;
            bool ok = true;
            for (const AlignedPair& ap : ae) {
                const long long o = (long long)ap.ref_pos - r.ref_start_pos;
                const long long step = (long long)ap.read_pos - prev_ev;
                if (o <= prev_off || o >= len || step > 32767 || step < -32767) { ok = false; break; }
                d[o] = (int16_t)step;
                prev_off = o; prev_ev = ap.read_pos;
            }
            if (!ok) {
#pragma omp atomic write
                compact_ok = 0;
            }
        }
    }
    m_compact_ok = compact_ok != 0;
}

size_t MethylationCaller::add_read(const EventAlignedRead& r, int region_start, int region_end)
{
    if (m_mode == Mode::HostEnumeration) return add_read_host(r, region_start, region_end);
    const size_t read_idx = m_reads.size();
    const EventAlignedRead* one = &r;
    stage(&one, 1, region_start, region_end);
    return read_idx;
}

size_t MethylationCaller::add_read_host(const EventAlignedRead& r, int region_start, int region_end)
{
    const size_t read_idx = m_reads.size();
    m_reads.emplace_back();
    m_reads.back().name = r.read_name; m_reads.back().is_reverse = r.is_reverse; m_reads.back().sites_built = true;
    std::map<int, ScoredSite>& site_score_map = m_reads.back().sites;
    const std::string& ref_seq = r.ref_seq;
    if (ref_seq.empty()) return read_idx;
    const Alphabet* alphabet = m_params.alphabet;

    for (size_t strand_idx = 0; strand_idx < 2; ++strand_idx) {
        if (!r.read->has_events_for_strand(strand_idx)) continue;
        const size_t k = r.read->get_model_k(strand_idx);
        const PoreModel* motif_model = r.read->get_model(strand_idx, m_params.methylation_type);
        if (!motif_model) continue;                          // no model for this motif on this strand
        const std::vector<AlignedPair>& aligned_events = r.aligned_events[strand_idx];

        // scan for motifs, then batch them into groups separated by more than min_separation
        // (a site can only start where its first symbol stands — position 0 aside, where the reference's matcher also
        // accepts a string that lies wholly inside a site — so the full matcher runs on those positions only)
        bool first_symbol[256] = {false};
        for (size_t s = 0; s < alphabet->num_recognition_sites(); ++s) first_symbol[(unsigned char)alphabet->get_recognition_site(s)[0]] = true;
        std::vector<int> motif_sites;
        for (size_t i = 0; i + 1 < ref_seq.size(); ++i)
            if ((i == 0 || first_symbol[(unsigned char)ref_seq[i]]) && alphabet->is_motif_match(ref_seq, i)) motif_sites.push_back((int)i);
        std::vector<std::pair<size_t, size_t>> groups;
        size_t curr_idx = 0;
        while (curr_idx < motif_sites.size()) {
            size_t end_idx = curr_idx + 1;
            while (end_idx < motif_sites.size()) {
                if (motif_sites[end_idx] - motif_sites[end_idx - 1] > m_params.min_separation) break;
                end_idx += 1;
            }
            groups.push_back({curr_idx, end_idx});
            curr_idx = end_idx;
        }

        for (const auto& g : groups) {
            const size_t start_idx = g.first, end_idx = g.second;
            const int sub_start_pos = motif_sites[start_idx] - m_params.min_flank;
            const int sub_end_pos = motif_sites[end_idx - 1] + m_params.min_flank;
            const int span = motif_sites[end_idx - 1] - motif_sites[start_idx];
            if (sub_start_pos <= m_params.min_separation || span > 200) continue;

            std::string subseq = ref_seq.substr(sub_start_pos, sub_end_pos - sub_start_pos + 1);
            const int calling_start = sub_start_pos + r.ref_start_pos;
            const int calling_end = sub_end_pos + r.ref_start_pos;

            int e1 = 0, e2 = 0;
            const bool bounded = find_by_ref_bounds(aligned_events, calling_start, calling_end, e1, e2);
            // (the reference divides by calling_start - calling_end, a negative number, so this ratio never trips)
            const double ratio = std::fabs((double)(e2 - e1)) / (calling_start - calling_end);
            if (!bounded || std::abs(e2 - e1) <= 10 || ratio > MAX_EVENT_TO_BP_RATIO) continue;

            const uint32_t hmm_flags = HAF_ALLOW_PRE_CLIP | HAF_ALLOW_POST_CLIP;
            HMMInputData data;
            data.read = r.read;
            data.pore_model = motif_model;
            data.strand = (uint8_t)strand_idx;
            data.rc = r.rc[strand_idx];
            data.event_start_idx = (uint32_t)e1;
            data.event_stop_idx = (uint32_t)e2;
            data.event_stride = data.event_start_idx <= data.event_stop_idx ? 1 : -1;

            const int start_position = motif_sites[start_idx] + r.ref_start_pos;
            const int end_position = motif_sites[end_idx - 1] + r.ref_start_pos;
            // the reference scores first and filters by region afterwards; filtering first yields the same output
            if ((region_start != -1 && start_position < region_start) || (region_end != -1 && end_position >= region_end)) continue;

            std::string m_subseq = alphabet->methylate(subseq);
            // the jobs of this read only ever ask for the strand data.rc selects: the other strand's strings (the
            // reference builds all four) are left empty
            const bool need_rc = data.rc != 0;
            std::string rc_subseq = need_rc ? alphabet->reverse_complement(subseq) : std::string();
            std::string rc_m_subseq = need_rc ? alphabet->reverse_complement(m_subseq) : std::string();
            HMMInputSequence unmethylated(std::move(subseq), std::move(rc_subseq), alphabet);
            HMMInputSequence methylated(std::move(m_subseq), std::move(rc_m_subseq), alphabet);
            const size_t ju = m_batch.add(unmethylated, data, hmm_flags);
            const size_t jm = m_batch.add(methylated, data, hmm_flags);

            auto iter = site_score_map.find(start_position);
            if (iter == site_score_map.end()) {
                ScoredSite ss;
                ss.chromosome = r.contig;
                ss.start_position = start_position;
                ss.end_position = end_position;
                ss.n_motif = (int)(end_idx - start_idx);
                const size_t site_output_start = motif_sites[start_idx] - k + 1;
                const size_t site_output_end = motif_sites[end_idx - 1] + k;
                ss.sequence = ref_seq.substr(site_output_start, site_output_end - site_output_start);
                iter = site_score_map.insert({start_position, ss}).first;
            }
            m_pending.push_back(Pending{read_idx, start_position, strand_idx, ju, jm});
        }
    }
    return read_idx;
}

size_t MethylationCaller::add_reads(const std::vector<EventAlignedRead>& reads, int region_start, int region_end)
{
    const size_t first = m_reads.size();
    const size_t n = reads.size();
    if (m_mode == Mode::DeviceEnumeration) {
        std::vector<const EventAlignedRead*> ptrs(n);
        for (size_t i = 0; i < n; ++i) ptrs[i] = &reads[i];
        stage(ptrs.data(), n, region_start, region_end);
        return first;
    }
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)host_threads(), (n + 15) / 16));
    if (T == 1) {
        for (const EventAlignedRead& r : reads) add_read(r, region_start, region_end);
        return first;
    }
    // contiguous blocks of reads per worker: splicing the workers' lists in worker order reproduces the sequential order
    std::vector<std::unique_ptr<MethylationCaller>> locals((size_t)T);     // separately allocated: no false sharing of their cursors
    for (auto& l : locals) l.reset(new MethylationCaller(m_params, Mode::HostEnumeration));
    std::vector<std::string> errors((size_t)T);
#pragma omp parallel for schedule(static, 1) num_threads(T)
    for (int t = 0; t < T; ++t) {
        const size_t b = n * (size_t)t / (size_t)T, e = n * ((size_t)t + 1) / (size_t)T;
        try {
            for (size_t i = b; i < e; ++i) locals[t]->add_read(reads[i], region_start, region_end);
        } catch (const std::exception& ex) { errors[t] = ex.what(); }
    }
    for (const std::string& e : errors) if (!e.empty()) throw Error(NPH_ERR_INVALID, e);
    for (int t = 0; t < T; ++t) {
        MethylationCaller& l = *locals[t];
        const size_t read_base = m_reads.size(), job_base = m_batch.size();
        for (Pending p : l.m_pending) { p.read += read_base; p.job_u += job_base; p.job_m += job_base; m_pending.push_back(p); }
        for (ReadEntry& re : l.m_reads) m_reads.push_back(std::move(re));
        m_batch.append(std::move(l.m_batch));
    }
    return first;
}

void MethylationCaller::run(Engine& engine, double indel_bias)
{
    if (m_mode == Mode::DeviceEnumeration) {
        m_site_off.assign(m_records.size() + 1, 0);
        m_n_sites = 0; m_scored_events = 0;
        for (ReadEntry& re : m_reads) { re.sites.clear(); re.sites_built = false; }
        m_ran = true;
        if (m_records.empty()) return;
        // one nph_read per distinct (SquiggleRead, strand); consecutive records of one read are the common case
        std::vector<std::pair<const SquiggleRead*, uint8_t>> uniq;
        std::map<std::pair<const SquiggleRead*, uint8_t>, uint32_t> index;
        uint32_t k = 0;
        for (size_t i = 0; i < m_records.size(); ++i) {
            const Record& rm = m_record_meta[i];
            const std::pair<const SquiggleRead*, uint8_t> key(rm.read, rm.strand);
            uint32_t ridx;
            if (!uniq.empty() && uniq.back() == key) ridx = (uint32_t)uniq.size() - 1;
            else {
                auto it = index.find(key);
                if (it == index.end()) { ridx = (uint32_t)uniq.size(); index[key] = ridx; uniq.push_back(key); }
                else ridx = it->second;
            }
            m_records[i].read = ridx;
            m_records[i].model_id = engine.model_id(rm.model);
            if (k && rm.model->k != k) throw Error(NPH_ERR_UNSUPPORTED, "models with different k in one call-methylation batch");
            k = rm.model->k;
        }
        const detail::FlatReads fr = detail::flatten_reads(engine, uniq);
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
        return;
    }
    const std::vector<float> ll = m_batch.run(engine, indel_bias);
    for (const Pending& p : m_pending) {
        ScoredSite& ss = m_reads[p.read].sites[p.site_key];
        ss.ll_unmethylated[p.strand] = ll[p.job_u];       // float -> double, like `double s = profile_hmm_score(...)`
        ss.ll_methylated[p.strand] = ll[p.job_m];
        ss.strands_scored += 1;
    }
    m_pending.clear();
    m_batch.clear();
}

// one TSV row (write_methylation_results_as_tsv, call_methylation.cpp:532-550): chromosome, strand, start, end, read_name,
// log_lik_ratio %.2lf, log_lik_methylated %.2lf, log_lik_unmethylated %.2lf, num_calling_strands, num_motifs, sequence.
// Rows are written straight into a growing character buffer: "%d" by a reversed-digit loop, "%.2lf" by format_fixed (exact
// integer arithmetic, nph_host.cpp) — no printf and no per-field string appends.
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
inline char* put_uint(char* o, uint32_t v)
{
    char tmp[12];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10u); v /= 10u; } while (v);
    while (n) *o++ = tmp[--n];
    return o;
}
inline char* put_int(char* o, int v)
{
    if (v < 0) { *o++ = '-'; return put_uint(o, (uint32_t)(-(int64_t)v)); }
    return put_uint(o, (uint32_t)v);
}
const size_t kRowOverhead = 3 * 48 + 64;            // three %.2lf fields (format_fixed falls back to printf beyond 2^52), integers, tabs
inline void put_row(RowBuffer& out, const char* chromosome, size_t chromosome_len, bool is_reverse, int start_position, int end_position,
                    const char* name, size_t name_len, double sum_ll_m, double sum_ll_u, int strands_scored, int n_motif,
                    const char* sequence, size_t sequence_len)
{
    char* o = out.room(chromosome_len + name_len + sequence_len + kRowOverhead);
    char* const o0 = o;
    const double diff = sum_ll_m - sum_ll_u;
    std::memcpy(o, chromosome, chromosome_len); o += chromosome_len;
    *o++ = '\t'; *o++ = is_reverse ? '-' : '+'; *o++ = '\t';
    o = put_int(o, start_position); *o++ = '\t';
    o = put_int(o, end_position); *o++ = '\t';
    std::memcpy(o, name, name_len); o += name_len; *o++ = '\t';
    o += format_fixed(o, diff, 2); *o++ = '\t';
    o += format_fixed(o, sum_ll_m, 2); *o++ = '\t';
    o += format_fixed(o, sum_ll_u, 2); *o++ = '\t';
    o = put_int(o, strands_scored); *o++ = '\t';
    o = put_int(o, n_motif); *o++ = '\t';
    std::memcpy(o, sequence, sequence_len); o += sequence_len;
    *o++ = '\n';
    out.n += (size_t)(o - o0);
}
} // namespace

// Device mode: the ScoredSite map of one read from its site records (the strands of a read meet at start_position,
// exactly as the reference's find-or-insert does, basemods.cpp:403-425).
void MethylationCaller::build_sites(size_t read_idx) const
{
    const ReadEntry& re = m_reads[read_idx];
    if (re.sites_built) return;
    if (!m_ran) throw Error(NPH_ERR_STATE, "MethylationCaller::sites before run()");
    const char* ref = m_ref.data() + re.ref_off;
    for (size_t rec = re.first_record; rec < re.first_record + re.n_records; ++rec) {
        const size_t strand = m_records[rec].strand;
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
                const size_t site_output_start = (size_t)(ms.start_position - re.ref_start_pos) - re.k + 1;
                const size_t site_output_end = std::min<size_t>((size_t)(ms.end_position - re.ref_start_pos) + re.k, re.ref_len);
                ss.sequence.assign(ref + site_output_start, site_output_end - site_output_start);
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
    if (m_mode == Mode::DeviceEnumeration) build_sites(read_idx);
    return m_reads[read_idx].sites;
}

// rows of a record that is its read's only scored strand: the site records are already the rows, in ascending position
static void put_single_strand_rows(RowBuffer& out, const std::string& contig, bool is_reverse, const char* name, size_t name_len, const char* ref,
                                   size_t ref_len, int ref_start_pos, uint32_t k, size_t strand, const nph_meth_site* sites, size_t n)
{
    for (size_t s = 0; s < n; ++s) {
        const nph_meth_site& ms = sites[s];
        double ll_m[2] = {0, 0}, ll_u[2] = {0, 0};
        ll_m[strand] = ms.ll_methylated; ll_u[strand] = ms.ll_unmethylated;       // the other strand's entries stay 0, as in a fresh ScoredSite
        const size_t b = (size_t)(ms.start_position - ref_start_pos) - k + 1;
        const size_t e = std::min<size_t>((size_t)(ms.end_position - ref_start_pos) + k, ref_len);
        put_row(out, contig.data(), contig.size(), is_reverse, ms.start_position, ms.end_position, name, name_len, ll_m[0] + ll_m[1], ll_u[0] + ll_u[1], 1,
                (int)ms.n_motif, ref + b, e - b);
    }
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
    if (m_mode == Mode::DeviceEnumeration && re.n_records == 1 && !re.sites_built) {
        if (!m_ran) throw Error(NPH_ERR_STATE, "MethylationCaller::tsv before run()");
        const size_t rec = re.first_record;
        put_single_strand_rows(out, re.contig, re.is_reverse, re.name.data(), re.name.size(), m_ref.data() + re.ref_off, re.ref_len, re.ref_start_pos,
                               re.k, m_records[rec].strand, m_sites.data() + m_site_off[rec], (size_t)(m_site_off[rec + 1] - m_site_off[rec]));
        return;
    }
    for (const auto& kv : sites(read_idx)) {
        const ScoredSite& ss = kv.second;
        put_row(out, ss.chromosome.data(), ss.chromosome.size(), re.is_reverse, ss.start_position, ss.end_position, re.name.data(), re.name.size(),
                ss.ll_methylated[0] + ss.ll_methylated[1], ss.ll_unmethylated[0] + ss.ll_unmethylated[1], ss.strands_scored, ss.n_motif,
                ss.sequence.data(), ss.sequence.size());
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
#pragma omp parallel for schedule(dynamic, 16) num_threads(host_threads()) if (m_reads.size() > 64)
    for (long long i = 0; i < (long long)m_reads.size(); ++i) out[i] = tsv((size_t)i);
    return out;
}

size_t MethylationCaller::tsv_all(char* out, size_t cap) const
{
    // contiguous blocks of reads per worker: format into a private buffer, then copy to the block's offset
    const size_t n = m_reads.size();
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)host_threads(), (n + 63) / 64));
    std::vector<RowBuffer> parts((size_t)T);
    std::vector<std::string> errors((size_t)T);
#pragma omp parallel for schedule(static, 1) num_threads(T) if (T > 1)
    for (int t = 0; t < T; ++t) {
        const size_t b = n * (size_t)t / (size_t)T, e = n * ((size_t)t + 1) / (size_t)T;
        try {
            parts[t].room((e - b) * 4096);
            for (size_t i = b; i < e; ++i) put_rows(&parts[t], i);
        } catch (const std::exception& ex) { errors[t] = ex.what(); }
    }
    for (const std::string& e : errors) if (!e.empty()) throw Error(NPH_ERR_INVALID, e);
    std::vector<size_t> off((size_t)T + 1, 0);
    for (int t = 0; t < T; ++t) off[t + 1] = off[t] + parts[t].n;
    if (off[T] > cap || !out) return off[T];
#pragma omp parallel for schedule(static, 1) num_threads(T) if (T > 1)
    for (int t = 0; t < T; ++t) if (parts[t].n) std::memcpy(out + off[t], parts[t].p.get(), parts[t].n);
    return off[T];
}

// The whole of call-methylation for a batch that already sits in flat host buffers (the layout of nph_methylation_batch):
// device call(s), then the TSV rows formatted by host_threads() workers straight from the site records.  A large batch whose
// records map one-to-one onto its reads is cut into four sub-batches and pipelined: while the device scores sub-batch i + 1
// (the calling thread sits in the driver), the workers format the rows of sub-batch i — the two stages cost about the same,
// so the batch takes roughly max(device, TSV) + a quarter of each instead of their sum.
namespace {
void format_records(const FlatMethylationBatch& b, uint32_t k, size_t rec_lo, size_t rec_hi, const uint64_t* site_off /* relative to rec_lo */,
                    const nph_meth_site* sites, std::vector<RowBuffer>& parts)
{
    const size_t n = rec_hi - rec_lo;
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)host_threads(), (n + 63) / 64));
    parts.clear();
    parts.resize((size_t)T);
    const std::string contig(b.contig ? b.contig : "");
#pragma omp parallel for schedule(static, 1) num_threads(T) if (T > 1)
    for (int t = 0; t < T; ++t) {
        const size_t lo = n * (size_t)t / (size_t)T, hi = n * ((size_t)t + 1) / (size_t)T;
        RowBuffer& out = parts[t];
        out.room((size_t)(site_off[hi] - site_off[lo]) * 96 + 64);
        for (size_t r = lo; r < hi; ++r) {
            const nph_meth_record& rec = b.records[rec_lo + r];
            const char* name = b.read_names[rec_lo + r];
            put_single_strand_rows(out, contig, b.is_reverse[rec_lo + r] != 0, name, std::strlen(name), b.ref_bases + rec.ref_off, rec.ref_len,
                                   rec.ref_start_pos, k, rec.strand, sites + site_off[r], (size_t)(site_off[r + 1] - site_off[r]));
        }
    }
}
} // namespace

size_t call_methylation_flat(Engine& engine, const FlatMethylationBatch& b, const MethylationCallingParameters& params, uint32_t k,
                             double indel_bias, char* tsv_out, size_t cap, FlatMethylationStats* stats)
{
    auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    const nph_meth_params mp = make_meth_params(params, k, b.region_start, b.region_end);
    const size_t n = b.n_records;
    // sub-batches need records i <-> reads i with events and (compact) alignments laid out in that order
    bool identity = b.event_deltas != nullptr && n == b.n_reads && n >= 2048;
    for (size_t r = 0; identity && r < n; ++r)
        identity = b.records[r].read == r && (r == 0 || (b.reads[r].event_off == b.reads[r - 1].event_off + b.reads[r - 1].n_events &&
                                                         b.records[r].ref_off == b.records[r - 1].ref_off + b.records[r - 1].ref_len));
    // One call rather than pipelined sub-batches: every sub-batch pays the
    // call's fixed costs (two read-backs, ten class launches, the scheduler) and the formatter's thread teams compete with the driver
    // thread for the container's CPU quota.  One call it is; the sub-batch path stays behind $NPH_METH_PIPELINE for larger batches.
    static const bool want_pipeline = std::getenv("NPH_METH_PIPELINE") != nullptr;
    // Rows formatted on the device (nph_methylation_batch_compact_tsv): the site records never leave it and the host's share of the call
    // is the name table.  Needs the compact event alignment and a destination; $NPH_METH_HOST_TSV keeps the host formatter (A/B, tests).
    static const bool host_tsv = std::getenv("NPH_METH_HOST_TSV") != nullptr;
    if (b.event_deltas && tsv_out && !host_tsv && !want_pipeline && n > 0) {
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
    const size_t n_chunks = (identity && want_pipeline) ? 4 : 1;
    std::vector<size_t> cut(n_chunks + 1);
    for (size_t c = 0; c <= n_chunks; ++c) cut[c] = n * c / n_chunks;
    std::vector<size_t> site_cap(n_chunks, 0);
    size_t site_cap_total = 0;
    for (size_t c = 0; c < n_chunks; ++c) {
        for (size_t r = cut[c]; r < cut[c + 1]; ++r) site_cap[c] += b.records[r].ref_len / (size_t)(params.min_separation + 1) + 2;
        site_cap_total += site_cap[c];
    }
    nph_meth_site* sites = static_cast<nph_meth_site*>(engine.pinned(3, sizeof(nph_meth_site) * std::max<size_t>(site_cap_total, 1)));
    std::vector<std::vector<uint64_t>> site_off(n_chunks);
    std::vector<std::vector<RowBuffer>> parts(n_chunks);
    std::vector<nph_read> sub_reads;
    std::vector<nph_meth_record> sub_recs;
    uint64_t scored_total = 0, sites_total = 0;
    double device_s = 0.0;
    std::string error;
    std::thread formatter;
    size_t site_base = 0;
    for (size_t c = 0; c < n_chunks; ++c) {
        const size_t lo = cut[c], hi = cut[c + 1], m = hi - lo;
        site_off[c].assign(m + 1, 0);
        uint64_t scored = 0;
        const double td = now();
        int rc;
        if (n_chunks == 1) {
            rc = b.event_deltas
                ? nph_methylation_batch_compact(engine.ctx(), b.reads, b.n_reads, b.ev_mean, b.ev_start_time, b.n_events, b.ref_bases, b.event_deltas,
                                                b.n_ref, b.first_event, b.records, n, &mp, indel_bias, site_off[c].data(), sites, site_cap_total, &scored)
                : nph_methylation_batch(engine.ctx(), b.reads, b.n_reads, b.ev_mean, b.ev_start_time, b.n_events, b.ref_bases, b.n_ref,
                                        b.aligned_events, b.n_pairs, b.records, n, &mp, indel_bias, site_off[c].data(), sites, site_cap_total, &scored);
        } else {
            // the sub-batch's slices of the event, reference and alignment arrays, offsets rebased to the slice
            const uint64_t ev0 = b.reads[lo].event_off, ref0 = b.records[lo].ref_off;
            const uint64_t ev1 = b.reads[hi - 1].event_off + b.reads[hi - 1].n_events, ref1 = b.records[hi - 1].ref_off + b.records[hi - 1].ref_len;
            sub_reads.assign(b.reads + lo, b.reads + hi);
            sub_recs.assign(b.records + lo, b.records + hi);
            for (size_t i = 0; i < m; ++i) { sub_reads[i].event_off -= ev0; sub_recs[i].ref_off -= ref0; sub_recs[i].read = (uint32_t)i; }
            rc = nph_methylation_batch_compact(engine.ctx(), sub_reads.data(), m, b.ev_mean + ev0, b.ev_start_time ? b.ev_start_time + ev0 : nullptr,
                                               (size_t)(ev1 - ev0), b.ref_bases + ref0, b.event_deltas + ref0, (size_t)(ref1 - ref0), b.first_event + lo,
                                               sub_recs.data(), m, &mp, indel_bias, site_off[c].data(), sites + site_base, site_cap[c], &scored);
        }
        device_s += now() - td;
        if (formatter.joinable()) formatter.join();
        engine.check(rc, b.event_deltas ? "nph_methylation_batch_compact" : "nph_methylation_batch");
        scored_total += scored; sites_total += site_off[c][m];
        const nph_meth_site* chunk_sites = sites + site_base;
        // (the site records of a sub-batch carry sub-batch record numbers; the formatter only needs them per record, by offset)
        formatter = std::thread([&, c, lo, hi, chunk_sites] {
            try { format_records(b, k, lo, hi, site_off[c].data(), chunk_sites, parts[c]); }
            catch (const std::exception& ex) { error = ex.what(); }
        });
        site_base += site_cap[c];
    }
    if (formatter.joinable()) formatter.join();
    if (!error.empty()) throw Error(NPH_ERR_INVALID, error);
    const double t1 = now();
    size_t total = 0;
    std::vector<std::pair<const RowBuffer*, size_t>> pieces;
    for (size_t c = 0; c < n_chunks; ++c) for (const RowBuffer& rb : parts[c]) { pieces.push_back({&rb, total}); total += rb.n; }
    if (stats) { stats->n_sites = sites_total; stats->scored_events = scored_total; }
    if (tsv_out && total <= cap) {
#pragma omp parallel for schedule(static, 1) num_threads(host_threads()) if (pieces.size() > 1)
        for (long long i = 0; i < (long long)pieces.size(); ++i)
            if (pieces[(size_t)i].first->n) std::memcpy(tsv_out + pieces[(size_t)i].second, pieces[(size_t)i].first->p.get(), pieces[(size_t)i].first->n);
    }
    // device_seconds: time inside the device calls (the formatter of the previous sub-batch runs concurrently); tsv_seconds: what the
    // formatting added on top — the last sub-batch's rows and the final copy
    if (stats) { stats->device_seconds = device_s; stats->tsv_seconds = (now() - t0) - device_s; (void)t1; }
    return total;
}

void MethylationCaller::write_tsv(FILE* fp, size_t read_idx) const
{
    const std::string s = tsv(read_idx);
    fwrite(s.data(), 1, s.size(), fp);
}

} // namespace nph
