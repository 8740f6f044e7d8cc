// nph_variants.cpp — see nph_variants.hpp (SURVEY.md section 8f, row N2).
#include "nph_variants.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <iomanip>
#include <sstream>

namespace nph {

const size_t Haplotype::INSERTED_POSITION = std::string::npos;

Haplotype::Haplotype(const std::string& ref_name, size_t ref_position, const std::string& ref_sequence)
    : m_ref_name(ref_name), m_ref_position(ref_position), m_reference(ref_sequence), m_sequence(ref_sequence)
{
    m_coordinate_map.resize(m_reference.size());
    for (size_t i = 0; i < m_coordinate_map.size(); ++i) m_coordinate_map[i] = m_ref_position + i;
}

// The first base with a reference position >= ref_index (the reference scans linearly).  The positions of the bases that have one
// ascend, so the position of the first such base at or after i is a non-decreasing function of i: a bisection over i finds it.
size_t Haplotype::find_derived_index_by_ref_lower_bound(size_t ref_index) const
{
    const size_t n = m_coordinate_map.size();
    const auto next = [&](size_t i) { while (i < n && m_coordinate_map[i] == INSERTED_POSITION) ++i; return i; };
    size_t lo = 0, hi = n;
    while (lo < hi) {
        const size_t mid = lo + (hi - lo) / 2, j = next(mid);
        if (j == n || m_coordinate_map[j] >= ref_index) hi = mid;
        else lo = j + 1;
    }
    return next(lo);
}

// Replace ref_seq by alt_seq at the haplotype position that still maps to v.ref_position; refuse (leaving the
// haplotype untouched) when that reference base was already replaced or the reference allele does not match.
bool Haplotype::apply_variant(const Variant& v)
{
    const size_t idx = find_derived_index_by_ref_lower_bound(v.ref_position);
    if (idx == m_coordinate_map.size() || m_coordinate_map[idx] != v.ref_position) return false;
    const size_t rl = v.ref_seq.length(), al = v.alt_seq.length();
    if (m_sequence.substr(idx, rl) != v.ref_seq) return false;
    m_sequence.replace(idx, rl, v.alt_seq);
    auto first = m_coordinate_map.begin() + idx;
    auto it = m_coordinate_map.erase(first, first + rl);
    m_coordinate_map.insert(it, al, INSERTED_POSITION);     // inserted bases have no reference coordinate
    m_variants.push_back(v);
    return true;
}

bool Haplotype::apply_variants(const std::vector<Variant>& variants)
{
    bool good = true;
    for (const Variant& v : variants) good = good && apply_variant(v);
    return good;
}

size_t Haplotype::get_reference_position_for_haplotype_base(size_t i) const
{
    return m_coordinate_map[i] == INSERTED_POSITION ? std::string::npos : m_coordinate_map[i];
}

Haplotype Haplotype::substr_by_reference(size_t start, size_t end) const
{
    if (start < m_ref_position || start > get_reference_end() || end < m_ref_position || end > get_reference_end())
        throw Error(NPH_ERR_INVALID, "substr_by_reference: range outside the haplotype");
    size_t s = find_derived_index_by_ref_lower_bound(start);
    const size_t e = find_derived_index_by_ref_lower_bound(end);
    while (s >= m_coordinate_map.size() || m_coordinate_map[s] == INSERTED_POSITION || m_coordinate_map[s] > start) {
        if (s == 0) throw Error(NPH_ERR_INVALID, "substr_by_reference: no base at or before the start");
        --s;
    }
    if (e == m_coordinate_map.size()) throw Error(NPH_ERR_INVALID, "substr_by_reference: no base at or after the end");
    start = m_coordinate_map[s];
    end = m_coordinate_map[e];
    Haplotype ret(m_ref_name, start, m_reference.substr(start - m_ref_position, end - start + 1));
    ret.m_sequence = m_sequence.substr(s, e - s + 1);
    ret.m_coordinate_map.assign(m_coordinate_map.begin() + s, m_coordinate_map.begin() + e + 1);
    return ret;
}

void Haplotype::get_enclosing_reference_range_for_haplotype_range(size_t& hap_lower, size_t& hap_upper, size_t& ref_lower, size_t& ref_upper) const
{
    while (hap_lower > 0 && m_coordinate_map[hap_lower] == INSERTED_POSITION) --hap_lower;
    while (hap_upper < m_coordinate_map.size() && m_coordinate_map[hap_upper] == INSERTED_POSITION) ++hap_upper;
    if (hap_lower == 0 || hap_upper >= m_coordinate_map.size()) {
        hap_lower = hap_upper = ref_lower = ref_upper = std::string::npos;
    } else {
        ref_lower = m_coordinate_map[hap_lower];
        ref_upper = m_coordinate_map[hap_upper];
    }
}

std::vector<HMMInputSequence> generate_methylated_alternatives(const HMMInputSequence& sequence,
                                                               const std::vector<std::string>& methylation_types)
{
    std::vector<HMMInputSequence> out;
    out.push_back(sequence);
    for (const std::string& name : methylation_types) {
        const Alphabet* alphabet = get_alphabet_by_name(name);
        std::string methylated = alphabet->methylate(sequence.get_sequence());
        if (methylated != sequence.get_sequence()) out.emplace_back(methylated, alphabet);
    }
    return out;
}

namespace {

// Adds the jobs of profile_hmm_score_set(sequences, data) to the batch; returns (first job, count).
// `ranks` has one RankCache per sequence: a haplotype is scored against every read of the pile-up, its k-mer ranks are
// computed and shipped once per strand.
std::pair<size_t, size_t> add_score_set(HmmBatch& batch, const std::vector<HMMInputSequence>& sequences, std::vector<RankCache>& ranks,
                                        const HMMInputData& data, uint32_t flags)
{
    const size_t first = batch.size();
    ranks.resize(sequences.size());
    batch.add(sequences[0], data, flags, ranks[0]);
    for (size_t i = 1; i < sequences.size(); ++i) {
        HMMInputData alt = data;
        alt.pore_model = data.read->get_model(data.strand, sequences[i].get_alphabet()->get_name());
        if (!alt.pore_model) throw Error(NPH_ERR_INVALID, std::string("read has no pore model for alphabet ") + sequences[i].get_alphabet()->get_name());
        batch.add(sequences[i], alt, flags, ranks[i]);
    }
    return {first, sequences.size()};
}

double combine(const std::vector<float>& scores, std::pair<size_t, size_t> span)
{
    float out = 0.0f;
    int rc = nph_score_set_combine(scores.data() + span.first, 1, (uint32_t)span.second, &out);
    if (rc != NPH_OK) throw Error(rc, "nph_score_set_combine");
    return out;     // profile_hmm_score_set returns float; callers hold it in a double
}

} // namespace

std::vector<std::vector<double>> score_haplotypes(const std::vector<Haplotype>& haplotypes, const std::vector<HMMInputData>& input,
                                                  uint32_t alignment_flags, const std::vector<std::string>& methylation_types,
                                                  Engine& engine, double indel_bias)
{
    HmmBatch batch;
    std::vector<std::vector<HMMInputSequence>> alts;
    for (const Haplotype& h : haplotypes) alts.push_back(generate_methylated_alternatives(HMMInputSequence(h.get_sequence()), methylation_types));
    std::vector<std::vector<RankCache>> alt_ranks(haplotypes.size());
    std::vector<std::vector<std::pair<size_t, size_t>>> spans(input.size(), std::vector<std::pair<size_t, size_t>>(haplotypes.size()));
    for (size_t ri = 0; ri < input.size(); ++ri)
        for (size_t hi = 0; hi < haplotypes.size(); ++hi) spans[ri][hi] = add_score_set(batch, alts[hi], alt_ranks[hi], input[ri], alignment_flags);
    const std::vector<float> s = batch.run(engine, indel_bias);
    std::vector<std::vector<double>> out(input.size(), std::vector<double>(haplotypes.size()));
    for (size_t ri = 0; ri < input.size(); ++ri)
        for (size_t hi = 0; hi < haplotypes.size(); ++hi) out[ri][hi] = combine(s, spans[ri][hi]);
    return out;
}

size_t nChoosek(size_t n, size_t k)
{
    if (k > n) return 0;
    if (k * 2 > n) k = n - k;
    if (k == 0) return 1;
    int result = (int)n;                                       // the reference accumulates in an int
    for (int i = 2; i <= (int)k; ++i) {
        result *= (int)(n - i + 1);
        result /= i;
    }
    return (size_t)result;
}

VariantCombinations variant_combinations(const std::vector<Variant>& variants, const Haplotype& base_haplotype, int max_haplotypes)
{
    const size_t num_variants = variants.size();
    // the largest number of variants that can be tested jointly without exceeding max_haplotypes
    size_t sum_num_haplotypes = 0, max_r = 1;
    while (max_r <= num_variants) {
        const size_t num_haplotypes_r = nChoosek(num_variants, max_r);
        if (num_haplotypes_r + sum_num_haplotypes < (size_t)max_haplotypes) sum_num_haplotypes += num_haplotypes_r;
        else break;
        max_r += 1;
    }
    max_r -= 1;
    VariantCombinations out;
    out.max_r = max_r;
    for (size_t r = 0; r <= max_r; ++r) {
        std::vector<size_t> idx(r);
        for (size_t i = 0; i < r; ++i) idx[i] = i;
        for (;;) {
            Haplotype current = base_haplotype;
            std::vector<Variant> subset;
            for (size_t i : idx) subset.push_back(variants[i]);
            if (current.apply_variants(subset)) { out.combinations.push_back(idx); out.haplotypes.push_back(current); }
            // next r-subset of {0..n-1} in lexicographic order
            int i = (int)r - 1;
            while (i >= 0 && idx[i] == num_variants - r + (size_t)i) --i;
            if (i < 0) break;
            ++idx[i];
            for (size_t j = (size_t)i + 1; j < r; ++j) idx[j] = idx[j - 1] + 1;
        }
    }
    return out;
}

VariantGroupScores score_variant_group(const std::vector<Variant>& variants, const Haplotype& base_haplotype,
                                       const std::vector<HMMInputData>& input, int max_haplotypes, uint32_t alignment_flags,
                                       const std::vector<std::string>& methylation_types, Engine& engine, double indel_bias)
{
    VariantCombinations vc = variant_combinations(variants, base_haplotype, max_haplotypes);
    VariantGroupScores out;
    out.max_r = vc.max_r;
    out.combinations = std::move(vc.combinations);
    const std::vector<Haplotype>& haplotypes = vc.haplotypes;
    const std::vector<std::vector<double>> by_read = score_haplotypes(haplotypes, input, alignment_flags, methylation_types, engine, indel_bias);
    out.scores.assign(haplotypes.size(), std::vector<double>(input.size()));
    for (size_t ri = 0; ri < input.size(); ++ri)
        for (size_t hi = 0; hi < haplotypes.size(); ++hi) out.scores[hi][ri] = by_read[ri][hi];
    return out;
}

std::vector<Variant> score_variants_thresholded(const std::vector<Variant>& input_variants, const Haplotype& base_haplotype,
                                                const std::vector<HMMInputData>& input, uint32_t alignment_flags,
                                                uint32_t score_threshold, const std::vector<std::string>& methylation_types,
                                                Engine& engine, double indel_bias)
{
    std::vector<Variant> out = input_variants;
    HmmBatch batch;
    const std::vector<HMMInputSequence> base_seqs =
        generate_methylated_alternatives(HMMInputSequence(base_haplotype.get_sequence()), methylation_types);
    std::vector<std::pair<size_t, size_t>> base_span(input.size());
    std::vector<RankCache> base_ranks;
    for (size_t j = 0; j < input.size(); ++j) base_span[j] = add_score_set(batch, base_seqs, base_ranks, input[j], alignment_flags);   // once per read

    std::vector<char> applies(input_variants.size(), 0);
    std::vector<std::vector<std::pair<size_t, size_t>>> var_span(input_variants.size());
    for (size_t v = 0; v < input_variants.size(); ++v) {
        Haplotype hap = base_haplotype;
        // the reference applies the variant without checking the result: an incompatible variant leaves the
        // haplotype unchanged, so variant_score == base_score and the quality stays 0
        applies[v] = hap.apply_variant(input_variants[v]) ? 1 : 0;
        if (!applies[v]) continue;
        const std::vector<HMMInputSequence> seqs = generate_methylated_alternatives(HMMInputSequence(hap.get_sequence()), methylation_types);
        var_span[v].resize(input.size());
        std::vector<RankCache> var_ranks;
        for (size_t j = 0; j < input.size(); ++j) var_span[v][j] = add_score_set(batch, seqs, var_ranks, input[j], alignment_flags);
    }
    const std::vector<float> s = batch.run(engine, indel_bias);
    std::vector<double> base(input.size());
    for (size_t j = 0; j < input.size(); ++j) base[j] = combine(s, base_span[j]);
    for (size_t v = 0; v < input_variants.size(); ++v) {
        double total = 0.0f;
        if (applies[v]) {
            for (size_t j = 0; j < input.size(); ++j) {
                if (std::fabs(total) < score_threshold) total += (combine(s, var_span[v][j]) - base[j]);
            }
        }
        out[v].quality = total;
    }
    return out;
}

Variant score_variant_thresholded(const Variant& input_variant, Haplotype base_haplotype, const std::vector<HMMInputData>& input,
                                  uint32_t alignment_flags, uint32_t score_threshold, const std::vector<std::string>& methylation_types)
{
    return score_variants_thresholded({input_variant}, base_haplotype, input, alignment_flags, score_threshold, methylation_types,
                                      Engine::thread_default())[0];
}

std::vector<HomopolymerWindow> homopolymer_windows(const Haplotype& haplotype, int region_start, int region_end, int min_flanking_sequence)
{
    const std::string& s = haplotype.get_sequence();
    const size_t flank = (size_t)min_flanking_sequence, k = 6;
    std::vector<HomopolymerWindow> out;
    size_t i = 0;
    while (i < s.size()) {
        const char hp_base = s[i];
        const size_t hap_hp_start = i;
        while (i < s.size() && s[i] == hp_base) ++i;
        if (i >= s.size()) break;                                           // the last run is never considered
        const size_t hap_hp_end = i, hp_length = hap_hp_end - hap_hp_start;
        if (hp_length < NPH_HP_MIN_LENGTH || hp_length > NPH_HP_MAX_LENGTH) continue;
        if (hap_hp_start < flank || hap_hp_end + flank >= s.size()) continue;
        size_t hap_calling_start = hap_hp_start - flank, hap_calling_end = hap_hp_end + flank, ref_calling_start, ref_calling_end;
        haplotype.get_enclosing_reference_range_for_haplotype_range(hap_calling_start, hap_calling_end, ref_calling_start, ref_calling_end);
        if (ref_calling_start == std::string::npos || ref_calling_end == std::string::npos) continue;
        if (ref_calling_start < (size_t)region_start || ref_calling_end >= (size_t)region_end) continue;
        if (ref_calling_start < haplotype.get_reference_position() || ref_calling_end >= haplotype.get_reference_end()) continue;
        HomopolymerWindow w;
        w.hp_start = hap_hp_start; w.hp_end = hap_hp_end;
        w.calling = haplotype.substr_by_reference(ref_calling_start, ref_calling_end).get_sequence();
        std::memset(&w.dev, 0, sizeof(w.dev));
        w.dev.seq_len = (uint32_t)w.calling.size();
        w.dev.ref_calling_start = (int32_t)ref_calling_start; w.dev.ref_calling_end = (int32_t)ref_calling_end;
        w.dev.edit_offset = (uint32_t)(hap_hp_start - hap_calling_start);
        w.dev.k0 = (uint32_t)(hap_hp_start - hap_calling_start - k + 1);
        w.dev.hp_length = (uint32_t)hp_length; w.dev.hp_base = hp_base; w.dev.k = (uint32_t)k;
        out.push_back(std::move(w));
    }
    return out;
}

HomopolymerCall homopolymer_call(const nph_hp_likelihoods& lik, size_t hp_length)
{
    double score_by_length[NPH_HP_MAX_LENGTH + 1] = {};
    double max_score = -INFINITY;
    size_t call = (size_t)-1;
    for (size_t len = NPH_HP_MIN_LENGTH; len <= NPH_HP_MAX_LENGTH; ++len) {
        const double score = lik.duration_lik[len - NPH_HP_MIN_LENGTH] + lik.event_lik[len - NPH_HP_MIN_LENGTH];
        score_by_length[len] = score;
        if (score > max_score) { max_score = score; call = len; }
    }
    HomopolymerCall out;
    out.call = call;
    out.quality = max_score - score_by_length[hp_length];
    out.size_diff = (int)(call - hp_length);
    out.kept = !(out.quality < 10);
    return out;
}

namespace {

// The region in screening's flat layout: per record its compact event alignment over the span of its aligned_events, the reads
// its records name, and their event start times
struct RegionLayout {
    detail::ReadTable reads;
    std::vector<nph_meth_record> recs;
    std::vector<int16_t> deltas;
    std::vector<int32_t> first;
    detail::FlatReads fr;
    std::vector<double> time;
};

RegionLayout region_layout(const HomopolymerRegion& region, Engine& engine, const char* caller)
{
    RegionLayout rl;
    for (const EventAlignedRead& r : region.records) {
        const std::vector<AlignedPair>& ae = r.aligned_events[0];
        nph_meth_record rec;
        std::memset(&rec, 0, sizeof(rec));
        rec.read = rl.reads.index(r.read, 0);
        rec.model_id = engine.model_id(r.read->get_base_model(0));
        rec.rc = r.rc[0] ? 1 : 0;
        rec.ref_off = rl.deltas.size();
        int32_t f = 0;
        if (!ae.empty() && r.read->has_events_for_strand(0)) {
            rec.ref_start_pos = ae.front().ref_pos;
            rec.ref_len = (uint32_t)(ae.back().ref_pos - ae.front().ref_pos + 1);
            rl.deltas.resize(rl.deltas.size() + rec.ref_len);
            if (!compact_event_alignment(ae, rec.ref_start_pos, rec.ref_len, rl.deltas.data() + rec.ref_off, &f))
                throw Error(NPH_ERR_UNSUPPORTED, std::string(caller) + ": an event alignment with a step beyond int16");
        }
        rl.first.push_back(f);
        rl.recs.push_back(rec);
    }
    rl.fr = detail::flatten_reads(engine, rl.reads);
    rl.time.resize(std::max<size_t>(rl.fr.n_events, 1));
    for (size_t i = 0; i < rl.reads.size(); ++i) {
        const std::vector<SquiggleEvent>& ev = rl.reads.reads()[i].first->events[rl.reads.reads()[i].second];
        for (size_t e = 0; e < ev.size(); ++e) rl.time[rl.fr.reads[i].event_off + e] = ev[e].start_time;
    }
    return rl;
}

// The -q types as the device calls take them: each alphabet, and per record the read's model of each type (SquiggleRead::get_model,
// as profile_hmm_score_set asks), plus one trailing id so that the array is never empty
void methylation_args(const RegionAlignments& alignments, const std::vector<std::string>& methylation_types, uint32_t k, Engine& engine,
                      const char* caller, nph_screen_methylation& meth, std::vector<uint32_t>& alt_models)
{
    std::memset(&meth, 0, sizeof(meth));
    if (methylation_types.size() > NPH_SCREEN_MAX_TYPES) throw Error(NPH_ERR_INVALID, std::string(caller) + ": more than NPH_SCREEN_MAX_TYPES methylation types");
    meth.n_types = (uint32_t)methylation_types.size();
    for (size_t t = 0; t < methylation_types.size(); ++t) {
        MethylationCallingParameters mp;
        mp.methylation_type = methylation_types[t];
        meth.alphabets[t] = make_meth_params(mp, k, 0, 0);
    }
    for (const EventAlignedRead& r : alignments.records)
        for (const std::string& type : methylation_types) {
            const PoreModel* m = r.read->get_model(0, type);
            if (!m) throw Error(NPH_ERR_INVALID, std::string(caller) + ": a read without a model of methylation type " + type);
            alt_models.push_back(engine.model_id(m));
        }
    alt_models.push_back(0);
}

} // namespace

Haplotype fix_homopolymers(const Haplotype& input, const HomopolymerRegion& region, int min_flanking_sequence, Engine& engine, double indel_bias,
                           nph_hp_counts* counts_out)
{
    const int region_end = region.region_start + (int)region.reference.size() - 1;
    std::vector<HomopolymerWindow> wins = homopolymer_windows(input, region.region_start, region_end, min_flanking_sequence);
    std::string seqs;
    std::vector<nph_hp_window> dev(wins.size());
    for (size_t i = 0; i < wins.size(); ++i) {
        wins[i].dev.seq_off = seqs.size();
        seqs += wins[i].calling;
        dev[i] = wins[i].dev;
    }
    const RegionLayout rl = region_layout(region, engine, "fix_homopolymers");
    const detail::FlatReads& fr = rl.fr;
    std::vector<float> duration(std::max<size_t>(fr.n_events, 1));
    for (size_t i = 0; i < rl.reads.size(); ++i) {
        const std::vector<SquiggleEvent>& ev = rl.reads.reads()[i].first->events[rl.reads.reads()[i].second];
        for (size_t e = 0; e < ev.size(); ++e) duration[fr.reads[i].event_off + e] = ev[e].duration;
    }
    nph_hp_params params;
    std::memset(&params, 0, sizeof(params));
    params.region_start = region.region_start;
    params.min_flanking_sequence = min_flanking_sequence;
    std::vector<nph_hp_likelihoods> lik(std::max<size_t>(wins.size(), 1));
    nph_hp_counts counts;
    engine.check(nph_homopolymer_likelihoods_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, rl.time.data(), duration.data(), fr.n_events,
                                                   region.reference.data(), region.reference.size(), rl.deltas.data(), rl.deltas.size(), rl.first.data(),
                                                   rl.recs.data(), rl.recs.size(), &params, seqs.data(), seqs.size(), dev.data(), dev.size(), indel_bias,
                                                   lik.data(), &counts),
                 "nph_homopolymer_likelihoods_batch");
    if (counts_out) *counts_out = counts;

    Haplotype fixed = input;
    for (size_t wi = 0; wi < wins.size(); ++wi) {
        const HomopolymerWindow& w = wins[wi];
        const nph_hp_likelihoods& L = lik[wi];
        const char hp_base = w.dev.hp_base;
        const HomopolymerCall hc = homopolymer_call(L, w.dev.hp_length);
        if (!hc.kept) continue;
        const int size_diff = hc.size_diff;
        const double score = hc.quality;
        Variant v;
        v.ref_name = fixed.get_reference_name();
        v.add_info("TotalReads", (size_t)L.total_reads);
        v.add_info("AlleleCount", 1);
        for (size_t k = w.hp_start; k <= w.hp_end && size_diff != 0; ++k) {
            v.ref_position = input.get_reference_position_for_haplotype_base(k);
            if (v.ref_position == std::string::npos) continue;
            if (size_diff > 0) {
                v.ref_seq = fixed.substr_by_reference(v.ref_position, v.ref_position).get_sequence();
                if (v.ref_seq.size() != 1 || v.ref_seq[0] != hp_base) continue;
                v.alt_seq = v.ref_seq + hp_base;
            } else {
                v.ref_seq = fixed.substr_by_reference(v.ref_position, v.ref_position + 1).get_sequence();
                if (v.ref_seq.size() != 2 || v.ref_seq[0] != hp_base || v.ref_seq[1] != hp_base) continue;
                v.alt_seq = v.ref_seq.substr(0, 1);
            }
            v.quality = score;
            if (fixed.apply_variant(v)) break;
        }
    }
    return fixed;
}

void annotate_variants_with_all_support(std::vector<Variant>& input, const RegionAlignments& alignments, int min_flanking_sequence,
                                        uint32_t alignment_flags, Engine& engine, double indel_bias, nph_support_counts* counts_out)
{
    std::string ref_seqs;
    std::vector<nph_support_variant> dev(std::max<size_t>(input.size(), 1));
    for (size_t i = 0; i < input.size(); ++i) {
        const Variant& v = input[i];
        if (v.ref_name != alignments.contig)
            throw Error(NPH_ERR_INVALID, "annotate_variants_with_all_support: variant " + std::to_string(i) + " is on another contig than the region");
        if (v.ref_position > (size_t)INT32_MAX)
            throw Error(NPH_ERR_INVALID, "annotate_variants_with_all_support: variant " + std::to_string(i) + " lies beyond int32");
        std::memset(&dev[i], 0, sizeof(dev[i]));
        dev[i].ref_position = (int32_t)v.ref_position;
        dev[i].ref_seq_len = (uint32_t)v.ref_seq.size();
        dev[i].ref_seq_off = ref_seqs.size();
        ref_seqs += v.ref_seq;
    }
    const RegionLayout rl = region_layout(alignments, engine, "annotate_variants_with_all_support");
    const detail::FlatReads& fr = rl.fr;
    nph_support_params params;
    std::memset(&params, 0, sizeof(params));
    params.region_start = alignments.region_start;
    params.flank = min_flanking_sequence;
    params.alignment_flags = alignment_flags;
    // every record's base model has this k (the device call checks); the DNA models of the reads are 6-mers
    params.k = alignments.records.empty() ? 6 : alignments.records[0].read->get_base_model(0)->k;
    std::vector<nph_support_result> out(std::max<size_t>(input.size(), 1));
    nph_support_counts counts;
    engine.check(nph_all_support_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, rl.time.data(), fr.n_events,
                                       alignments.reference.data(), alignments.reference.size(), rl.deltas.data(), rl.deltas.size(), rl.first.data(),
                                       rl.recs.data(), rl.recs.size(), &params, ref_seqs.data(), ref_seqs.size(), dev.data(), input.size(), indel_bias,
                                       out.data(), &counts),
                 "nph_all_support_batch");
    if (counts_out) *counts_out = counts;
    for (size_t i = 0; i < input.size(); ++i) {
        std::stringstream ss;
        ss << std::fixed << std::setprecision(3);
        for (int hi = 0; hi < 4; ++hi) {
            ss << out[i].support[hi];
            if (hi != 3) ss << ",";
        }
        input[i].add_info("SupportFractionByBase", ss.str());
    }
}

std::vector<Variant> screen_variants_by_score(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants,
                                              uint32_t alignment_flags, int flank, uint32_t score_threshold,
                                              const std::vector<std::string>& methylation_types, Engine& engine, double indel_bias,
                                              nph_screen_list_counts* counts_out)
{
    std::string alleles;
    std::vector<nph_screen_candidate> dev(std::max<size_t>(candidate_variants.size(), 1));
    for (size_t i = 0; i < candidate_variants.size(); ++i) {
        const Variant& v = candidate_variants[i];
        if (v.ref_position > (size_t)INT32_MAX)
            throw Error(NPH_ERR_INVALID, "screen_variants_by_score: candidate " + std::to_string(i) + " lies beyond int32");
        std::memset(&dev[i], 0, sizeof(dev[i]));
        dev[i].ref_position = (int64_t)v.ref_position;
        dev[i].ref_seq_len = (uint32_t)v.ref_seq.size();
        dev[i].alt_seq_len = (uint32_t)v.alt_seq.size();
        dev[i].ref_seq_off = alleles.size();
        alleles += v.ref_seq;
        dev[i].alt_seq_off = alleles.size();
        alleles += v.alt_seq;
    }
    const RegionLayout rl = region_layout(alignments, engine, "screen_variants_by_score");
    const detail::FlatReads& fr = rl.fr;
    nph_screen_list_params params;
    std::memset(&params, 0, sizeof(params));
    params.region_start = alignments.region_start;
    params.flank = flank;
    params.score_threshold = score_threshold;
    params.alignment_flags = alignment_flags;
    // every record's base model has this k (the device call checks); the DNA models of the reads are 6-mers
    params.k = alignments.records.empty() ? 6 : alignments.records[0].read->get_base_model(0)->k;
    params.reads_per_round = 8;
    nph_screen_methylation meth;
    std::vector<uint32_t> alt_models;
    methylation_args(alignments, methylation_types, params.k, engine, "screen_variants_by_score", meth, alt_models);
    std::vector<nph_screen_result> out(std::max<size_t>(candidate_variants.size(), 1));
    nph_screen_list_counts counts;
    engine.check(nph_screen_variants_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, rl.time.data(), fr.n_events,
                                           alignments.reference.data(), alignments.reference.size(), rl.deltas.data(), rl.deltas.size(),
                                           rl.first.data(), rl.recs.data(), rl.recs.size(), &params, alleles.data(), alleles.size(), dev.data(),
                                           candidate_variants.size(), indel_bias, methylation_types.empty() ? nullptr : &meth, alt_models.data(),
                                           out.data(), &counts),
                 "nph_screen_variants_batch");
    if (counts_out) *counts_out = counts;
    std::vector<Variant> kept;
    for (size_t i = 0; i < candidate_variants.size(); ++i) {
        if (out[i].status == NPH_SCREEN_OUTSIDE || !(out[i].quality > 0)) continue;
        Variant v = candidate_variants[i];
        v.quality = out[i].quality;
        v.info = "";
        kept.push_back(v);
    }
    return kept;
}

std::vector<Variant> expand_variants(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants, int min_flanking_sequence)
{
    const int region_start = alignments.region_start;
    const int region_end = alignments.region_start + (int)alignments.reference.size() - 1;
    std::vector<Variant> out;
    for (size_t vi = 0; vi < candidate_variants.size(); ++vi) {
        const Variant& in = candidate_variants[vi];
        out.push_back(in);
        if (in.ref_seq.size() == 1 && in.alt_seq.size() == 1) continue;
        // the deletion extended by one base, where it stays in the region and more than min_flanking_sequence bases from its end
        const int start = (int)in.ref_position;
        const int deletion_end = (int)(in.ref_position + in.ref_seq.size());
        if (in.ref_name == alignments.contig && start >= region_start && deletion_end <= region_end &&
            region_end - deletion_end > min_flanking_sequence) {
            Variant v = in;
            v.ref_seq = alignments.reference.substr((size_t)(start - region_start), (size_t)(deletion_end - start + 1));
            if (v.ref_seq.compare(0, in.ref_seq.size(), in.ref_seq) != 0)
                throw Error(NPH_ERR_INVALID, "expand_variants: candidate " + std::to_string(vi) + "'s ref_seq is not the region's (the reference asserts)");
            out.push_back(v);
        }
        for (int j = 0; j < 4; ++j) {
            Variant v = in;
            v.alt_seq.append(1, "ACGT"[j]);
            out.push_back(v);
        }
    }
    return out;
}

namespace {

// The probability of the 2x2 table whose first cell is x, its margins fixed: exp of log-binomials, or, when x is next to the
// previous x and neither a multiple of 11 nor a table with an empty fourth cell, the previous probability times the ratio of the
// two tables' probabilities, in kt_fisher_exact's operation order
struct TableProbability {
    int row1, col1, n, x;
    double p;
    static double log_choose(int a, int b) { return (b == 0 || a == b) ? 0 : std::lgamma(a + 1) - std::lgamma(b + 1) - std::lgamma(a - b + 1); }
    double direct(int v) const { return std::exp(log_choose(row1, v) + log_choose(n - row1, col1 - v) - log_choose(n, col1)); }
    double at(int v)
    {
        const int n22 = v + n - row1 - col1;
        if (v % 11 && n22) {
            if (v == x + 1) { p *= (double)(row1 - x) / v * (col1 - x) / n22; x = v; return p; }
            if (v == x - 1) { p *= (double)x / (row1 - v) * (x + n - row1 - col1) / (col1 - v); x = v; return p; }
        }
        x = v;
        p = direct(v);
        return p;
    }
};

std::string format_double(double v)
{
    std::stringstream ss;
    ss << v;
    return ss.str();
}

} // namespace

double fisher_exact_two_sided(int n11, int n12, int n21, int n22)
{
    const int row1 = n11 + n12, col1 = n11 + n21, n = n11 + n12 + n21 + n22;
    const int hi = col1 < row1 ? col1 : row1;
    const int lo = std::max(0, row1 + col1 - n);
    if (lo == hi) return 1.0;
    TableProbability t{row1, col1, n, n11, 0.0};
    t.p = t.direct(n11);
    const double q = t.p;
    double left = 0.0, right = 0.0;
    double p = t.at(lo);
    for (int i = lo + 1; p < 0.99999999 * q; ++i) { left += p; p = t.at(i); }
    if (p < 1.00000001 * q) left += p;
    p = t.at(hi);
    for (int j = hi - 1; p < 0.99999999 * q; --j) { right += p; p = t.at(j); }
    if (p < 1.00000001 * q) right += p;
    const double two = left + right;
    return two > 1.0 ? 1.0 : two;
}

double calculate_sor(double ref_fwd, double ref_rev, double alt_fwd, double alt_rev)
{
    ref_fwd += 1; ref_rev += 1; alt_fwd += 1; alt_rev += 1;                    // no zeros
    const double r = (ref_fwd * alt_rev) / (alt_fwd * ref_rev);
    const double sym_ratio = r + (1.0 / r);
    const double ref_ratio = std::min(ref_fwd, ref_rev) / std::max(ref_fwd, ref_rev);
    const double alt_ratio = std::min(alt_fwd, alt_rev) / std::max(alt_fwd, alt_rev);
    return std::log(sym_ratio) + std::log(ref_ratio) - std::log(alt_ratio);
}

std::string make_genotype(size_t alt_alleles, size_t ploidy)
{
    if (alt_alleles > ploidy) throw Error(NPH_ERR_INVALID, "make_genotype: more alternative alleles than the ploidy");
    std::string out(2 * ploidy - 1, '/');
    for (size_t a = 0; a < ploidy; ++a) out[2 * a] = a < ploidy - alt_alleles ? '0' : '1';
    return out;
}

Haplotype call_haplotype_from_candidates(const RegionAlignments& alignments, const std::vector<Variant>& candidate_variants,
                                         uint32_t alignment_flags, int flank, int min_distance, int max_haplotypes, int ploidy,
                                         bool genotype_only, const std::vector<std::string>& methylation_types, bool calculate_all_support,
                                         Engine& engine, double indel_bias, nph_call_counts* counts_out)
{
    const Haplotype region_haplotype(alignments.contig, (size_t)alignments.region_start, alignments.reference);
    for (size_t i = 0; i < candidate_variants.size(); ++i)
        if (candidate_variants[i].ref_position > (size_t)INT32_MAX)
            throw Error(NPH_ERR_INVALID, "call_haplotype_from_candidates: candidate " + std::to_string(i) + " lies beyond int32");
    // the groups of :790-854 that get called, with their combinations
    struct Group { size_t first, n; VariantCombinations vc; };
    std::vector<Group> called;
    std::vector<nph_call_group> dev_groups;
    std::vector<nph_call_haplotype> dev_haps;
    std::string bases;
    std::vector<uint32_t> cvars;
    size_t n_var_results = 0;
    for (size_t cur = 0; cur < candidate_variants.size();) {
        size_t end = cur + 1;
        while (end < candidate_variants.size()) {
            const int distance = (int)candidate_variants[end].ref_position - (int)candidate_variants[end - 1].ref_position;
            if (distance > min_distance) break;
            end++;
        }
        const int calling_start = (int)candidate_variants[cur].ref_position - flank;
        const int calling_end = (int)(candidate_variants[end - 1].ref_position + candidate_variants[end - 1].ref_seq.length()) + flank;
        if (calling_end - calling_start <= 200) {
            if (calling_start < 0) throw Error(NPH_ERR_INVALID, "call_haplotype_from_candidates: a window before the contig's start");
            const Haplotype calling = region_haplotype.substr_by_reference((size_t)calling_start, (size_t)calling_end);
            const std::vector<Variant> vs(candidate_variants.begin() + cur, candidate_variants.begin() + end);
            Group g{cur, end - cur, variant_combinations(vs, calling, max_haplotypes)};
            if (g.vc.combinations.size() > 1) {                                   // simple_call skips a group with one combination
                nph_call_group d;
                std::memset(&d, 0, sizeof(d));
                d.calling_start = calling_start; d.calling_end = calling_end;
                d.hap_first = (uint32_t)dev_haps.size(); d.n_haplotypes = (uint32_t)g.vc.combinations.size();
                d.var_first = (uint32_t)n_var_results; d.n_variants = (uint32_t)g.n;
                n_var_results += g.n;
                for (size_t c = 0; c < g.vc.combinations.size(); ++c) {
                    nph_call_haplotype h;
                    std::memset(&h, 0, sizeof(h));
                    const std::string& seq = g.vc.haplotypes[c].get_sequence();
                    h.seq_off = bases.size(); h.seq_len = (uint32_t)seq.size();
                    h.var_off = cvars.size(); h.n_var = (uint32_t)g.vc.combinations[c].size();
                    bases += seq;
                    for (size_t id : g.vc.combinations[c]) cvars.push_back((uint32_t)id);
                    dev_haps.push_back(h);
                }
                dev_groups.push_back(d);
                called.push_back(std::move(g));
            }
        }
        cur = end;
    }
    const RegionLayout rl = region_layout(alignments, engine, "call_haplotype_from_candidates");
    const detail::FlatReads& fr = rl.fr;
    // VariantGroup's read keys "read_name:strand" (every record is strand 0 of its read), ranked as std::map orders them
    std::vector<std::string> keys(rl.reads.size());
    for (size_t i = 0; i < rl.reads.size(); ++i) keys[i] = rl.reads.reads()[i].first->read_name + ":" + std::to_string(rl.reads.reads()[i].second);
    std::vector<std::string> sorted = keys;
    std::sort(sorted.begin(), sorted.end());
    sorted.erase(std::unique(sorted.begin(), sorted.end()), sorted.end());
    std::vector<uint32_t> key_rank(std::max<size_t>(keys.size(), 1));
    for (size_t i = 0; i < keys.size(); ++i) key_rank[i] = (uint32_t)(std::lower_bound(sorted.begin(), sorted.end(), keys[i]) - sorted.begin());
    nph_call_params params;
    std::memset(&params, 0, sizeof(params));
    params.region_start = alignments.region_start;
    params.ploidy = (uint32_t)ploidy;
    params.genotype_all = genotype_only ? 1u : 0u;
    params.alignment_flags = alignment_flags;
    // every record's base model has this k (the device call checks); the DNA models of the reads are 6-mers
    params.k = alignments.records.empty() ? 6 : alignments.records[0].read->get_base_model(0)->k;
    nph_screen_methylation meth;
    std::vector<uint32_t> alt_models;
    methylation_args(alignments, methylation_types, params.k, engine, "call_haplotype_from_candidates", meth, alt_models);
    if (ploidy < 1) throw Error(NPH_ERR_INVALID, "call_haplotype_from_candidates: ploidy below 1");
    std::vector<nph_call_group_result> gres(std::max<size_t>(dev_groups.size(), 1));
    std::vector<nph_call_variant_result> vres(std::max<size_t>(n_var_results, 1));
    nph_call_counts counts;
    if (bases.empty()) bases.push_back('\0');
    if (cvars.empty()) cvars.push_back(0);
    if (dev_haps.empty()) dev_haps.emplace_back();
    engine.check(nph_call_variant_groups_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, rl.time.data(), fr.n_events,
                                               alignments.reference.data(), alignments.reference.size(), rl.deltas.data(), rl.deltas.size(),
                                               rl.first.data(), rl.recs.data(), rl.recs.size(), key_rank.data(), &params, dev_groups.data(),
                                               dev_groups.size(), dev_haps.data(), dev_haps.size(), bases.data(), bases.size(), cvars.data(),
                                               cvars.size(), n_var_results, indel_bias, methylation_types.empty() ? nullptr : &meth,
                                               alt_models.data(), gres.data(), vres.data(), &counts),
                 "nph_call_variant_groups_batch");
    if (counts_out) *counts_out = counts;
    // simple_call's output per group (ref: src/common/nanopolish_variant.cpp:416-488)
    std::vector<std::vector<Variant>> calls(called.size());
    std::vector<Variant> all_calls;
    for (size_t gi = 0; gi < called.size(); ++gi) {
        const nph_call_group_result& R = gres[gi];
        const nph_call_variant_result* V = vres.data() + dev_groups[gi].var_first;
        const size_t total_reads = R.n_keys;
        for (size_t vi = 0; vi < called[gi].n; ++vi) {
            if (!V[vi].emit) continue;
            Variant v = candidate_variants[called[gi].first + vi];
            const size_t var_count = V[vi].var_count;
            v.quality = var_count > 0 ? R.best_score - R.base_score : 0.0;
            v.add_info("TotalReads", total_reads);
            v.add_info("AlleleCount", var_count);
            v.add_info("SupportFraction", format_double(V[vi].support_sum / total_reads));
            const double ref_fwd = V[vi].strand[0], ref_rev = V[vi].strand[1], alt_fwd = V[vi].strand[2], alt_rev = V[vi].strand[3];
            v.add_info("SupportFractionByStrand", format_double(alt_fwd / (ref_fwd + alt_fwd)) + "," + format_double(alt_rev / (ref_rev + alt_rev)));
            v.add_info("StrandSupport", std::to_string((int)std::round(ref_fwd)) + "," + std::to_string((int)std::round(ref_rev)) + "," +
                                        std::to_string((int)std::round(alt_fwd)) + "," + std::to_string((int)std::round(alt_rev)));
            // kt_fisher_exact takes int cells: the sums are truncated
            const double two = fisher_exact_two_sided((int)ref_fwd, (int)ref_rev, (int)alt_fwd, (int)alt_rev);
            int fisher_scaled = (int)(-4.343 * std::log(two) + .499);
            if (fisher_scaled < 0) fisher_scaled = 1000;                        // underflow
            v.add_info("StrandFisherTest", fisher_scaled);
            v.add_info("SOR", format_double(calculate_sor(ref_fwd, ref_rev, alt_fwd, alt_rev)));
            v.genotype = total_reads > 0 ? make_genotype(var_count, (size_t)ploidy) : ".";
            calls[gi].push_back(v);
        }
        all_calls.insert(all_calls.end(), calls[gi].begin(), calls[gi].end());
    }
    // per-variant results do not depend on the batch: one annotation of every called variant, split back into its groups
    if (calculate_all_support && !all_calls.empty()) {
        annotate_variants_with_all_support(all_calls, alignments, flank, alignment_flags, engine, indel_bias);
        size_t at = 0;
        for (std::vector<Variant>& c : calls)
            for (Variant& v : c) v = all_calls[at++];
    }
    Haplotype derived = region_haplotype;
    for (const std::vector<Variant>& c : calls)
        for (const Variant& v : c) derived.apply_variant(v);
    return derived;
}

} // namespace nph
