// nph_scorereads.cpp — see nph_scorereads.hpp.
#include "nph_scorereads.hpp"

#include <cstdio>
#include <cstdlib>

namespace nph {

void ScoreReads::clear()
{
    m_batch.clear(); m_segments.clear(); m_scores.clear(); m_strands.clear();
}

void TransitionTraining::add(const nph_transition_counts* counts)
{
    for (size_t g = 0; g < kStrands; ++g) {
        const uint64_t* in = reinterpret_cast<const uint64_t*>(&counts[g]);
        uint64_t* acc = reinterpret_cast<uint64_t*>(&m_counts[g]);
        for (size_t i = 0; i < sizeof(nph_transition_counts) / sizeof(uint64_t); ++i) acc[i] += in[i];
    }
}

TransitionTraining::Probs TransitionTraining::train(size_t strand, const Probs& prior) const
{
    const nph_transition_counts& c = m_counts[strand];
    const uint32_t pseudocount = 100;
    Probs p;
    for (size_t b = 0; b < NPH_TT_BINS; ++b) {
        double skip = prior[b] * pseudocount;
        // the reference's observations of a bin in any order: +1.0 per skip, +0.0 (no change) per other; total += 1 is exact
        for (uint64_t i = 0; i < c.skip_count[b]; ++i) skip += 1.0;
        const double total = (double)pseudocount + (double)c.skip_total[b];
        p[b] = skip / total;
    }
    return p;
}

std::string TransitionTraining::report() const
{
    std::string out;
    char line[96];
    for (size_t strand = 0; strand < kStrands; ++strand) {
        std::snprintf(line, sizeof(line), "Transition parameters for %zu\n", strand);
        out += line;
        const Probs p = train(strand);
        for (size_t b = 0; b < NPH_TT_BINS; ++b) {
            std::snprintf(line, sizeof(line), "skip_probabilities[%zu] = %.3lf;\n", b, p[b]);
            out += line;
        }
    }
    return out;
}

size_t ScoreReads::add_read(SquiggleRead& sr, size_t strand_idx, const std::vector<EventAlignment>& alignment_output,
                            const std::string& ref_seq, int ref_offset)
{
    const size_t read_idx = m_scores.size();
    m_scores.emplace_back();
    const PoreModel* pore_model = sr.get_model((uint32_t)strand_idx, "nucleotide");
    if (!pore_model) throw Error(NPH_ERR_INVALID, "read has no nucleotide model");
    const Alphabet* alphabet = pore_model->pmalphabet;
    const int eps = (int)m_events_per_segment;
    for (int align_start_idx = eps; align_start_idx < (int)alignment_output.size() - eps; align_start_idx += eps) {
        const EventAlignment& align_start = alignment_output[align_start_idx];
        const EventAlignment& align_end = alignment_output[align_start_idx + eps];
        HMMInputData data;
        data.read = &sr;
        data.pore_model = pore_model;
        data.strand = (uint8_t)strand_idx;
        data.rc = alignment_output.front().rc;
        data.event_start_idx = (uint32_t)align_start.event_idx;
        data.event_stop_idx = (uint32_t)align_end.event_idx;
        data.event_stride = data.event_start_idx <= data.event_stop_idx ? 1 : -1;
        const int ref_start_pos = align_start.ref_position, ref_end_pos = align_end.ref_position;
        if (ref_end_pos < ref_start_pos) throw Error(NPH_ERR_INVALID, "event alignment runs backwards on the reference");   // the reference asserts
        // get_reference_region_ts(fai, contig, start, end): end inclusive, clipped to what the index holds
        const long long first = (long long)ref_start_pos - ref_offset;
        if (first < 0 || first > (long long)ref_seq.size()) throw Error(NPH_ERR_INVALID, "segment outside the fetched reference");
        std::string seg = ref_seq.substr((size_t)first, (size_t)(ref_end_pos - ref_start_pos + 1));
        if ((int)seg.size() <= (int)sr.get_model_k((uint32_t)strand_idx)) continue;
        seg = alphabet->disambiguate(seg);
        HMMInputSequence sequence(seg, alphabet->reverse_complement(seg), alphabet);
        const int events_in_segment = std::abs((int)data.event_start_idx - (int)data.event_stop_idx) + 1;
        m_segments.push_back(Segment{read_idx, m_batch.add(sequence, data, 0), events_in_segment});
        m_strands.push_back((uint8_t)strand_idx);
    }
    return read_idx;
}

void ScoreReads::run(Engine& engine, double indel_bias)
{
    std::vector<float> s;
    if (m_train) {
        nph_tt_params params{(uint32_t)TransitionTraining::kStrands, 5, m_max_chunk_jobs, 0, 0.f, 0.f};   // ignore_edge_length = 5
        nph_transition_counts counts[TransitionTraining::kStrands];
        s = m_batch.run_training(engine, m_strands, params, counts, indel_bias);
        m_training.add(counts);
    } else {
        s = m_batch.run(engine, indel_bias);
    }
    std::vector<double> sum(m_scores.size(), 0.0);
    for (const Segment& g : m_segments) {
        sum[g.read] += s[g.job];                    // double accumulation of the float segment scores, in segment order
        m_scores[g.read].n_events += (size_t)g.events;
        m_scores[g.read].n_segments += 1;
    }
    for (size_t i = 0; i < m_scores.size(); ++i)
        m_scores[i].score = m_scores[i].n_events == 0 ? 1.0 : sum[i] / (double)m_scores[i].n_events;
    m_segments.clear();
    m_strands.clear();
    m_batch.clear();
}

} // namespace nph
