// nph_scorereads.hpp — the caller of profile_hmm_score in `nanopolish scorereads` (BASELINE configs[1]):
//
//   model_score                         ref: src/nanopolish_scorereads.cpp:116-203
//
// The reference walks a read's event alignment (the output of align_read_to_ref) in steps of events_per_segment
// entries, scores the reference stretch between the two boundary entries against the events between them with one
// profile_hmm_score call per segment, and returns sum(segment scores) / sum(events).  Here add_read() only enumerates the
// segments into one HmmBatch for a whole batch of reads; run() launches once and folds the per-read ratios.  The
// per-segment recalibration the reference prints on its SEGMENT lines does not feed the score and is not reproduced.
// With train_transitions (scorereads --train-transitions), run() also trains on profile_hmm_align's path of every segment
// (nph_train_transitions_batch, grouped by strand) and accumulates the counts into training().
#pragma once
#include "nph_eventalign.hpp"

#include <array>

namespace nph {

struct ReadScore {
    double score = 1.0;          // curr_score / nevents, or +1 when no segment was scored (the reference's convention)
    size_t n_events = 0;
    size_t n_segments = 0;
};

// The training half of TransitionParameters (ref: src/hmm/nanopolish_transition_parameters.cpp:294-448), one per strand as
// scorereads keeps them, over the counts the device accumulates.
class TransitionTraining {
public:
    static const size_t kStrands = 2;                   // NUM_STRANDS
    typedef std::array<double, NPH_TT_BINS> Probs;
    // adds kStrands records (what nph_train_transitions_batch writes with n_groups = kStrands)
    void add(const nph_transition_counts* counts);
    const nph_transition_counts& counts(size_t strand) const { return m_counts[strand]; }
    // TransitionParameters::train() from the skip probabilities `prior` (scorereads never initialize()s its tables: all zeros).
    // Per bin: skip = prior * 100 and total = 100, then +1.0 per skip observation and +1 per observation, one at a time as the
    // reference adds them, then skip / total.
    Probs train(size_t strand, const Probs& prior = Probs()) const;
    // scorereads' stderr after --train-transitions: per strand "Transition parameters for %zu" and print() of train(strand)
    std::string report() const;
    void clear() { m_counts[0] = m_counts[1] = nph_transition_counts{}; }

private:
    nph_transition_counts m_counts[kStrands] = {};
};

class ScoreReads {
public:
    explicit ScoreReads(size_t events_per_segment = 500, bool train_transitions = false)
        : m_events_per_segment(events_per_segment), m_train(train_transitions) {}
    // alignment_output: the read's EventAlignments (EventAligner::alignment(i)); ref_seq: the reference over
    // [ref_offset, ...] as the record's faidx fetch returns it (any case, IUPAC codes allowed).  Returns the read's index.
    size_t add_read(SquiggleRead& sr, size_t strand_idx, const std::vector<EventAlignment>& alignment_output,
                    const std::string& ref_seq, int ref_offset);
    void run(Engine& engine, double indel_bias = hmm_indel_bias_factor);
    const ReadScore& score(size_t read_idx) const { return m_scores[read_idx]; }
    size_t num_reads() const { return m_scores.size(); }
    const HmmBatch& batch() const { return m_batch; }
    // the counts of every run() so far (train_transitions only); clear() keeps them
    TransitionTraining& training() { return m_training; }
    // jobs per chunk of Viterbi states of the training call (0: as many as fit its budget)
    void set_max_chunk_jobs(uint32_t n) { m_max_chunk_jobs = n; }
    void clear();

private:
    struct Segment { size_t read; size_t job; int events; };
    size_t m_events_per_segment;
    bool m_train;
    uint32_t m_max_chunk_jobs = 0;
    TransitionTraining m_training;
    std::vector<uint8_t> m_strands;     // per job: the segment's strand (its training group)
    HmmBatch m_batch;
    std::vector<Segment> m_segments;
    std::vector<ReadScore> m_scores;
};

} // namespace nph
