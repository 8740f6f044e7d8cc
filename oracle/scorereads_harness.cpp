// scorereads_harness.cpp — TEST INFRASTRUCTURE ONLY.  Runs the reference's own model_score (src/nanopolish_scorereads.cpp:116-203,
// compiled here in place through the #include below) unmodified, with transition training, then TransitionParameters::train() and
// print() (src/hmm/nanopolish_transition_parameters.cpp:370-448), and returns what they computed.
//
// What model_score reaches outside its computation:
//   the faidx handle     the in-memory contig of ref_harness.cpp's faidx_fetch_seq test double (an NprefContig)
//   the SquiggleRead     a handle of ref_harness.cpp (npref_read_create, found by npref_read_of), strand 0
//   stdout               its SEGMENT lines, written to a memory stream and dropped
//   stderr               print()'s lines, written to a memory stream and returned
// Nothing of the reference is copied.
#include "nanopolish_scorereads.cpp"
#include "ref_harness.h"

#include <cstdio>

extern "C" {

// model_score(sr, 0, fai, alignment, eps, &tp) on read handle read_h (a built-in model, which model_score looks up by name), the
// alignment being n_align EventAlignments {ref_name = contig, ref_position = ref_pos[i], event_idx = event_idx[i], rc, strand 0}
// over the contig `contig_seq`; tp default-constructed (scorereads' prior, all zeros) or, with r9_prior, initialize()d with an R9
// template metadata.  Then tp.train() and tp.print().
//   score_out      model_score's return value
//   counts_out     81 words in the layout of nph_transition_counts: state_transitions (3 x 6), n_matches, n_merges, n_skips, and
//                  per bin of get_skip_bin's expression over training_data.kmer_transitions the observations and the skips
//   probs_out      the 30 skip probabilities after train()
//   text_out       print()'s bytes
// Returns the length of the text, -1 when cap is too small.
long long npref_model_score_train(int read_h, const char* contig, const char* contig_seq, int n_align, const int32_t* ref_pos,
                                  const int32_t* event_idx, int rc, int eps, int r9_prior, double* score_out, uint64_t* counts_out,
                                  double* probs_out, char* text_out, size_t cap)
{
    SquiggleRead* sr = npref_read_of(read_h);
    NprefContig fai{contig, contig_seq};
    std::vector<EventAlignment> ao(n_align);
    for (int i = 0; i < n_align; ++i) {
        ao[i].ref_name = contig; ao[i].ref_position = ref_pos[i]; ao[i].read_idx = 0; ao[i].strand_idx = 0;
        ao[i].event_idx = event_idx[i]; ao[i].rc = rc != 0; ao[i].hmm_state = 'M';
    }
    TransitionParameters tp;
    if (r9_prior) {
        ModelMetadata md;
        md.strand_idx = T_IDX; md.model_idx = 0; md.kit = KV_R9_4_450BPS;
        tp.initialize(md);
    }
    char* seg_text = nullptr; size_t seg_len = 0;
    FILE* saved_out = stdout;
    stdout = open_memstream(&seg_text, &seg_len);
    *score_out = model_score(*sr, 0, reinterpret_cast<const faidx_t*>(&fai), ao, (size_t)eps, &tp);
    fclose(stdout);
    stdout = saved_out;
    free(seg_text);

    const TransitionTrainingData& td = tp.training_data;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 6; ++c) counts_out[r * 6 + c] = get(td.state_transitions, r, c);
    counts_out[18] = td.n_matches; counts_out[19] = td.n_merges; counts_out[20] = td.n_skips;
    for (int b = 0; b < 60; ++b) counts_out[21 + b] = 0;
    for (const KmerTransitionObservation& to : td.kmer_transitions) {
        // get_skip_bin (nanopolish_transition_parameters.h:101-111)
        double d = fabs(to.level_1 - to.level_2);
        size_t bin = d / tp.skip_bin_width;
        bin = bin >= tp.skip_probabilities.size() ? tp.skip_probabilities.size() - 1 : bin;
        counts_out[21 + bin] += 1;
        counts_out[51 + bin] += to.state == 'K';
    }
    tp.train();
    for (int b = 0; b < 30; ++b) probs_out[b] = tp.skip_probabilities[b];
    char* text = nullptr; size_t len = 0;
    FILE* saved_err = stderr;
    stderr = open_memstream(&text, &len);
    tp.print();
    fclose(stderr);
    stderr = saved_err;
    std::string s(text, len);
    free(text);
    if (s.size() >= cap) return -1;
    std::memcpy(text_out, s.c_str(), s.size() + 1);
    return (long long)s.size();
}

// the 30 skip probabilities TransitionParameters::initialize gives an R9 template model (initialize_sqkmap007_template)
void npref_transition_prior_r9(double* out)
{
    TransitionParameters tp;
    ModelMetadata md;
    md.strand_idx = T_IDX; md.model_idx = 0; md.kit = KV_R9_4_450BPS;
    tp.initialize(md);
    for (int b = 0; b < 30; ++b) out[b] = tp.skip_probabilities[b];
}

} // extern "C"
