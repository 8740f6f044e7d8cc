// nph_eventalign.cpp — see nph_eventalign.hpp (SURVEY.md section 8f, row N1).
#include "nph_eventalign.hpp"
#include "../csrc/tsv_format.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace nph {

// ---------------------------------------------------------------------------------------------
// AlignBatch / profile_hmm_align
// ---------------------------------------------------------------------------------------------
size_t AlignBatch::add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags)
{
    nph_hmm_job j = detail::make_hmm_job(sequence, data, flags, m_reads);
    j.rank_off = m_ranks.size();
    sequence.append_kmer_ranks(data.pore_model->k, data.rc != 0, m_ranks);
    m_jobs.push_back(j);
    m_job_models.push_back(data.pore_model);
    return m_jobs.size() - 1;
}

void AlignBatch::clear_jobs()
{
    m_job_models.clear(); m_jobs.clear(); m_ranks.clear();
}

void AlignBatch::clear()
{
    clear_jobs();
    m_reads.clear(); m_reads_uploaded = 0;
}

std::vector<std::vector<HMMAlignmentState>> AlignBatch::run(Engine& engine, double indel_bias, bool reads_resident)
{
    std::vector<std::vector<HMMAlignmentState>> out(m_jobs.size());
    if (m_jobs.empty()) return out;
    detail::resolve_model_ids(engine, m_job_models, m_jobs);
    if (!reads_resident || m_reads_uploaded != m_reads.size()) {
        const detail::FlatReads fr = detail::flatten_reads(engine, m_reads);
        engine.check(nph_reads_load(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events), "nph_reads_load");
        m_reads_uploaded = m_reads.size();
    }
    std::vector<uint64_t> off(m_jobs.size() + 1, 0);
    for (size_t j = 0; j < m_jobs.size(); ++j) {
        const nph_hmm_job& jb = m_jobs[j];
        const uint64_t E = (jb.event_stop > jb.event_start ? jb.event_stop - jb.event_start : jb.event_start - jb.event_stop) + 1;
        off[j + 1] = off[j] + E + jb.n_kmers + 2;
    }
    std::vector<nph_align_state> states(off.back());
    std::vector<uint32_t> counts(m_jobs.size());
    engine.check(nph_hmm_align(engine.ctx(), m_ranks.data(), m_ranks.size(), m_jobs.data(), m_jobs.size(), indel_bias,
                               states.data(), off.data(), counts.data(), nullptr), "nph_hmm_align");
    for (size_t j = 0; j < m_jobs.size(); ++j) {
        out[j].resize(counts[j]);
        for (uint32_t i = 0; i < counts[j]; ++i) {
            const nph_align_state& s = states[off[j] + i];
            HMMAlignmentState& as = out[j][i];
            as.event_idx = s.event_idx;
            as.kmer_idx = s.kmer_idx;
            as.l_posterior = -INFINITY;
            as.l_fm = s.l_fm;
            as.log_transition_probability = -INFINITY;
            as.state = s.state;
        }
    }
    return out;
}

std::vector<HMMAlignmentState> profile_hmm_align(const HMMInputSequence& sequence, const HMMInputData& data, const uint32_t flags)
{
    AlignBatch b;
    b.add(sequence, data, flags);
    return b.run(Engine::thread_default())[0];
}

// ---------------------------------------------------------------------------------------------
// aligned pairs from the CIGAR
// ---------------------------------------------------------------------------------------------
std::vector<AlignedSegment> get_aligned_segments(int ref_pos, const std::vector<uint32_t>& cigar, int read_stride)
{
    std::vector<AlignedSegment> out(1);
    int read_pos = 0;
    for (uint32_t c : cigar) {
        const int len = (int)(c >> 4), op = (int)(c & 0xf);
        int read_inc = 0, ref_inc = 0;
        bool is_aligned = false;
        switch (op) {
            case NPH_CIGAR_M: case NPH_CIGAR_EQ: case NPH_CIGAR_X: is_aligned = true; read_inc = read_stride; ref_inc = 1; break;
            case NPH_CIGAR_D: ref_inc = 1; break;
            case NPH_CIGAR_N: out.push_back(AlignedSegment()); ref_inc = 1; break;     // a reference skip starts a new segment
            case NPH_CIGAR_I: read_inc = read_stride; break;
            case NPH_CIGAR_S: read_inc = 1; break;                                     // soft clips ignore read_stride
            case NPH_CIGAR_H: break;
            default: throw Error(NPH_ERR_INVALID, "unhandled CIGAR operation");        // the reference asserts
        }
        for (int j = 0; j < len; ++j) {
            if (is_aligned) out.back().push_back({ref_pos, read_pos});
            read_pos += read_inc;
            ref_pos += ref_inc;
        }
    }
    return out;
}

void trim_aligned_pairs_to_kmer(std::vector<AlignedPair>& aligned_pairs, int max_kmer_idx)
{
    int idx = (int)aligned_pairs.size() - 1;
    while (idx >= 0 && aligned_pairs[idx].read_pos > max_kmer_idx) idx -= 1;
    if (idx < 0) aligned_pairs.clear();
    else aligned_pairs.resize(idx + 1);
}

void trim_aligned_pairs_to_ref_region(std::vector<AlignedPair>& aligned_pairs, int ref_start, int ref_end)
{
    std::vector<AlignedPair> trimmed;
    for (const AlignedPair& p : aligned_pairs)
        if (p.ref_pos >= ref_start && p.ref_pos <= ref_end) trimmed.push_back(p);
    aligned_pairs.swap(trimmed);
}

// index of the pair with the highest ref_pos not above ref_pos_max, searching from pair_idx
int get_end_pair(const std::vector<AlignedPair>& aligned_pairs, int ref_pos_max, int pair_idx)
{
    while (pair_idx < (int)aligned_pairs.size()) {
        if (aligned_pairs[pair_idx].ref_pos > ref_pos_max) return pair_idx - 1;
        pair_idx += 1;
    }
    return (int)aligned_pairs.size() - 1;
}

// ---------------------------------------------------------------------------------------------
// EventAligner
// ---------------------------------------------------------------------------------------------
static const int ALIGN_STRIDE = 100;     // approximately how many reference bases to align to at once (eventalign.cpp:666)
static const int OUTPUT_STRIDE = 50;     // approximately how many event alignments to output at once (:667)

void EventAligner::clear()
{
    m_reads.clear(); m_round.clear(); m_batch.clear();
    m_lazy = Lazy();
}

size_t EventAligner::add_read(const EventAlignmentParameters& params)
{
    if (!params.sr) throw Error(NPH_ERR_INVALID, "EventAlignmentParameters without a read");
    if (params.strand_idx >= 2) throw Error(NPH_ERR_INVALID, "strand_idx out of range");
    if (!((params.region_start == -1 && params.region_end == -1) || params.region_start <= params.region_end))
        throw Error(NPH_ERR_INVALID, "region_start > region_end");
    m_reads.emplace_back();
    ReadState& rs = m_reads.back();
    rs.params = params;
    rs.pore_model = params.get_model();
    if (!rs.pore_model) throw Error(NPH_ERR_INVALID, "the read has no model for this strand / alphabet");
    rs.k = rs.pore_model->k;
    // upper case, ambiguity codes to their lexicographically lowest base (Alphabet::disambiguate upper-cases)
    rs.ref_seq = rs.pore_model->pmalphabet->disambiguate(params.ref_seq);
    rs.rc_ref_seq = rs.pore_model->pmalphabet->reverse_complement(rs.ref_seq);
    if ((params.flag & NPH_BAM_FUNMAP) != 0) { rs.done = true; return m_reads.size() - 1; }
    rs.segments = get_aligned_segments(params.ref_pos, params.cigar);
    rs.do_base_rc = (params.flag & NPH_BAM_FREVERSE) != 0;
    return m_reads.size() - 1;
}

// The head of the reference's per-segment loop body (eventalign.cpp:654-689): trims, then the events nearest to the
// segment's first and last aligned k-mer.  Depends only on the record, never on earlier paths.
bool EventAligner::setup_segment(ReadState& rs, size_t segment_idx, SegmentStart& out)
{
    AlignedSegment& aligned_pairs = rs.segments[segment_idx];
    const EventAlignmentParameters& p = rs.params;
    if (p.region_start != -1 && p.region_end != -1) trim_aligned_pairs_to_ref_region(aligned_pairs, p.region_start, p.region_end);
    const int max_kmer_idx = (int)p.sr->read_sequence.size() - (int)rs.k;
    trim_aligned_pairs_to_kmer(aligned_pairs, max_kmer_idx);
    if (aligned_pairs.empty()) return false;                 // the reference returns from the whole function here
    int read_kidx_start = aligned_pairs.front().read_pos;
    int read_kidx_end = aligned_pairs.back().read_pos;
    if (rs.do_base_rc) {
        read_kidx_start = p.sr->flip_k_strand(read_kidx_start, rs.k);
        read_kidx_end = p.sr->flip_k_strand(read_kidx_end, rs.k);
    }
    const int n_map = (int)p.sr->base_to_event_map.size();
    if (read_kidx_start < 0 || read_kidx_end < 0 || read_kidx_start >= n_map || read_kidx_end >= n_map)
        throw Error(NPH_ERR_INVALID, "aligned read position outside the base-to-event map");      // the reference asserts / reads out of bounds
    out.first_event = p.sr->get_closest_event_to(read_kidx_start, (uint32_t)p.strand_idx);
    out.last_event = p.sr->get_closest_event_to(read_kidx_end, (uint32_t)p.strand_idx);
    out.start_ref = aligned_pairs.front().ref_pos;
    return true;
}

bool EventAligner::enter_segment(ReadState& rs)
{
    if (rs.segment_idx >= rs.segments.size()) return false;
    SegmentStart st;
    if (!setup_segment(rs, rs.segment_idx, st)) return false;
    rs.last_event = st.last_event;
    rs.forward = st.first_event < st.last_event;
    rs.curr_start_event = st.first_event;
    rs.curr_start_ref = st.start_ref;
    rs.curr_pair_idx = 0;
    rs.in_segment = true;
    return true;
}

// The part of one iteration of the reference's while loop that comes before profile_hmm_align (eventalign.cpp:691-743).
bool EventAligner::prepare(ReadState& rs, AlignBatch& batch)
{
    while (!rs.done) {
        if (!rs.in_segment) {
            if (!enter_segment(rs)) { rs.done = true; break; }
        }
        const EventAlignmentParameters& p = rs.params;
        const AlignedSegment& aligned_pairs = rs.segments[rs.segment_idx];
        bool issued = false;
        if ((rs.forward && rs.curr_start_event < rs.last_event) || (!rs.forward && rs.curr_start_event > rs.last_event)) {
            const int end_pair_idx = get_end_pair(aligned_pairs, rs.curr_start_ref + ALIGN_STRIDE, rs.curr_pair_idx);
            if (end_pair_idx >= 0) {                              // (-1: the reference would index aligned_pairs[-1])
                const int curr_end_ref = aligned_pairs[end_pair_idx].ref_pos;
                int curr_end_read = aligned_pairs[end_pair_idx].read_pos;
                if (rs.do_base_rc) curr_end_read = p.sr->flip_k_strand(curr_end_read, rs.k);
                const int s = rs.curr_start_ref - p.ref_pos;
                const int l = curr_end_ref - rs.curr_start_ref + 1;
                const int n = (int)rs.ref_seq.length();
                const int n_map = (int)p.sr->base_to_event_map.size();
                if (curr_end_read >= 0 && curr_end_read < n_map && s >= 0 && l >= 0 && s + l <= n) {   // (outside: substr throws / the map is read out of bounds in the reference)
                    rs.fwd_subseq = rs.ref_seq.substr(s, l);
                    rs.rc_subseq = rs.rc_ref_seq.substr(n - s - l, l);
                    // require a minimum amount of sequence to align to
                    if (rs.fwd_subseq.length() >= 2 * rs.k) {
                        const int event_stop = p.sr->get_closest_event_to(curr_end_read, (uint32_t)p.strand_idx);
                        // segments with very few alignable events (large deletions) end the chain
                        if (event_stop >= 0 && rs.curr_start_event >= 0 && std::abs(rs.curr_start_event - event_stop) >= 2) {
                            HMMInputData input;
                            input.read = p.sr;
                            input.pore_model = rs.pore_model;
                            input.event_start_idx = (uint32_t)rs.curr_start_event;
                            input.event_stop_idx = (uint32_t)event_stop;
                            input.strand = (uint8_t)p.strand_idx;
                            input.event_stride = input.event_start_idx < input.event_stop_idx ? 1 : -1;
                            input.rc = p.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;      // rc_flags[strand]
                            HMMInputSequence hmm_sequence(rs.fwd_subseq, rs.rc_subseq, rs.pore_model->pmalphabet);
                            batch.add(hmm_sequence, input, 0);
                            rs.end_pair_idx = end_pair_idx;
                            rs.job_rc = input.rc;
                            rs.pending = true;
                            issued = true;
                        }
                    }
                }
            }
        }
        if (issued) return true;
        // the while loop of this BAM segment is over (condition false or a break): next segment
        rs.in_segment = false;
        rs.segment_idx += 1;
    }
    return false;
}

bool EventAligner::next_round(AlignBatch& batch)
{
    batch.clear_jobs();
    m_round.clear();
    for (size_t i = 0; i < m_reads.size(); ++i) {
        if (m_reads[i].done) continue;
        if (prepare(m_reads[i], batch)) m_round.push_back(i);
    }
    return !m_round.empty();
}

// The part after profile_hmm_align (eventalign.cpp:745-823).
void EventAligner::consume(const std::vector<std::vector<HMMAlignmentState>>& paths)
{
    if (paths.size() != m_round.size()) throw Error(NPH_ERR_STATE, "consume(): one path per job of the round");
    for (size_t j = 0; j < m_round.size(); ++j) {
        ReadState& rs = m_reads[m_round[j]];
        const std::vector<HMMAlignmentState>& event_alignment = paths[j];
        const AlignedSegment& aligned_pairs = rs.segments[rs.segment_idx];
        rs.pending = false;
        rs.segments_aligned += 1;

        size_t num_output = 0;
        // if we aligned to the last pair, output everything and stop
        const bool last_section = rs.end_pair_idx == (int)aligned_pairs.size() - 1;
        int last_event_output = 0;
        int last_ref_kmer_output = 0;
        for (size_t idx = 0; idx < event_alignment.size() && (num_output < (size_t)OUTPUT_STRIDE || last_section); idx++) {
            const HMMAlignmentState& as = event_alignment[idx];
            if (as.state != 'K' && (int)as.event_idx != rs.curr_start_event) {
                rs.output.push_back(Rec{rs.curr_start_ref + (int)as.kmer_idx, (int)as.event_idx, as.state});
                last_event_output = (int)as.event_idx;
                last_ref_kmer_output = rs.curr_start_ref + (int)as.kmer_idx;
                num_output += 1;
            }
        }
        // advance the cursor to where the output stopped
        rs.curr_start_event = last_event_output;
        rs.curr_start_ref = last_ref_kmer_output;
        rs.curr_pair_idx = get_end_pair(aligned_pairs, rs.curr_start_ref, rs.curr_pair_idx);
        if (num_output == 0) {        // break: on to the next BAM segment
            rs.in_segment = false;
            rs.segment_idx += 1;
        }
    }
    m_round.clear();
}

size_t EventAligner::run_rounds(Engine& engine, double indel_bias)
{
    size_t rounds = 0;
    m_batch.clear();
    while (next_round(m_batch)) {
        // AlignBatch uploads the read table again whenever a read shows up that was not resident
        consume(m_batch.run(engine, indel_bias, rounds > 0));
        rounds += 1;
    }
    m_batch.clear();
    return rounds;
}

// the k-mer columns of a record (nph_tsv::ea_kmers_at, the statement the device writer uses too), NUL-terminated
void EventAligner::kmers_at(const ReadState& rs, const Rec& r, char* ref_kmer, char* model_kmer)
{
    const bool rc = rs.params.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;
    const nph_tsv::EaKmers km = nph_tsv::ea_kmers_at(rs.ref_seq.data(), rs.rc_ref_seq.data(), rs.ref_seq.size(),
                                                     (size_t)(r.ref_position - rs.params.ref_pos), rs.k, rc, r.state);
    std::memcpy(ref_kmer, km.ref_kmer, km.ref_kmer_len);
    ref_kmer[km.ref_kmer_len] = 0;
    if (km.model_kmer) std::memcpy(model_kmer, km.model_kmer, rs.k); else std::memset(model_kmer, 'N', rs.k);
    model_kmer[rs.k] = 0;
}

EventAlignment EventAligner::materialize(const ReadState& rs, const Rec& r) const
{
    char ref_kmer[64], model_kmer[64];
    kmers_at(rs, r, ref_kmer, model_kmer);
    EventAlignment ea;
    ea.ref_name = rs.params.ref_name;
    ea.ref_position = r.ref_position;
    ea.ref_kmer = ref_kmer;
    ea.read_idx = (size_t)rs.params.read_idx;
    ea.strand_idx = (int)rs.params.strand_idx;
    ea.event_idx = r.event_idx;
    ea.rc = rs.params.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;
    ea.model_kmer = model_kmer;
    ea.hmm_state = r.state;
    return ea;
}

std::vector<EventAlignment> EventAligner::alignment(size_t read_idx) const
{
    ensure_records();
    const ReadState& rs = m_reads[read_idx];
    std::vector<EventAlignment> out;
    out.reserve(rs.output.size());
    for (const Rec& r : rs.output) out.push_back(materialize(rs, r));
    return out;
}

size_t EventAligner::run(Engine& engine, double indel_bias) { return run_device(engine, indel_bias, nullptr, nullptr); }

EventalignTsv EventAligner::run_tsv(Engine& engine, double indel_bias, const EventalignOptions& opt)
{
    for (const ReadState& rs : m_reads) require_samples(*rs.params.sr, opt);
    EventalignTsv out;
    out.batches = run_device(engine, indel_bias, &opt, &out);
    return out;
}

void EventAligner::require_samples(const SquiggleRead& sr, const EventalignOptions& opt)
{
    if ((opt.write_signal_index || opt.write_samples) && sr.samples.empty())
        throw Error(NPH_ERR_STATE, "--signal-index / --samples need the raw samples on the read (load_from_raw with SRF_LOAD_RAW_SAMPLES)");
}

// Copies the records of the last chain run into the reads' output vectors: chains [chain_first[i], chain_first[i + 1]) are read i's.
void EventAligner::scatter(const nph_ea_record* records, const std::vector<nph_ea_chain>& chains, const std::vector<nph_ea_result>& results,
                           const std::vector<uint64_t>& chain_first, const std::vector<char>& skip)
{
#pragma omp parallel for schedule(dynamic, 8) num_threads(host_threads())
    for (long long i = 0; i < (long long)m_reads.size(); ++i) {
        if (skip[i] || chain_first[i] == chain_first[i + 1]) continue;
        ReadState& rs = m_reads[i];
        size_t total = 0;
        for (size_t c = chain_first[i]; c < chain_first[i + 1]; ++c) total += results[c].n_records;
        rs.output.reserve(rs.output.size() + total);
        for (size_t c = chain_first[i]; c < chain_first[i + 1]; ++c) {
            const nph_ea_record* r = records + chains[c].out_off;
            for (uint32_t j = 0; j < results[c].n_records; ++j) rs.output.push_back(Rec{r[j].ref_position, r[j].event_idx, (char)r[j].hmm_state});
            rs.segments_aligned += results[c].n_windows;
        }
    }
}

void EventAligner::ensure_records() const
{
    if (!m_lazy.engine) return;
    EventAligner* self = const_cast<EventAligner*>(this);
    Engine& engine = *m_lazy.engine;
    self->m_lazy.engine = nullptr;
    nph_ea_record* const records = static_cast<nph_ea_record*>(
        engine.pinned(Engine::Staging::EventalignRecords, sizeof(nph_ea_record) * std::max<uint64_t>(m_lazy.records_total, 1)));
    engine.check(nph_eventalign_records_fetch(engine.ctx(), records, m_lazy.records_total), "nph_eventalign_records_fetch (the engine has run another alignment since run_tsv)");
    self->scatter(records, m_lazy.chains, m_lazy.results, m_lazy.chain_first, std::vector<char>(m_reads.size(), 0));
    self->m_lazy = Lazy();
}

// What nph_eventalign_tsv needs beyond the resident records, staged in page-locked memory; then the call.  Returns the device's
// bytes (in the engine's staging) with read_off and refused filled.
const char* EventAligner::device_tsv(Engine& engine, const EventalignOptions& opt, const std::vector<uint64_t>& chain_first,
                                     const std::vector<size_t>& owner, std::vector<uint64_t>& read_off, std::vector<uint8_t>& refused)
{
    const size_t nr = m_reads.size();
    const bool sample_idx = opt.write_signal_index || opt.write_samples;
    std::vector<nph_ea_tsv_read> tr(nr);
    uint64_t n_text = 0, n_ref = 0, n_events = 0, n_samples = 0;
    for (size_t i = 0; i < nr; ++i) {
        const ReadState& rs = m_reads[i];
        const SquiggleRead& sr = *rs.params.sr;
        nph_ea_tsv_read& t = tr[i];
        std::memset(&t, 0, sizeof(t));
        if (chain_first[i] == chain_first[i + 1]) continue;            // no chain, no row: empty slices
        t.contig_off = n_text; t.contig_len = (uint32_t)rs.params.ref_name.size(); n_text += t.contig_len;
        t.name_off = n_text; t.name_len = (uint32_t)sr.read_name.size(); n_text += t.name_len;
        t.ref_off = n_ref; t.ref_len = (uint32_t)rs.ref_seq.size(); n_ref += t.ref_len;
        t.event_off = n_events; t.n_events = (uint32_t)sr.events[rs.params.strand_idx].size(); n_events += t.n_events;
        if (opt.write_samples) { t.sample_off = n_samples; t.n_samples = sr.samples.size(); n_samples += t.n_samples; }
        t.read_idx = (uint64_t)(size_t)rs.params.read_idx;
        t.sample_start_time = sr.sample_start_time; t.sample_rate = sr.sample_rate;
        t.drift = sr.scalings[rs.params.strand_idx].drift;
        t.strand_idx = (uint32_t)rs.params.strand_idx;
    }
    // one staging block: start times | means | stdv | durations | samples | text | ref | rc_ref
    const size_t b_time = sizeof(double) * (sample_idx ? n_events : 0), b_f = sizeof(float) * n_events;
    char* const in = static_cast<char*>(engine.pinned(Engine::Staging::EventalignTsvIn, b_time + 3 * b_f + sizeof(float) * n_samples + n_text + 2 * n_ref + 8));
    double* const time = reinterpret_cast<double*>(in);
    float* const mean = reinterpret_cast<float*>(in + b_time);
    float* const stdv = mean + n_events;
    float* const dur = stdv + n_events;
    float* const samples = dur + n_events;
    char* const text = reinterpret_cast<char*>(samples + n_samples);
    char* const ref = text + n_text;
    char* const rc_ref = ref + n_ref;
    parallel_for(nr, host_threads(), 8, [&](size_t i) {
        const nph_ea_tsv_read& t = tr[i];
        if (chain_first[i] == chain_first[i + 1]) return;
        const ReadState& rs = m_reads[i];
        const SquiggleRead& sr = *rs.params.sr;
        const std::vector<SquiggleEvent>& ev = sr.events[rs.params.strand_idx];
        for (size_t e = 0; e < ev.size(); ++e) {
            mean[t.event_off + e] = ev[e].mean; stdv[t.event_off + e] = ev[e].stdv; dur[t.event_off + e] = ev[e].duration;
            if (sample_idx) time[t.event_off + e] = ev[e].start_time;
        }
        if (opt.write_samples) std::memcpy(samples + t.sample_off, sr.samples.data(), sizeof(float) * sr.samples.size());
        std::memcpy(text + t.contig_off, rs.params.ref_name.data(), t.contig_len);
        std::memcpy(text + t.name_off, sr.read_name.data(), t.name_len);
        std::memcpy(ref + t.ref_off, rs.ref_seq.data(), t.ref_len);
        std::memcpy(rc_ref + t.ref_off, rs.rc_ref_seq.data(), t.ref_len);
    });
    std::vector<uint32_t> chain_read(owner.size());
    for (size_t c = 0; c < owner.size(); ++c) chain_read[c] = (uint32_t)owner[c];
    nph_ea_tsv_batch b;
    std::memset(&b, 0, sizeof(b));
    b.reads = tr.data(); b.n_reads = nr; b.chain_read = chain_read.data();
    b.text = text; b.n_text = n_text; b.ref = ref; b.rc_ref = rc_ref; b.n_ref = n_ref;
    b.ev_mean = mean; b.ev_stdv = stdv; b.ev_duration = dur; b.ev_start_time = sample_idx ? time : nullptr; b.n_events = n_events;
    b.samples = opt.write_samples ? samples : nullptr; b.n_samples = n_samples;
    const nph_ea_tsv_options o{opt.print_read_names, opt.scale_events, opt.write_signal_index, opt.write_samples};
    read_off.assign(nr + 1, 0);
    refused.assign(nr, 0);
    // the staging of the previous batch is usually large enough; when it is not, the call reports the bytes it needs
    size_t cap = 0;
    char* buf = static_cast<char*>(engine.pinned_if_any(Engine::Staging::EventalignTsv, &cap));
    uint64_t n_bytes = 0;
    int rc = nph_eventalign_tsv(engine.ctx(), &b, &o, buf, cap, nullptr, read_off.data(), refused.data(), &n_bytes);
    if (rc == NPH_ERR_INVALID && n_bytes > cap) {
        buf = static_cast<char*>(engine.pinned(Engine::Staging::EventalignTsv, (size_t)n_bytes));
        rc = nph_eventalign_tsv(engine.ctx(), &b, &o, buf, (size_t)n_bytes, nullptr, read_off.data(), refused.data(), &n_bytes);
    }
    engine.check(rc, "nph_eventalign_tsv");
    return buf;
}

size_t EventAligner::run_device(Engine& engine, double indel_bias, const EventalignOptions* tsv_opt, EventalignTsv* tsv_out)
{
    m_lazy = Lazy();
    const size_t nr = m_reads.size();
    if (tsv_out) { tsv_out->read_off.assign(nr + 1, 0); tsv_out->on_host.assign(nr, 0); }
    // ---- phase 1 (parallel over reads): trims and start/stop events of every BAM segment, up to the first segment
    //      that trims to nothing (where the reference returns from align_read_to_ref) ----
    std::vector<std::vector<SegmentStart>> starts(nr);
    parallel_for(nr, host_threads(), 8, [&](size_t i) {
        ReadState& rs = m_reads[i];
        if (rs.done) return;
        if (rs.k >= 64) throw Error(NPH_ERR_UNSUPPORTED, "k-mer length");
        for (size_t sidx = 0; sidx < rs.segments.size(); ++sidx) {
            SegmentStart st;
            if (!setup_segment(rs, sidx, st)) break;
            starts[i].push_back(st);
        }
    });

    // ---- phase 2 (serial, O(reads)): read table, offsets ----
    detail::ReadTable read_table;
    std::vector<uint64_t> map_off;                          // per read_table entry: where its base-to-event map starts
    std::vector<uint32_t> read_of(nr, 0);                   // per read: its read_table entry
    std::vector<char> fills_map(nr, 0);
    std::vector<uint64_t> rank_off(nr, 0), chain_first(nr + 1, 0);
    std::vector<uint32_t> model_of(nr, 0);
    uint64_t n_map = 0, n_ranks = 0, n_pairs = 0, records_total = 0;
    for (size_t i = 0; i < nr; ++i) {
        chain_first[i + 1] = chain_first[i] + starts[i].size();
        if (starts[i].empty()) continue;
        const ReadState& rs = m_reads[i];
        const EventAlignmentParameters& p = rs.params;
        read_of[i] = read_table.index(p.sr, (uint8_t)p.strand_idx);
        if (read_of[i] == map_off.size()) {
            map_off.push_back(n_map);
            n_map += p.sr->base_to_event_map.size();
            fills_map[i] = 1;
        }
        rank_off[i] = n_ranks;
        n_ranks += rs.ref_seq.size() >= rs.k ? rs.ref_seq.size() - rs.k + 1 : 0;
        model_of[i] = engine.model_id(rs.pore_model);
    }
    const size_t n_chains = (size_t)chain_first[nr];
    for (ReadState& rs : m_reads) rs.done = true;             // nothing left for the round driver unless re-armed below
    if (n_chains == 0) return 0;
    std::vector<nph_ea_chain> chains(n_chains);
    std::vector<size_t> owner(n_chains);
    for (size_t i = 0; i < nr; ++i) {
        const ReadState& rs = m_reads[i];
        for (size_t sidx = 0; sidx < starts[i].size(); ++sidx) {
            const SegmentStart& st = starts[i][sidx];
            nph_ea_chain& c = chains[chain_first[i] + sidx];
            std::memset(&c, 0, sizeof(c));
            c.pair_off = n_pairs;
            c.n_pairs = (uint32_t)rs.segments[sidx].size();
            n_pairs += c.n_pairs;
            c.out_cap = (uint32_t)std::abs(st.last_event - st.first_event) + 2;
            c.out_off = records_total;
            records_total += c.out_cap;
            owner[chain_first[i] + sidx] = i;
        }
    }

    // ---- phase 3 (parallel over reads): pairs, event maps, rank tables, chain records ----
    std::vector<nph_aligned_pair> pairs(std::max<uint64_t>(n_pairs, 1));
    std::vector<int32_t> map_start(std::max<uint64_t>(n_map, 1));
    std::vector<uint32_t> ranks_fwd(std::max<uint64_t>(n_ranks, 1)), ranks_rc(std::max<uint64_t>(n_ranks, 1));
#pragma omp parallel for schedule(dynamic, 8) num_threads(host_threads())
    for (long long i = 0; i < (long long)nr; ++i) {
        if (starts[i].empty()) continue;
        const ReadState& rs = m_reads[i];
        const EventAlignmentParameters& p = rs.params;
        if (fills_map[i]) {
            int32_t* m = map_start.data() + map_off[read_of[i]];
            const std::vector<EventRangeForBase>& b2e = p.sr->base_to_event_map;
            for (size_t j = 0; j < b2e.size(); ++j) m[j] = b2e[j].indices[p.strand_idx].start;
        }
        const size_t n = rs.ref_seq.size();
        const Alphabet& alphabet = *rs.pore_model->pmalphabet;
        kmer_ranks(alphabet, rs.ref_seq.data(), n, rs.k, false, ranks_fwd.data() + rank_off[i]);
        // entry pos of the rc table = rank of rc_ref_seq's k-mer at n - pos - k (what get_kmer_rank(ki, k, true) resolves to)
        kmer_ranks(alphabet, rs.rc_ref_seq.data(), rs.rc_ref_seq.size(), rs.k, true, ranks_rc.data() + rank_off[i]);
        for (size_t sidx = 0; sidx < starts[i].size(); ++sidx) {
            const SegmentStart& st = starts[i][sidx];
            nph_ea_chain& c = chains[chain_first[i] + sidx];
            nph_aligned_pair* dst = pairs.data() + c.pair_off;
            const AlignedSegment& seg = rs.segments[sidx];
            for (size_t j = 0; j < seg.size(); ++j) dst[j] = nph_aligned_pair{seg[j].ref_pos, seg[j].read_pos};
            c.map_off = map_off[read_of[i]];
            c.map_len = (uint32_t)p.sr->base_to_event_map.size();
            c.rank_off = rank_off[i];
            c.ref_len = (uint32_t)n;
            c.read = read_of[i];
            c.model_id = model_of[i];
            c.read_seq_len = (uint32_t)p.sr->read_sequence.size();
            c.ref_offset = p.ref_pos;
            c.first_event = st.first_event;
            c.last_event = st.last_event;
            c.do_base_rc = rs.do_base_rc;
            c.rc = p.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;
            c.k = (uint8_t)rs.k;
        }
    }

    // ---- the device: reads up, one launch, records back ----
    const detail::FlatReads fr = detail::flatten_reads(engine, read_table);
    engine.check(nph_reads_load(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events), "nph_reads_load");
    std::vector<nph_ea_result> results(n_chains);
    engine.check(nph_eventalign_chain_run(engine.ctx(), pairs.data(), pairs.size(), map_start.data(), map_start.size(), ranks_fwd.data(),
                                          ranks_rc.data(), ranks_fwd.size(), chains.data(), n_chains, indel_bias, records_total, results.data()),
                 "nph_eventalign_chain_run");

    // ---- scatter (parallel over reads); a read with a window the chain kernel could not hold goes through the round
    //      driver instead ----
    std::vector<char> redo(nr, 0);
    for (size_t c = 0; c < n_chains; ++c) {
        const int st = results[c].status;
        if (st & NPH_EA_RC_STRIDE) throw Error(NPH_ERR_INVALID, "rc and event_stride disagree");     // ref asserts (profile_hmm_r9.inl:275)
        if (st & NPH_EA_BAD_EVENT) throw Error(NPH_ERR_INVALID, "event index outside the read");
        if (st & NPH_EA_OUT_OVERFLOW) throw Error(NPH_ERR_STATE, "eventalign chain: record room exceeded");
        if (st & NPH_EA_WINDOW_TOO_LARGE) redo[owner[c]] = 1;
    }
    size_t n_redo = 0;
    for (size_t i = 0; i < nr; ++i) n_redo += redo[i] != 0;
    // the rows, where the records are: every read but those the writer refuses or the round driver re-runs
    const char* dev_text = nullptr;
    std::vector<uint64_t> dev_off;
    std::vector<uint8_t> refused;
    bool any_refused = false;
    if (tsv_opt) {
        dev_text = device_tsv(engine, *tsv_opt, chain_first, owner, dev_off, refused);
        for (size_t i = 0; i < nr; ++i) any_refused = any_refused || (refused[i] && !redo[i]);
    }
    if (tsv_opt && !n_redo && !any_refused) {
        // nothing needs the records on the host now: they are fetched if alignment(), sam() or summarize() ask
        m_lazy.engine = &engine; m_lazy.records_total = records_total;
        m_lazy.chains.swap(chains); m_lazy.results.swap(results); m_lazy.chain_first = chain_first;
        tsv_out->m_view = dev_text; tsv_out->m_size = (size_t)dev_off[nr]; tsv_out->read_off = dev_off;
        return 1;
    }
    nph_ea_record* const records = static_cast<nph_ea_record*>(
        engine.pinned(Engine::Staging::EventalignRecords, sizeof(nph_ea_record) * std::max<uint64_t>(records_total, 1)));
    engine.check(nph_eventalign_records_fetch(engine.ctx(), records, records_total), "nph_eventalign_records_fetch");
    scatter(records, chains, results, chain_first, redo);
    for (size_t i = 0; i < nr; ++i) {
        if (!redo[i]) continue;
        ReadState& rs = m_reads[i];
        rs.done = false; rs.in_segment = false; rs.segment_idx = 0; rs.pending = false;
        rs.output.clear(); rs.segments_aligned = 0;
    }
    const size_t batches = 1 + (n_redo ? run_rounds(engine, indel_bias) : 0);
    if (tsv_opt) {
        // the reads the device did not write take the host writer; the others keep the device's bytes
        std::vector<std::string> host_rows(nr);
        parallel_for(nr, host_threads(), 4, [&](size_t i) { if (redo[i] || refused[i]) host_rows[i] = tsv(i, *tsv_opt); });
        for (size_t i = 0; i < nr; ++i) {
            const bool on_host = redo[i] || refused[i];
            tsv_out->on_host[i] = on_host;
            tsv_out->read_off[i + 1] = tsv_out->read_off[i] + (on_host ? host_rows[i].size() : dev_off[i + 1] - dev_off[i]);
        }
        tsv_out->m_owned.resize((size_t)tsv_out->read_off[nr]);
        parallel_for(nr, host_threads(), 4, [&](size_t i) {
            if (tsv_out->read_off[i + 1] == tsv_out->read_off[i]) return;
            char* dst = &tsv_out->m_owned[0] + tsv_out->read_off[i];
            if (tsv_out->on_host[i]) std::memcpy(dst, host_rows[i].data(), host_rows[i].size());
            else std::memcpy(dst, dev_text + dev_off[i], (size_t)(dev_off[i + 1] - dev_off[i]));
        });
        tsv_out->m_view = nullptr; tsv_out->m_size = tsv_out->m_owned.size();
    }
    return batches;
}

// ---------------------------------------------------------------------------------------------
// writers
// ---------------------------------------------------------------------------------------------
using nph_tsv::put_i64;
static inline char* put_str(char* o, const char* s, size_t n) { std::memcpy(o, s, n); return o + n; }

std::string EventAligner::tsv_header(const EventalignOptions& opt)
{
    std::string h = "contig\tposition\treference_kmer\t";
    h += opt.print_read_names ? "read_name" : "read_index";
    h += "\tstrand\tevent_index\tevent_level_mean\tevent_stdv\tevent_length\tmodel_kmer\tmodel_mean\tmodel_stdv\tstandardized_level";
    if (opt.write_signal_index) h += "\tstart_idx\tend_idx";
    if (opt.write_samples) h += "\tsamples";
    h += "\n";
    return h;
}

std::string EventAligner::tsv(size_t read_idx, const EventalignOptions& opt) const
{
    ensure_records();
    const ReadState& rs = m_reads[read_idx];
    const SquiggleRead& sr = *rs.params.sr;
    const PoreModel* pore_model = rs.pore_model;
    const uint32_t k = pore_model->k;
    const uint32_t strand = (uint32_t)rs.params.strand_idx;
    const std::string& ref_name = rs.params.ref_name;
    // the read column: read_idx as %zu, or the read name with -n
    const std::string who_s = opt.print_read_names ? sr.read_name : std::to_string((size_t)rs.params.read_idx);
    const double sqrt_var = std::sqrt(sr.scalings[strand].var);
    require_samples(sr, opt);
    // room per row: six numbers of at most 47 characters; with the sample columns, 16 characters per raw sample of the
    // events written (%g, six significant digits) + two indices
    size_t extra = 0;
    if (opt.write_signal_index) extra += 48 * rs.output.size();
    if (opt.write_samples)
        for (const Rec& r : rs.output) {
            const std::pair<size_t, size_t> si = sr.get_event_sample_idx(strand, r.event_idx);
            extra += 2 + 16 * (si.second > si.first ? si.second - si.first : 0);
        }
    std::string out;
    out.resize(rs.output.size() * (ref_name.size() + who_s.size() + 2 * (size_t)k + 340) + extra);
    char* const base = &out[0];
    char* o = base;
    const bool rc = rs.params.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;
    const bool sample_idx = opt.write_signal_index || opt.write_samples;
    const SquiggleScalings& sc = sr.scalings[strand];
    const nph_tsv::EaRead rd{sc.scale, sc.shift, sc.drift, sc.var, sqrt_var, sr.sample_rate, sr.sample_start_time};
    nph_tsv::EaRow w;
    w.contig = ref_name.data(); w.contig_len = (uint32_t)ref_name.size();
    w.k = k;
    w.name = opt.print_read_names ? who_s.data() : nullptr; w.name_len = (uint32_t)who_s.size();
    w.read_idx = (uint64_t)(size_t)rs.params.read_idx;
    w.strand = "tc"[strand];
    w.signal_index = opt.write_signal_index;
    for (const Rec& r : rs.output) {
        // the row rule of csrc/tsv_format.cuh, shared with the device writer
        w.kmers = nph_tsv::ea_kmers_at(rs.ref_seq.data(), rs.rc_ref_seq.data(), rs.ref_seq.size(), (size_t)(r.ref_position - rs.params.ref_pos),
                                       k, rc, r.state);
        w.ref_position = r.ref_position;
        w.event_idx = r.event_idx;
        PoreModelStateParams model;
        if (r.state != 'B') model = pore_model->get_parameters(pore_model->pmalphabet->kmer_rank(w.kmers.model_kmer, k));
        const SquiggleEvent& ev = sr.events[strand][r.event_idx];
        const nph_tsv::EaRowNums n = nph_tsv::ea_row_numbers(ev.mean, opt.scale_events ? sr.get_drift_scaled_level(r.event_idx, strand) : 0.0f, ev.stdv,
                                                             ev.duration, ev.start_time, r.state, model.level_mean, model.level_stdv, rd,
                                                             opt.scale_events, sample_idx);
        if (n.ok) {
            o = nph_tsv::put_ea_row(o, w, n);
        } else {
            // a value the exact formatter does not take: this row through the C library
            o = put_str(o, ref_name.data(), ref_name.size()); *o++ = '\t';
            o = put_i64(o, r.ref_position); *o++ = '\t';
            o = put_str(o, w.kmers.ref_kmer, w.kmers.ref_kmer_len); *o++ = '\t';
            o = put_str(o, who_s.data(), who_s.size()); *o++ = '\t';
            *o++ = w.strand; *o++ = '\t';
            o = put_i64(o, r.event_idx); *o++ = '\t';
            o += format_fixed(o, n.event_mean, 2); *o++ = '\t';
            o += format_fixed(o, ev.stdv, 3); *o++ = '\t';
            o += format_fixed(o, ev.duration, 5); *o++ = '\t';
            if (w.kmers.model_kmer) o = put_str(o, w.kmers.model_kmer, k); else { std::memset(o, 'N', k); o += k; }
            *o++ = '\t';
            o += format_fixed(o, n.model_mean, 2); *o++ = '\t';
            o += format_fixed(o, n.model_stdv, 2); *o++ = '\t';
            o += format_fixed(o, n.standard_level, 2);
            if (opt.write_signal_index) {
                const std::pair<size_t, size_t> si = sr.get_event_sample_idx(strand, r.event_idx);
                o += snprintf(o, 48, "\t%zu\t%zu", si.first, si.second);
            }
        }
        if (opt.write_samples) {
            // the reference streams the floats through an ostream (%g, 6 significant digits) with ',' after each and
            // drops the last comma (an event without samples makes it resize() to npos and throw; here: an empty column)
            const std::pair<size_t, size_t> si = sr.get_event_sample_idx(strand, r.event_idx);
            *o++ = '\t';
            for (size_t i = si.first; i < si.second; ++i) {
                if (i != si.first) *o++ = ',';
                const float v = nph_tsv::ea_scaled_sample(sr.samples.at(i), i, rd);
                const nph_tsv::G6 g = nph_tsv::g6_of(v);
                if (g.ok) o = nph_tsv::put_g6(o, g); else o += snprintf(o, 32, "%g", (double)v);
            }
        }
        *o++ = '\n';
    }
    out.resize((size_t)(o - base));
    return out;
}

std::vector<std::string> EventAligner::tsv_batch(const EventalignOptions& opt) const
{
    ensure_records();
    std::vector<std::string> out(m_reads.size());
    // rows of different reads are independent; the reference formats them one read at a time inside an omp critical
    parallel_for(m_reads.size(), host_threads(), 4, [&](size_t i) { out[i] = tsv(i, opt); });
    return out;
}

std::vector<uint32_t> event_alignment_to_cigar(const std::vector<EventAlignment>& alignments)
{
    std::vector<uint32_t> out;
    if (alignments.empty()) return out;
    // a soft clip accounts for unaligned events at the beginning of the read
    if (alignments[0].event_idx > 0) out.push_back((uint32_t)alignments[0].event_idx << 4 | NPH_CIGAR_S);
    out.push_back(1u << 4 | NPH_CIGAR_M);       // always starts with a match
    int prev_r_idx = alignments[0].ref_position;
    int prev_e_idx = alignments[0].event_idx;
    for (size_t ai = 1; ai < alignments.size(); ++ai) {
        const int r_idx = alignments[ai].ref_position, e_idx = alignments[ai].event_idx;
        const int r_step = std::abs(r_idx - prev_r_idx), e_step = std::abs(e_idx - prev_e_idx);
        uint32_t incoming;
        if (r_step == 1 && e_step == 1) {
            incoming = 1u << 4 | NPH_CIGAR_M;
        } else if (r_step > 1) {
            // a reference jump of more than one is a deletion followed by a new match (the reference asserts e_step == 1)
            out.push_back((uint32_t)(r_step - 1) << 4 | NPH_CIGAR_D);
            incoming = 1u << 4 | NPH_CIGAR_M;
        } else {
            incoming = 1u << 4 | NPH_CIGAR_I;   // (the reference asserts e_step == 1 && r_step == 0)
        }
        if ((out.back() & 0xf) == (incoming & 0xf)) out.back() = ((out.back() >> 4) + (incoming >> 4)) << 4 | (incoming & 0xf);
        else out.push_back(incoming);
        prev_r_idx = r_idx;
        prev_e_idx = e_idx;
    }
    return out;
}

std::string cigar_ops_to_string(const std::vector<uint32_t>& ops)
{
    std::string s;
    for (uint32_t c : ops) { s += std::to_string(c >> 4); s += "MIDNSHP=XB"[c & 0xf]; }
    return s;
}

std::string EventAligner::event_cigar(size_t read_idx) const
{
    return cigar_ops_to_string(event_alignment_to_cigar(alignment(read_idx)));
}

std::string EventAligner::sam(size_t read_idx) const
{
    ensure_records();
    const ReadState& rs = m_reads[read_idx];
    const std::vector<Rec>& al = rs.output;
    if (al.empty()) return std::string();
    const bool rc = rs.params.strand_idx == 0 ? rs.do_base_rc : !rs.do_base_rc;
    const std::string qname = rs.params.sr->read_name + (rs.params.strand_idx == 0 ? ".template" : ".complement");
    const int stride = al.front().event_idx < al.back().event_idx ? 1 : -1;
    // QNAME FLAG RNAME POS MAPQ CIGAR RNEXT PNEXT TLEN SEQ QUAL + the event-stride tag
    return qname + "\t" + std::to_string(rc ? 16 : 0) + "\t" + rs.params.ref_name + "\t" + std::to_string(al.front().ref_position + 1) + "\t" +
           std::to_string((int)rs.params.mapq) + "\t" + event_cigar(read_idx) + "\t*\t0\t0\t*\t*\tES:i:" + std::to_string(stride) + "\n";
}

EventalignSummary EventAligner::summarize(size_t read_idx) const
{
    ensure_records();
    const ReadState& rs = m_reads[read_idx];
    const SquiggleRead& sr = *rs.params.sr;
    EventalignSummary summary;
    uint64_t prev_ref_pos = ~(uint64_t)0;                  // std::string::npos
    const uint32_t strand = (uint32_t)rs.params.strand_idx;
    char ref_kmer[64], model_kmer[64];
    for (size_t i = 0; i < rs.output.size(); ++i) {
        const Rec& ea = rs.output[i];
        summary.num_events += 1;
        const uint64_t ref_move = (uint64_t)(int64_t)ea.ref_position - prev_ref_pos;    // size_t arithmetic, as the reference
        if (ref_move == 0) summary.num_stays += 1;
        else if (i != 0 && ref_move > 1) summary.num_skips += 1;
        else if (i != 0 && ref_move == 1) summary.num_steps += 1;
        summary.sum_duration += sr.get_duration(ea.event_idx, strand);
        if (ea.state == 'M') {
            kmers_at(rs, ea, ref_kmer, model_kmer);
            const uint32_t rank = rs.pore_model->pmalphabet->kmer_rank(model_kmer, rs.k);
            // z_score (src/hmm/nanopolish_emissions.h:32-41): float arithmetic
            const float level = sr.get_drift_scaled_level(ea.event_idx, strand);
            const GaussianParameters gp = sr.get_scaled_gaussian_from_pore_model_state(*rs.pore_model, strand, rank);
            const float z = (level - gp.mean) / gp.stdv;
            summary.sum_z_score += z;
        }
        prev_ref_pos = (uint64_t)(int64_t)ea.ref_position;
    }
    summary.alignment_edit_distance = rs.params.edit_distance;
    if (!rs.output.empty()) summary.reference_span = rs.output.back().ref_position - rs.output.front().ref_position + 1;
    return summary;
}

std::string EventAligner::summary_row(size_t read_idx, const std::string& fast5_path) const
{
    const ReadState& rs = m_reads[read_idx];
    const EventalignSummary summary = summarize(read_idx);
    if (summary.num_events <= 0) return std::string();
    const SquiggleScalings& scalings = rs.params.sr->scalings[rs.params.strand_idx];
    char buf[2048];
    std::string out;
    snprintf(buf, sizeof(buf), "%zu\t%s\t%s\t", (size_t)rs.params.read_idx, rs.params.sr->read_name.c_str(), fast5_path.c_str());
    out += buf;
    snprintf(buf, sizeof(buf), "%s\t%s\t", rs.pore_model->name.c_str(), rs.params.strand_idx == 0 ? "template" : "complement");
    out += buf;
    snprintf(buf, sizeof(buf), "%d\t%d\t%d\t%d\t", summary.num_events, summary.num_steps, summary.num_skips, summary.num_stays);
    out += buf;
    snprintf(buf, sizeof(buf), "%.2lf\t%.3lf\t%.3lf\t%.3lf\t%.3lf\n", summary.sum_duration, scalings.shift, scalings.scale, scalings.drift, scalings.var);
    out += buf;
    return out;
}

} // namespace nph
