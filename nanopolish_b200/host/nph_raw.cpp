// nph_raw.cpp — see nph_raw.hpp.
#include "nph_raw.hpp"

#include <algorithm>
#include <cmath>

namespace nph {

const nph_event_params event_detection_defaults = {3, 6, 1.4f, 9.0f, 0.2f, 0};
const nph_event_params event_detection_rna = {7, 14, 2.5f, 9.0f, 1.0f, 1};      // + events turned around to 5'->3' by load_from_raw

namespace {

// event detection over [start, end) of each signal; grows the per-read room once if the first guess was short
std::vector<std::vector<nph_event>> detect_batch(Engine& engine, const std::vector<float>& flat, const std::vector<uint64_t>& off,
                                                 const std::vector<nph_raw_range>& range, const nph_event_params& prm)
{
    const size_t n = range.size();
    std::vector<std::vector<nph_event>> out(n);
    std::vector<uint32_t> live;
    for (size_t i = 0; i < n; ++i) if (range[i].end > range[i].start) live.push_back((uint32_t)i);
    if (live.empty()) return out;
    for (int attempt = 0; attempt < 2; ++attempt) {
        std::vector<nph_raw_read> rr(live.size());
        uint64_t room = 0;
        for (size_t t = 0; t < live.size(); ++t) {
            const uint32_t i = live[t];
            const uint32_t ns = range[i].end - range[i].start;
            rr[t].sample_off = off[i] + range[i].start;
            rr[t].n_samples = ns;
            rr[t].event_cap = attempt == 0 ? ns / 2 + 8 : ns;      // n_samples always suffices
            rr[t].event_off = room;
            room += rr[t].event_cap;
        }
        std::vector<nph_event> ev(room);
        std::vector<uint32_t> cnt(live.size());
        const int rc = nph_detect_events_batch(engine.ctx(), flat.data(), flat.size(), rr.data(), rr.size(), &prm, ev.data(), ev.size(), cnt.data());
        if (rc == NPH_ERR_UNSUPPORTED && attempt == 0) continue;
        engine.check(rc, "nph_detect_events_batch");
        for (size_t t = 0; t < live.size(); ++t) out[live[t]].assign(ev.begin() + rr[t].event_off, ev.begin() + rr[t].event_off + cnt[t]);
        break;
    }
    return out;
}

} // namespace

std::vector<nph_event> detect_events(Engine& engine, const std::vector<float>& samples, const nph_event_params& params)
{
    if (samples.empty()) return {};
    return detect_batch(engine, samples, {0}, {nph_raw_range{0u, (uint32_t)samples.size()}}, params)[0];
}

nph_raw_range trim_and_segment_raw(Engine& engine, const std::vector<float>& samples, int trim_start, int trim_end, int varseg_chunk,
                                   float varseg_thresh)
{
    nph_raw_range out{0, 0};
    if (samples.empty()) return out;
    nph_raw_read rr{};
    rr.n_samples = (uint32_t)samples.size();
    engine.check(nph_trim_raw_batch(engine.ctx(), samples.data(), samples.size(), &rr, 1, trim_start, trim_end, varseg_chunk, varseg_thresh, &out),
                 "nph_trim_raw_batch");
    return out;
}

std::vector<std::unique_ptr<SquiggleRead>> load_from_raw(Engine& engine, const PoreModel& base_model, const std::vector<RawRead>& raw,
                                                         LoadFromRawStats* stats, uint32_t flags)
{
    const size_t n = raw.size();
    LoadFromRawStats st;
    st.total = n;
    std::vector<std::unique_ptr<SquiggleRead>> reads(n);
    const uint32_t k = base_model.k;
    // direct RNA (squiggle_read.cpp:192-213): the caller passes the r9.4_70bps u_to_t_rna 5-mer model; the basecall's
    // U become T, the RNA detector parameters apply and the events are turned around to 5'->3'
    bool rna = false;
    for (size_t i = 0; i < n; ++i) rna = rna || raw[i].nucleotide_type == SRNT_RNA;
    for (size_t i = 0; i < n; ++i)
        if ((raw[i].nucleotide_type == SRNT_RNA) != rna) throw Error(NPH_ERR_INVALID, "load_from_raw: DNA and RNA reads in one batch (they use different models)");
    for (size_t i = 0; i < n; ++i) {
        reads[i].reset(new SquiggleRead());
        SquiggleRead& sr = *reads[i];
        sr.read_name = raw[i].read_name;
        sr.read_sequence = raw[i].read_sequence;
        sr.nucleotide_type = raw[i].nucleotide_type;
        if (rna) std::replace(sr.read_sequence.begin(), sr.read_sequence.end(), 'U', 'T');
        sr.pore_type = PORETYPE_R9;
        sr.base_model[0] = &base_model;
        sr.sample_rate = raw[i].sample_rate;
    }
    // reads the device call cannot take (no samples, sequence shorter than a k-mer) fail like a read that trims to nothing
    std::vector<uint32_t> sent;
    std::vector<nph_raw_job> jobs;
    std::vector<uint32_t> ranks;
    size_t total = 0;
    for (size_t i = 0; i < n; ++i) {
        const std::string& seq = reads[i]->read_sequence;
        if (raw[i].samples.empty() || seq.size() < k || !(raw[i].sample_rate > 0.0)) { ++st.empty_after_trim; continue; }
        const uint32_t n_kmers = (uint32_t)(seq.size() - k + 1);
        jobs.push_back(nph_raw_job{total, ranks.size(), (uint32_t)raw[i].samples.size(), n_kmers, raw[i].sample_rate});
        ranks.resize(ranks.size() + n_kmers);
        kmer_ranks(*base_model.pmalphabet, seq.data(), seq.size(), k, false, ranks.data() + jobs.back().rank_off);
        total += raw[i].samples.size();
        sent.push_back((uint32_t)i);
    }
    if (sent.empty()) { if (stats) *stats = st; return reads; }
    std::vector<float> flat(total);
    for (size_t t = 0; t < sent.size(); ++t) std::copy(raw[sent[t]].samples.begin(), raw[sent[t]].samples.end(), flat.begin() + jobs[t].sample_off);

    const size_t cap = total / 3 + 16 * sent.size();
    std::vector<uint64_t> off(sent.size() + 1);
    std::vector<float> mean(cap), stdv(cap), dur(cap);
    std::vector<double> start(cap);
    std::vector<nph_event_range> b2e(ranks.size());
    std::vector<nph_calibration> cal(sent.size());
    engine.check(nph_load_from_raw_batch(engine.ctx(), flat.data(), flat.size(), ranks.data(), ranks.size(), jobs.data(), jobs.size(),
                                         engine.model_id(&base_model), rna ? &event_detection_rna : &event_detection_defaults, off.data(), mean.data(), stdv.data(),
                                         start.data(), dur.data(), cap, b2e.data(), cal.data()),
                 "nph_load_from_raw_batch");

    if (flags & SRF_LOAD_RAW_SAMPLES) {         // squiggle_read.cpp:251-258, before any of the read's QC
        std::vector<nph_raw_range> kept(sent.size());
        engine.check(nph_last_trim_ranges(engine.ctx(), kept.data(), kept.size()), "nph_last_trim_ranges");
        for (size_t t = 0; t < sent.size(); ++t) {
            SquiggleRead& sr = *reads[sent[t]];
            sr.sample_start_time = 0;
            sr.samples.assign(raw[sent[t]].samples.begin() + kept[t].start, raw[sent[t]].samples.begin() + kept[t].end);
        }
    }
    for (size_t t = 0; t < sent.size(); ++t) {
        SquiggleRead& sr = *reads[sent[t]];
        const nph_calibration& c = cal[t];
        if (c.status & NPH_CAL_EMPTY_AFTER_TRIM) { ++st.empty_after_trim; continue; }
        // scalings: the MoM estimate, replaced by the recalibrated set unless recalibration was refused
        sr.scalings[0].set4(c.shift, c.scale, c.drift, c.var);
        if (c.status & NPH_CAL_NOT_ALIGNED) {                      // squiggle_read.cpp:324-329
            sr.events_per_base[0] = 0.0;
            ++st.failed_alignment;
            continue;
        }
        sr.base_to_event_map.resize(jobs[t].n_kmers);
        for (uint32_t i = 0; i < jobs[t].n_kmers; ++i) {
            const nph_event_range& r = b2e[jobs[t].rank_off + i];
            sr.base_to_event_map[i].indices[0] = IndexPair{r.start, r.stop};
        }
        sr.events_per_base[0] = c.events_per_base;
        if (c.status & (NPH_CAL_TOO_FEW_EVENTS | NPH_CAL_HIGH_VAR)) { ++st.failed_calibration; continue; }   // :319-323
        if (c.status & NPH_CAL_TOO_MANY_STAYS) { ++st.qc_fail; continue; }                                      // :331-336
        const size_t ne = off[t + 1] - off[t];
        sr.events[0].resize(ne);
        for (size_t e = 0; e < ne; ++e) {
            const size_t g = off[t] + e;
            sr.events[0][e] = SquiggleEvent{mean[g], stdv[g], start[g], dur[g], logf(stdv[g])};
        }
        sr.event_mean_cache[0].assign(mean.begin() + (long)off[t], mean.begin() + (long)(off[t] + ne));        // the contiguous copy batching reads from (nph_host.hpp)
    }
    if (stats) *stats = st;
    return reads;
}

} // namespace nph
