// nph_polya.cpp — see nph_polya.hpp
#include "nph_polya.hpp"

#include <cstdio>

namespace nph {

namespace {

// add()'s rules, the same for polya and detect-polyi: false (no row) for a secondary alignment
bool accept(const PolyaRecord& rec, const char* who)
{
    if (rec.flag & BAM_FSECONDARY) return false;                     // :743-745
    if (rec.cigar.empty()) throw Error(NPH_ERR_INVALID, std::string(who) + ": record " + rec.read_name + " has no CIGAR");
    if (rec.read && !rec.raw) throw Error(NPH_ERR_INVALID, std::string(who) + ": record " + rec.read_name + " has a read but no raw signal");
    return true;
}

// The arrays of one nph_polya_batch / nph_detect_polyi_batch call
struct PolyaInputs {
    std::vector<nph_polya_job> jobs;
    std::vector<float> raw, dur;
    std::vector<nph_event_range> b2e;
};

PolyaInputs pack(const std::vector<PolyaRecord>& records)
{
    const size_t n = records.size();
    PolyaInputs in;
    in.jobs.resize(n);
    size_t n_samples = 0, n_events = 0, n_ranks = 0;
    for (size_t i = 0; i < n; ++i) {
        const PolyaRecord& r = records[i];
        nph_polya_job& j = in.jobs[i];
        j = nph_polya_job{};
        j.suffix_clip = r.cigar.back() >> 4;                        // bam_cigar_oplen of the LAST operation (:755-758)
        // sr.fast5_path == "" || sr.events[0].empty() (:762): not loaded
        if (!r.read || r.read->events[0].empty()) continue;
        const SquiggleRead& sr = *r.read;
        j.loaded = 1;
        j.sample_off = n_samples; j.n_samples = (uint32_t)r.raw->samples.size();
        j.event_off = n_events;   j.n_events = (uint32_t)sr.events[0].size();
        j.rank_off = n_ranks;     j.n_kmers = (uint32_t)sr.base_to_event_map.size();
        j.sample_rate = r.raw->sample_rate;
        j.scale = sr.scalings[0].scale; j.shift = sr.scalings[0].shift; j.var = sr.scalings[0].var;
        n_samples += j.n_samples; n_events += j.n_events; n_ranks += j.n_kmers;
    }
    in.raw.resize(n_samples); in.dur.resize(n_events); in.b2e.resize(n_ranks);
    for (size_t i = 0; i < n; ++i) {
        const nph_polya_job& j = in.jobs[i];
        if (!j.loaded) continue;
        const SquiggleRead& sr = *records[i].read;
        std::copy(records[i].raw->samples.begin(), records[i].raw->samples.end(), in.raw.begin() + j.sample_off);
        for (uint32_t e = 0; e < j.n_events; ++e) in.dur[j.event_off + e] = sr.events[0][e].duration;
        for (uint32_t k = 0; k < j.n_kmers; ++k)
            in.b2e[j.rank_off + k] = nph_event_range{sr.base_to_event_map[k].indices[0].start, sr.base_to_event_map[k].indices[0].stop};
    }
    return in;
}

const char* const kQcTags[] = {"PASS", "NOREGION", "ADAPTER", "SUFFCLIP", "READ_FAILED_LOAD"};

// Appends one snprintf row to out, growing buf until it fits
template <class... Args>
void append_row(std::string& out, std::vector<char>& buf, const char* fmt, Args... args)
{
    for (;;) {
        const int len = snprintf(buf.data(), buf.size(), fmt, args...);
        if (len >= 0 && (size_t)len < buf.size()) { out.append(buf.data(), (size_t)len); return; }
        buf.resize(len >= 0 ? (size_t)len + 1 : buf.size() * 2);
    }
}

// The READ_FAILED_LOAD row, the same in both (:765-766; detect_polyi.cpp:1040-1041)
void append_failed_row(std::string& out, std::vector<char>& buf, const PolyaRecord& r)
{
    append_row(out, buf, "%s\t%s\t%d\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n", r.read_name.c_str(), r.contig.c_str(), r.pos);
}

} // namespace

bool PolyaBatch::add(const PolyaRecord& rec)
{
    if (!accept(rec, "nph::PolyaBatch::add")) return false;
    m_records.push_back(rec);
    return true;
}

void PolyaBatch::clear() { m_records.clear(); m_results.clear(); m_done.clear(); }

void PolyaBatch::run(Engine& engine)
{
    const size_t n = m_records.size();
    PolyaInputs in = pack(m_records);
    std::vector<nph_polya_result> res(n);
    engine.check(nph_polya_batch(engine.ctx(), in.raw.data(), in.raw.size(), in.jobs.data(), n, in.dur.data(), in.dur.size(), in.b2e.data(),
                                 in.b2e.size(), res.data()), "nph_polya_batch");
    m_results.swap(res);
    m_done.swap(m_records);
    m_records.clear();
}

std::string PolyaBatch::tsv(bool header) const
{
    std::string out;
    if (header)     // :877
        out += "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\tpolya_length\tqc_tag\n";
    std::vector<char> buf(256);
    for (size_t i = 0; i < m_done.size(); ++i) {
        const PolyaRecord& r = m_done[i];
        const nph_polya_result& s = m_results[i];
        if (s.qc == NPH_POLYA_READ_FAILED_LOAD)
            append_failed_row(out, buf, r);
        else                                           // :816-826, the indices + 1 in size_t
            append_row(out, buf, "%s\t%s\t%d\t%.1lf\t%.1lf\t%.1lf\t%.1lf\t%.2lf\t%.2lf\t%s\n",
                       r.read_name.c_str(), r.contig.c_str(), r.pos, (double)(uint64_t)(s.start + 1), (double)(uint64_t)(s.leader + 1),
                       (double)(uint64_t)(s.adapter + 1), (double)(uint64_t)(s.polya + 1), s.read_rate, s.polya_length, kQcTags[s.qc]);
    }
    return out;
}

bool DetectPolyiBatch::add(const PolyaRecord& rec)
{
    if (!accept(rec, "nph::DetectPolyiBatch::add")) return false;   // detect_polyi.cpp:1018-1020
    m_records.push_back(rec);
    return true;
}

void DetectPolyiBatch::clear() { m_records.clear(); m_results.clear(); m_done.clear(); }

void DetectPolyiBatch::run(Engine& engine)
{
    const size_t n = m_records.size();
    PolyaInputs in = pack(m_records);
    std::vector<nph_polyi_result> res(n);
    engine.check(nph_detect_polyi_batch(engine.ctx(), in.raw.data(), in.raw.size(), in.jobs.data(), n, in.dur.data(), in.dur.size(),
                                        in.b2e.data(), in.b2e.size(), res.data()), "nph_detect_polyi_batch");
    m_results.swap(res);
    m_done.swap(m_records);
    m_records.clear();
}

std::string DetectPolyiBatch::tsv(bool header) const
{
    static const char* const kDetected[] = {"NONE", "POLYA-ONLY", "POLYI-ONLY", "A+I"};
    std::string out;
    if (header)     // detect_polyi.cpp:1159
        out += "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\tpolya_length\tdetected\tqc_tag\n";
    std::vector<char> buf(256);
    for (size_t i = 0; i < m_done.size(); ++i) {
        const PolyaRecord& r = m_done[i];
        const nph_polyi_result& d = m_results[i];
        const nph_polya_result& s = d.seg;
        if (s.qc == NPH_POLYA_READ_FAILED_LOAD)
            append_failed_row(out, buf, r);
        else                                           // detect_polyi.cpp:1098-1108
            append_row(out, buf, "%s\t%s\t%d\t%.1lf\t%.1lf\t%.1lf\t%.1lf\t%.2lf\t%.2lf\t%s\t%s\n",
                       r.read_name.c_str(), r.contig.c_str(), r.pos, (double)(uint64_t)(s.start + 1), (double)(uint64_t)(s.leader + 1),
                       (double)(uint64_t)(s.adapter + 1), (double)(uint64_t)(s.polya + 1), s.read_rate, s.polya_length,
                       kDetected[d.detected], kQcTags[s.qc]);
    }
    return out;
}

} // namespace nph
