// nph_polya.cpp — see nph_polya.hpp
#include "nph_polya.hpp"

#include <cstdio>

namespace nph {

bool PolyaBatch::add(const PolyaRecord& rec)
{
    if (rec.flag & BAM_FSECONDARY) return false;                     // :743-745
    if (rec.cigar.empty()) throw Error(NPH_ERR_INVALID, "nph::PolyaBatch::add: record " + rec.read_name + " has no CIGAR");
    if (rec.read && !rec.raw) throw Error(NPH_ERR_INVALID, "nph::PolyaBatch::add: record " + rec.read_name + " has a read but no raw signal");
    m_records.push_back(rec);
    return true;
}

void PolyaBatch::clear() { m_records.clear(); m_results.clear(); m_done.clear(); }

void PolyaBatch::run(Engine& engine)
{
    const size_t n = m_records.size();
    std::vector<nph_polya_job> jobs(n);
    size_t n_samples = 0, n_events = 0, n_ranks = 0;
    for (size_t i = 0; i < n; ++i) {
        const PolyaRecord& r = m_records[i];
        nph_polya_job& j = jobs[i];
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
    std::vector<float> raw(n_samples), dur(n_events);
    std::vector<nph_event_range> b2e(n_ranks);
    for (size_t i = 0; i < n; ++i) {
        const nph_polya_job& j = jobs[i];
        if (!j.loaded) continue;
        const SquiggleRead& sr = *m_records[i].read;
        std::copy(m_records[i].raw->samples.begin(), m_records[i].raw->samples.end(), raw.begin() + j.sample_off);
        for (uint32_t e = 0; e < j.n_events; ++e) dur[j.event_off + e] = sr.events[0][e].duration;
        for (uint32_t k = 0; k < j.n_kmers; ++k)
            b2e[j.rank_off + k] = nph_event_range{sr.base_to_event_map[k].indices[0].start, sr.base_to_event_map[k].indices[0].stop};
    }
    std::vector<nph_polya_result> res(n);
    engine.check(nph_polya_batch(engine.ctx(), raw.data(), raw.size(), jobs.data(), n, dur.data(), dur.size(), b2e.data(), b2e.size(),
                                 res.data()), "nph_polya_batch");
    m_results.swap(res);
    m_done.swap(m_records);
    m_records.clear();
}

std::string PolyaBatch::tsv(bool header) const
{
    static const char* const kTags[] = {"PASS", "NOREGION", "ADAPTER", "SUFFCLIP", "READ_FAILED_LOAD"};
    std::string out;
    if (header)     // :877
        out += "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\tpolya_length\tqc_tag\n";
    std::vector<char> buf(256);
    for (size_t i = 0; i < m_done.size(); ++i) {
        const PolyaRecord& r = m_done[i];
        const nph_polya_result& s = m_results[i];
        for (;;) {
            int len;
            if (s.qc == NPH_POLYA_READ_FAILED_LOAD)        // :765-766
                len = snprintf(buf.data(), buf.size(), "%s\t%s\t%d\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n",
                               r.read_name.c_str(), r.contig.c_str(), r.pos);
            else                                           // :816-826, the indices + 1 in size_t
                len = snprintf(buf.data(), buf.size(), "%s\t%s\t%d\t%.1lf\t%.1lf\t%.1lf\t%.1lf\t%.2lf\t%.2lf\t%s\n",
                               r.read_name.c_str(), r.contig.c_str(), r.pos, (double)(uint64_t)(s.start + 1), (double)(uint64_t)(s.leader + 1),
                               (double)(uint64_t)(s.adapter + 1), (double)(uint64_t)(s.polya + 1), s.read_rate, s.polya_length, kTags[s.qc]);
            if (len >= 0 && (size_t)len < buf.size()) { out.append(buf.data(), (size_t)len); break; }
            buf.resize(len >= 0 ? (size_t)len + 1 : buf.size() * 2);
        }
    }
    return out;
}

} // namespace nph
