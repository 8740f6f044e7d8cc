// nph_phase_reads.cpp — see nph_phase_reads.hpp
#include "nph_phase_reads.hpp"
#include <algorithm>
#include <cstring>

namespace nph {

namespace {
// sortByPosition (ref: src/common/nanopolish_variant.h:106-111)
bool by_position(const Variant& a, const Variant& b)
{
    return a.ref_name == b.ref_name ? a.ref_position < b.ref_position : a.ref_name < b.ref_name;
}

const char kNt16[] = "=ACMGRSVTWYHKDBN";
// a base through the 4-bit code of the SAM/BAM specification and back: IUPAC codes and '=' keep their letter (upper-cased),
// the digits 0-3 read as A, C, G, T (the specification's table), every other byte becomes N
char nt16_round_trip(char c)
{
    if (c >= '0' && c <= '3') return "ACGT"[c - '0'];
    const char u = (char)std::toupper((unsigned char)c);
    const char* p = u ? std::strchr(kNt16, u) : nullptr;
    return p ? *p : 'N';
}
} // namespace

PhaseReads::PhaseReads(const std::vector<Variant>& sorted_variants) : m_variants(sorted_variants)
{
    m_dev_variants.resize(m_variants.size());
    for (size_t i = 0; i < m_variants.size(); ++i) {
        const Variant& v = m_variants[i];
        nph_phase_variant& d = m_dev_variants[i];
        std::memset(&d, 0, sizeof(d));
        d.ref_position = (int32_t)v.ref_position;
        d.ref_base = v.ref_seq.empty() ? 0 : v.ref_seq[0];
        d.alt_base = v.alt_seq.empty() ? 0 : v.alt_seq[0];
        d.is_snp = v.ref_seq.size() == 1 && v.alt_seq.size() == 1;           // Variant::is_snp
    }
}

void PhaseReads::clear()
{
    m_entries.clear(); m_ref.clear(); m_deltas.clear(); m_first_event.clear(); m_records.clear(); m_range.clear();
    m_call_off.clear(); m_calls.clear(); m_ran = false;
}

bool PhaseReads::add_read(const EventAlignedRead& r, uint16_t flag, uint8_t mapq)
{
    Variant lower, upper;
    lower.ref_name = upper.ref_name = r.contig;
    lower.ref_position = (size_t)r.ref_start_pos;
    upper.ref_position = (size_t)r.ref_start_pos + r.ref_seq.size() - 1;      // bam_endpos: faidx fetched [pos, bam_endpos]
    const auto lo = std::lower_bound(m_variants.begin(), m_variants.end(), lower, by_position);
    const auto hi = std::upper_bound(m_variants.begin(), m_variants.end(), upper, by_position);
    if (lo == m_variants.end()) return false;                                  // no variants to phase
    if (!r.read->has_events_for_strand(0)) return false;                       // only the template strand writes a record
    m_ran = false;
    nph_meth_record rec;
    std::memset(&rec, 0, sizeof(rec));
    rec.ref_off = m_ref.size(); rec.ref_len = (uint32_t)r.ref_seq.size(); rec.ref_start_pos = r.ref_start_pos; rec.rc = r.rc[0] ? 1 : 0;
    m_ref.insert(m_ref.end(), r.ref_seq.begin(), r.ref_seq.end());
    m_deltas.resize(m_ref.size());
    int32_t first = 0;
    if (!compact_event_alignment(r.aligned_events[0], r.ref_start_pos, r.ref_seq.size(), m_deltas.data() + rec.ref_off, &first))
        throw Error(NPH_ERR_UNSUPPORTED, "phase-reads: an event alignment outside the reference or with a step beyond int16");
    m_first_event.push_back(first);
    m_records.push_back(rec);
    const uint32_t a = (uint32_t)(lo - m_variants.begin()), b = (uint32_t)(hi - m_variants.begin());
    m_range.push_back(a);
    m_range.push_back(std::max(a, b));
    m_entries.push_back(Entry{r.read_name, r.contig, flag, mapq, r.read, r.read->get_base_model(0)});
    return true;
}

void PhaseReads::run(Engine& engine, double indel_bias)
{
    m_call_off.assign(m_records.size() + 1, 0);
    m_calls.clear();
    m_ran = true;
    if (m_records.empty()) return;
    detail::ReadTable reads;
    size_t cap = 0;
    for (size_t i = 0; i < m_records.size(); ++i) {
        m_records[i].read = reads.index(m_entries[i].read, 0);
        m_records[i].model_id = engine.model_id(m_entries[i].model);
        cap += m_range[2 * i + 1] - m_range[2 * i];
    }
    const detail::FlatReads fr = detail::flatten_reads(engine, reads);
    m_calls.resize(std::max<size_t>(cap, 1));
    uint64_t scored = 0;
    engine.check(nph_phase_reads_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events, m_ref.data(),
                                       m_deltas.data(), m_ref.size(), m_first_event.data(), m_records.data(), m_records.size(),
                                       m_dev_variants.data(), m_dev_variants.size(), m_range.data(), indel_bias, m_call_off.data(),
                                       m_calls.data(), cap, &scored),
                 "nph_phase_reads_batch");
    m_calls.resize((size_t)m_call_off.back());
}

std::vector<std::string> PhaseReads::sam() const
{
    if (!m_ran) throw Error(NPH_ERR_STATE, "PhaseReads::sam before run");
    std::vector<std::string> out(m_records.size());
    for (size_t i = 0; i < m_records.size(); ++i) {
        const nph_meth_record& R = m_records[i];
        const Entry& e = m_entries[i];
        std::string seq(m_ref.data() + R.ref_off, R.ref_len);
        std::string qual(R.ref_len, (char)30);                               // MAX_Q_SCORE + BAM_Q_OFFSET
        for (uint64_t c = m_call_off[i]; c < m_call_off[i + 1]; ++c) {       // list order: a later variant at one position wins
            const nph_phase_call& pc = m_calls[c];
            const size_t o = (size_t)(m_dev_variants[pc.variant].ref_position - R.ref_start_pos);
            seq[o] = pc.call;
            qual[o] = (char)pc.qual;
        }
        std::string& s = out[i];
        s = e.name + "\t" + std::to_string(e.flag) + "\t" + e.contig + "\t" + std::to_string(R.ref_start_pos + 1) + "\t" +
            std::to_string(e.mapq) + "\t" + std::to_string(R.ref_len) + "M\t*\t0\t0\t";
        for (char c : seq) s += nt16_round_trip(c);
        s += "\t";
        for (char q : qual) s += (char)(q + 33);
        s += "\n";
    }
    return out;
}

} // namespace nph
