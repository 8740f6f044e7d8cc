// nph_host.cpp — implementation of the C++ host mirror (see nph_host.hpp).
#include "nph_host.hpp"
#include "../csrc/tsv_format.cuh"
#ifdef _OPENMP
#include <omp.h>
#endif

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace nph {

double hmm_indel_bias_factor = 1.0;

// ---------------------------------------------------------------------------------------------
// Alphabet.  Behaviour follows src/common/nanopolish_alphabet.h:27-330 (match_to_site, reverse_complement,
// disambiguate, methylate, unmethylate, is_motif_match) and the tables of nanopolish_alphabet.cpp:15-194.
// ---------------------------------------------------------------------------------------------
Alphabet::Alphabet(const char* name, const char* bases, const char* complements,
                   std::vector<std::string> sites, std::vector<std::string> sites_methylated,
                   std::vector<std::string> sites_methylated_complement)
    : m_name(name), m_bases(bases), m_complement(complements), m_sites(std::move(sites)),
      m_sites_m(std::move(sites_methylated)), m_sites_mc(std::move(sites_methylated_complement))
{
    std::memset(m_rank, 0, sizeof(m_rank));          // unknown symbols rank 0, like the reference's tables
    for (size_t i = 0; i < m_bases.size(); ++i) m_rank[(unsigned char)m_bases[i]] = (uint8_t)i;
}

const Alphabet gDNAAlphabet("nucleotide", "ACGT", "TGCA", {}, {}, {});
const Alphabet gUtoTRNAAlphabet("u_to_t_rna", "ACGT", "TGCA", {}, {}, {});
const Alphabet gMCpGAlphabet("cpg", "ACGMT", "TGCGA", {"CG"}, {"MG"}, {"GM"});
const Alphabet gMethylGpCAlphabet("gpc", "ACGMT", "TGCGA", {"GC"}, {"GM"}, {"MG"});
const Alphabet gMethylDamAlphabet("dam", "ACGMT", "TGCTA", {"GATC"}, {"GMTC"}, {"CTMG"});
const Alphabet gMethylDcmAlphabet("dcm", "ACGMT", "TGCGA", {"CCAGG", "CCTGG"}, {"CMAGG", "CMTGG"}, {"GGTMC", "GGAMC"});

static const Alphabet* const kAlphabets[] = {&gDNAAlphabet, &gMCpGAlphabet, &gMethylGpCAlphabet,
                                             &gMethylDamAlphabet, &gMethylDcmAlphabet, &gUtoTRNAAlphabet};

const Alphabet* get_alphabet_by_name(const std::string& name)
{
    for (const Alphabet* a : kAlphabets)
        if (name == a->get_name()) return a;
    throw Error(NPH_ERR_INVALID, "unknown alphabet name: " + name);   // the reference exits here
}

const Alphabet* best_alphabet(const char* bases)
{
    for (const Alphabet* a : kAlphabets)
        if (a->contains_all(bases)) return a;
    return nullptr;
}

bool Alphabet::contains_all(const char* bases) const
{
    return std::strspn(bases, m_bases.c_str()) == std::strlen(bases);
}

void Alphabet::lexicographic_next(std::string& str) const
{
    int carry = 1;
    int i = (int)str.size() - 1;
    do {
        uint32_t r = rank(str[i]) + carry;
        str[i] = base((uint8_t)(r % size()));
        carry = (int)(r / size());
        i -= 1;
    } while (carry > 0 && i >= 0);
}

// Does a recognition site start at position i of str?  Two cases, as in the reference:
//  (1) i == 0 and the whole string is a substring of the site; (2) the suffix str[i..] starts with a
//  prefix of the site (a site cut off by the end of the string still matches).
Alphabet::Match Alphabet::match_to_site(const std::string& str, size_t i, const std::string& site) const
{
    Match m;
    const size_t rl = recognition_length();
    // case (1) needs the whole string inside the site: only strings no longer than the site can qualify, and only at i == 0
    const char* p = (i == 0 && str.length() <= site.length()) ? std::strstr(site.c_str(), str.c_str()) : nullptr;
    if (p != nullptr) {
        m.offset = (unsigned)(p - site.c_str());
        m.length = (unsigned)str.length();
    } else {
        size_t cl = std::min(rl, str.length() - i);
        if (str.compare(i, cl, site, 0, cl) == 0) {
            m.offset = 0;
            m.length = (unsigned)cl;
        }
    }
    if (m.length > 0)
        m.covers_methylated_site = std::memchr(str.data() + i, METHYLATED_SYMBOL, m.length) != nullptr;
    return m;
}

std::string Alphabet::reverse_complement(const std::string& str) const
{
    std::string out(str.length(), 'A');
    // a site is only treated as a unit when the match covers a methylated symbol: without one in the string this is the
    // plain base-by-base reverse complement
    if (std::memchr(str.data(), METHYLATED_SYMBOL, str.size()) == nullptr) {
        const size_t n = str.size();
        for (size_t t = 0; t < n; ++t) out[n - 1 - t] = complement(str[t]);
        return out;
    }
    size_t i = 0;
    int j = (int)str.length() - 1;
    while (i < str.length()) {
        int site = -1;
        Match m;
        // past position 0 a site can only match where its first symbol stands (match_to_site's case 2 compares from the
        // site's start); at position 0 a string lying inside a site also counts, so the matcher always runs there
        for (size_t s = 0; s < num_recognition_sites(); ++s) {
            if (i > 0 && str[i] != m_sites_m[s][0]) continue;
            m = match_to_site(str, i, m_sites_m[s]);
            if (m.length > 0 && m.covers_methylated_site) { site = (int)s; break; }
        }
        if (site != -1) {
            // a methylated site: emit the methylated complement of the matched part
            for (size_t t = m.offset; t < m.offset + m.length; ++t) {
                out[j--] = m_sites_mc[site][t];
                i += 1;
            }
        } else {
            out[j--] = complement(str[i++]);
        }
    }
    return out;
}

static char iupac_first(char c)
{
    switch (c) {
        case 'A': case 'M': case 'R': case 'W': case 'V': case 'H': case 'D': case 'N': return 'A';
        case 'C': case 'S': case 'Y': case 'B': return 'C';
        case 'G': case 'K': return 'G';
        case 'T': return 'T';
    }
    throw Error(NPH_ERR_INVALID, std::string("invalid IUPAC symbol: ") + c);   // the reference asserts
}

std::string Alphabet::disambiguate(const std::string& str) const
{
    std::string out(str);
    std::transform(out.begin(), out.end(), out.begin(), [](unsigned char c) { return (char)std::toupper(c); });
    size_t i = 0;
    while (i < out.length()) {
        size_t stride = 1;
        bool is_site = false;
        for (size_t s = 0; s < num_recognition_sites(); ++s) {
            Match m = match_to_site(out, i, m_sites_m[s]);
            if (m.length > 0) { stride = m.length; is_site = true; break; }
        }
        if (!is_site) { out[i] = iupac_first(out[i]); stride = 1; }
        i += stride;
    }
    return out;
}

std::string Alphabet::methylate(const std::string& str) const
{
    std::string out(str);
    size_t i = 0;
    while (i < out.length()) {
        size_t stride = 1;
        for (size_t s = 0; s < num_recognition_sites(); ++s) {
            if (i > 0 && str[i] != m_sites[s][0]) continue;          // see reverse_complement
            Match m = match_to_site(str, i, m_sites[s]);
            if (m.length == recognition_length()) {     // only complete sites are methylated
                out.replace(i, recognition_length(), m_sites_m[s]);
                stride = m.length;
                break;
            }
        }
        i += stride;
    }
    return out;
}

std::string Alphabet::unmethylate(const std::string& str) const
{
    std::string out(str);
    size_t i = 0;
    while (i < out.length()) {
        size_t stride = 1;
        for (size_t s = 0; s < num_recognition_sites(); ++s) {
            if (i > 0 && str[i] != m_sites_m[s][0]) continue;        // see reverse_complement
            Match m = match_to_site(str, i, m_sites_m[s]);
            if (m.length > 0) {
                out.replace(i, m.length, m_sites[s].c_str() + m.offset, m.length);
                stride = m.length;
                break;
            }
        }
        i += stride;
    }
    return out;
}

bool Alphabet::is_motif_match(const std::string& str, size_t i) const
{
    // a complete site needs recognition_length() symbols from i on; the partial matches match_to_site also reports
    // (string end, string inside a site) never have that length unless the whole string is the site, which the
    // comparison below covers too
    const size_t rl = recognition_length();
    if (rl > 0 && str.size() >= rl) {
        if (i + rl > str.size()) return false;
        for (size_t s = 0; s < num_recognition_sites(); ++s)
            if (std::memcmp(str.data() + i, m_sites[s].data(), rl) == 0) return true;
        return false;
    }
    for (size_t s = 0; s < num_recognition_sites(); ++s) {
        if (i > 0 && str[i] != m_sites[s][0]) continue;              // see reverse_complement
        Match m = match_to_site(str, i, m_sites[s]);
        if (m.length == recognition_length()) return true;
    }
    return false;
}

// ---------------------------------------------------------------------------------------------
// Engine
// ---------------------------------------------------------------------------------------------
void Engine::check(int status, const char* what) const
{
    if (status != NPH_OK)
        throw Error(status, std::string(what) + ": " + nph_strerror(status) + (m_ctx ? std::string(" / ") + nph_last_error(m_ctx) : ""));
}

Engine::Engine(int device)
{
    int rc = nph_create(&m_ctx, device);
    if (rc != NPH_OK) { m_ctx = nullptr; check(rc, "nph_create"); }
}

Engine::~Engine()
{
    for (Pinned& b : m_pinned) if (b.p) nph_host_free(b.p);
    if (m_ctx) nph_destroy(m_ctx);
}

void* Engine::pinned(Staging use, size_t bytes)
{
    Pinned& b = m_pinned[(int)use];
    if (b.bytes < bytes) {
        if (b.p) nph_host_free(b.p);
        b.p = nullptr; b.bytes = 0;
        const size_t want = bytes + bytes / 4;
        check(nph_host_alloc(&b.p, want), "nph_host_alloc");
        b.bytes = want;
    }
    return b.p;
}

Engine& Engine::thread_default()
{
    thread_local std::unique_ptr<Engine> eng;
    if (!eng) {
        const char* d = std::getenv("NPH_DEVICE");
        eng.reset(new Engine(d ? std::atoi(d) : 0));
    }
    return *eng;
}

uint32_t Engine::model_id(const PoreModel* model)
{
    auto it = m_models.find(model);
    if (it != m_models.end()) return it->second;
    const size_t n = model->states.size();
    std::vector<double> mean(n), sd(n), lsd(n);
    for (size_t i = 0; i < n; ++i) {
        mean[i] = model->states[i].level_mean;
        sd[i] = model->states[i].level_stdv;
        lsd[i] = model->states[i].level_log_stdv;
    }
    uint32_t id = 0;
    check(nph_model_upload(m_ctx, mean.data(), sd.data(), lsd.data(), (uint32_t)n, model->k, model->pmalphabet->size(), &id),
          "nph_model_upload");
    m_models[model] = id;
    return id;
}

// ---------------------------------------------------------------------------------------------
// Batches
// ---------------------------------------------------------------------------------------------
// format_fixed: csrc/tsv_format.cuh's exact formatter where it takes the value and the precision, snprintf elsewhere
namespace {
template <int N, typename T>
size_t fixed_or_printf(char* dst, T v)
{
    const nph_tsv::Fixed f = nph_tsv::fixed_of<N>(v);
    if (!f.ok) return (size_t)snprintf(dst, 400, "%.*lf", N, (double)v);
    char* const o = nph_tsv::put_fixed<N>(dst, f);
    *o = 0;
    return (size_t)(o - dst);
}
} // namespace

size_t format_fixed(char* dst, float v, int prec)
{
    switch (prec) {
    case 0: return fixed_or_printf<0>(dst, v);
    case 1: return fixed_or_printf<1>(dst, v);
    case 2: return fixed_or_printf<2>(dst, v);
    case 3: return fixed_or_printf<3>(dst, v);
    case 4: return fixed_or_printf<4>(dst, v);
    case 5: return fixed_or_printf<5>(dst, v);
    }
    return (size_t)snprintf(dst, 64, "%.*lf", prec, (double)v);
}

size_t format_fixed(char* dst, double v, int prec)
{
    switch (prec) {
    case 0: return fixed_or_printf<0>(dst, v);
    case 1: return fixed_or_printf<1>(dst, v);
    case 2: return fixed_or_printf<2>(dst, v);
    case 3: return fixed_or_printf<3>(dst, v);
    }
    return (size_t)snprintf(dst, 400, "%.*lf", prec, v);
}

int host_threads()
{
    static const int n = [] {
        int t = 32;
#ifdef _OPENMP
        t = std::min(omp_get_max_threads(), 32);
#endif
        if (const char* e = std::getenv("NPH_HOST_THREADS")) { const int v = std::atoi(e); if (v > 0) t = v; }
        return std::max(1, t);
    }();
    return n;
}

namespace detail {
FlatReads flatten_reads(Engine& engine, const ReadTable& table)
{
    const std::vector<ReadTable::Key>& reads = table.reads();
    FlatReads fr;
    fr.reads.resize(reads.size());
    std::vector<size_t> offs(reads.size() + 1, 0);
    bool any_drift = false;
    for (size_t i = 0; i < reads.size(); ++i) {
        offs[i + 1] = offs[i] + reads[i].first->events[reads[i].second].size();
        any_drift = any_drift || reads[i].first->scalings[reads[i].second].drift != 0.0;
    }
    const size_t total = offs.back();
    fr.n_events = total;
    float* const mean = static_cast<float*>(engine.pinned(Engine::Staging::EventMeans, sizeof(float) * std::max<size_t>(total, 1)));
    double* const time = any_drift ? static_cast<double*>(engine.pinned(Engine::Staging::StartTimes, sizeof(double) * std::max<size_t>(total, 1)))
                                   : nullptr;
    fr.mean = mean;
    fr.time = time;
#pragma omp parallel for schedule(dynamic, 8) num_threads(host_threads()) if (total > (size_t)1 << 18)
    for (long long ii = 0; ii < (long long)reads.size(); ++ii) {
        const size_t i = (size_t)ii, off = offs[i];
        const SquiggleRead* sr = reads[i].first;
        const uint8_t st = reads[i].second;
        const std::vector<SquiggleEvent>& ev = sr->events[st];
        nph_read& o = fr.reads[i];
        o.event_off = off;
        o.n_events = (uint32_t)ev.size();
        o.reserved = 0;
        const SquiggleScalings& s = sr->scalings[st];
        o.scale = s.scale; o.shift = s.shift; o.drift = s.drift; o.var = s.var; o.log_var = s.log_var;
        o.events_per_base = sr->events_per_base[st];
        const std::vector<float>& cache = sr->event_mean_cache[st];
        if (cache.size() == ev.size() && !ev.empty()) std::memcpy(mean + off, cache.data(), sizeof(float) * ev.size());
        else for (size_t e = 0; e < ev.size(); ++e) mean[off + e] = ev[e].mean;
        if (time) for (size_t e = 0; e < ev.size(); ++e) time[off + e] = ev[e].start_time;
    }
    return fr;
}

nph_hmm_job make_hmm_job(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags, ReadTable& reads)
{
    if (!data.read || !data.pore_model) throw Error(NPH_ERR_INVALID, "HMMInputData without read or pore_model");
    if (data.read->pore_type != PORETYPE_R9) throw Error(NPH_ERR_UNSUPPORTED, "only R9 reads are supported (load_from_raw always makes R9)");
    const uint32_t k = data.pore_model->k;
    if (data.pore_model->states.size() != sequence.get_num_kmer_ranks(k))
        throw Error(NPH_ERR_INVALID, "sequence alphabet does not match the pore model's state space");   // ref asserts (profile_hmm_r9.inl:305)
    if (!((data.rc && data.event_stride == -1) || (!data.rc && data.event_stride == 1)))
        throw Error(NPH_ERR_INVALID, "rc and event_stride disagree");                                       // ref asserts (profile_hmm_r9.inl:275)
    if (sequence.length() < k) throw Error(NPH_ERR_INVALID, "sequence shorter than k");
    nph_hmm_job j;
    j.rank_off = 0;
    j.read = reads.index(data.read, data.strand);
    j.model_id = 0;
    j.event_start = data.event_start_idx;
    j.event_stop = data.event_stop_idx;
    j.n_kmers = (uint32_t)(sequence.length() - k + 1);
    j.stride = data.event_stride;
    j.rc = data.rc;
    j.flags = (uint8_t)flags;
    j.reserved = 0;
    return j;
}

void resolve_model_ids(Engine& engine, const std::vector<const PoreModel*>& models, std::vector<nph_hmm_job>& jobs)
{
    const PoreModel* last_model = nullptr;
    uint32_t last_id = 0;
    for (size_t j = 0; j < jobs.size(); ++j) {
        if (models[j] != last_model) { last_model = models[j]; last_id = engine.model_id(last_model); }
        jobs[j].model_id = last_id;
    }
}
} // namespace detail
using detail::flatten_reads;

size_t HmmBatch::add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags)
{
    RankCache once;
    return add(sequence, data, flags, once);
}

size_t HmmBatch::add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags, RankCache& cache)
{
    nph_hmm_job j = detail::make_hmm_job(sequence, data, flags, m_reads);
    const uint32_t k = data.pore_model->k;
    const int strand_slot = data.rc != 0 ? 1 : 0;
    if (cache.k != k) { cache.off[0] = cache.off[1] = ~(uint64_t)0; cache.k = k; }
    if (cache.off[strand_slot] == ~(uint64_t)0) {
        cache.off[strand_slot] = m_codes.size();
        sequence.append_codes(data.rc != 0, m_codes);
    }
    j.rank_off = cache.off[strand_slot];
    m_jobs.push_back(j);
    m_job_models.push_back(data.pore_model);
    return m_jobs.size() - 1;
}

// rank(i + 1) = (rank(i) mod A^(k-1)) * A + rank(s[i + k])
void kmer_ranks(const Alphabet& alphabet, const char* s, size_t len, uint32_t k, bool reversed, uint32_t* out)
{
    if (len < k) return;
    const size_t n = len - k + 1;
    const uint64_t A = alphabet.size();
    uint64_t top = 1;
    for (uint32_t i = 1; i < k; ++i) top *= A;
    uint64_t r = 0;
    for (uint32_t i = 0; i < k; ++i) r = r * A + alphabet.rank(s[i]);
    for (size_t pos = 0;; ++pos) {
        out[reversed ? n - 1 - pos : pos] = (uint32_t)r;
        if (pos + 1 == n) break;
        r = (r % top) * A + alphabet.rank(s[pos + k]);
    }
}

// with do_rc the i-th rank is that of the rc string's k-mer at length - i - k: the rc string's ranks back to front
void HMMInputSequence::append_kmer_ranks(uint32_t k, bool do_rc, std::vector<uint32_t>& out) const
{
    const std::string& s = do_rc ? m_rc_seq : m_seq;
    if (s.size() < k) return;
    const size_t base = out.size();
    out.resize(base + s.size() - k + 1);
    kmer_ranks(*m_alphabet, s.data(), s.size(), k, do_rc, out.data() + base);
}

void HMMInputSequence::append_codes(bool do_rc, std::vector<uint8_t>& out) const
{
    const std::string& s = do_rc ? m_rc_seq : m_seq;
    const size_t base = out.size();
    out.resize(base + s.size());
    for (size_t i = 0; i < s.size(); ++i) out[base + i] = m_alphabet->rank(s[i]);
}

std::vector<uint32_t> HmmBatch::ranks() const
{
    std::vector<uint32_t> out(m_codes.size(), 0);
    for (size_t j = 0; j < m_jobs.size(); ++j) {
        const nph_hmm_job& jb = m_jobs[j];
        const uint32_t k = m_job_models[j]->k, A = m_job_models[j]->pmalphabet->size();
        const uint8_t* cd = m_codes.data() + jb.rank_off;
        for (uint32_t i = 0; i < jb.n_kmers; ++i) {
            const uint8_t* km = cd + (jb.rc ? jb.n_kmers - 1 - i : i);
            uint32_t r = 0;
            for (uint32_t t = 0; t < k; ++t) r = r * A + km[t];
            out[jb.rank_off + i] = r;
        }
    }
    return out;
}

void HmmBatch::clear()
{
    m_reads.clear(); m_job_models.clear(); m_jobs.clear(); m_codes.clear();
}

std::vector<float> HmmBatch::run(Engine& engine, double indel_bias)
{
    std::vector<float> scores(m_jobs.size());
    if (m_jobs.empty()) return scores;
    detail::resolve_model_ids(engine, m_job_models, m_jobs);
    const detail::FlatReads fr = flatten_reads(engine, m_reads);
    engine.check(nph_hmm_score_batch_seq(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events,
                                         m_codes.data(), m_codes.size(), m_jobs.data(), m_jobs.size(), indel_bias, scores.data()),
                 "nph_hmm_score_batch_seq");
    return scores;
}

std::vector<float> HmmBatch::run_training(Engine& engine, const std::vector<uint8_t>& groups, nph_tt_params& params, nph_transition_counts* counts,
                                          double indel_bias)
{
    if (!groups.empty() && groups.size() != m_jobs.size()) throw Error(NPH_ERR_INVALID, "one group per job");
    std::vector<float> scores(m_jobs.size());
    if (m_jobs.empty()) {
        engine.check(nph_train_transitions_batch(engine.ctx(), nullptr, 0, nullptr, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, &params, indel_bias,
                                                 nullptr, counts), "nph_train_transitions_batch");
        return scores;
    }
    detail::resolve_model_ids(engine, m_job_models, m_jobs);
    const detail::FlatReads fr = flatten_reads(engine, m_reads);
    engine.check(nph_train_transitions_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events, m_codes.data(),
                                             m_codes.size(), m_jobs.data(), m_jobs.size(), groups.empty() ? nullptr : groups.data(), &params,
                                             indel_bias, scores.data(), counts),
                 "nph_train_transitions_batch");
    return scores;
}

size_t AbeaBatch::add(SquiggleRead& read, const PoreModel& pore_model, const std::string& sequence)
{
    if (m_model && m_model != &pore_model) throw Error(NPH_ERR_INVALID, "one pore model per AbeaBatch");
    m_model = &pore_model;
    const uint32_t k = pore_model.k;
    if (sequence.size() < k || read.events[0].empty()) throw Error(NPH_ERR_INVALID, "empty read or sequence shorter than k");
    const uint32_t n_kmers = (uint32_t)(sequence.size() - k + 1);
    nph_abea_job j;
    j.rank_off = m_ranks.size();
    j.pairs_off = m_pairs_total;
    j.read = m_reads.index(&read, 0);                  // strand 0, like the reference (raw_loader.cpp:79)
    j.n_kmers = n_kmers;
    j.pairs_cap = (uint32_t)read.events[0].size() + n_kmers;
    j.reserved = 0;
    m_ranks.resize(j.rank_off + n_kmers);
    kmer_ranks(*pore_model.pmalphabet, sequence.data(), sequence.size(), k, false, m_ranks.data() + j.rank_off);
    m_pairs_total += j.pairs_cap;
    m_jobs.push_back(j);
    return m_jobs.size() - 1;
}

void AbeaBatch::clear()
{
    m_reads.clear(); m_jobs.clear(); m_ranks.clear(); m_pairs_total = 0; m_model = nullptr;
}

std::vector<std::vector<AlignedPair>> AbeaBatch::run(Engine& engine)
{
    std::vector<std::vector<AlignedPair>> out(m_jobs.size());
    if (m_jobs.empty()) return out;
    const detail::FlatReads fr = flatten_reads(engine, m_reads);
    std::vector<nph_aligned_pair> pairs(m_pairs_total);
    std::vector<nph_abea_result> res(m_jobs.size());
    engine.check(nph_abea_batch(engine.ctx(), fr.reads.data(), fr.reads.size(), fr.mean, fr.time, fr.n_events,
                                m_ranks.data(), m_ranks.size(), m_jobs.data(), m_jobs.size(), engine.model_id(m_model),
                                pairs.data(), pairs.size(), res.data()),
                 "nph_abea_batch");
    for (size_t j = 0; j < m_jobs.size(); ++j) {
        out[j].resize(res[j].n_pairs);     // 0 == the reference's empty vector (failed QC)
        for (uint32_t i = 0; i < res[j].n_pairs; ++i) {
            const nph_aligned_pair& p = pairs[m_jobs[j].pairs_off + i];
            out[j][i] = AlignedPair{p.ref_pos, p.read_pos};
        }
    }
    return out;
}

// ---------------------------------------------------------------------------------------------
// The reference's free functions
// ---------------------------------------------------------------------------------------------
float profile_hmm_score(const HMMInputSequence& sequence, const HMMInputData& data, const uint32_t flags)
{
    HmmBatch b;
    b.add(sequence, data, flags);
    return b.run(Engine::thread_default())[0];
}

float profile_hmm_score(const HMMInputSequence& sequence, const std::vector<HMMInputData>& data, const uint32_t flags)
{
    HmmBatch b;
    for (const HMMInputData& d : data) b.add(sequence, d, flags);
    std::vector<float> s = b.run(Engine::thread_default());
    float score = 0.0f;
    for (float v : s) score += v;        // float sum in input order, like the reference's loop
    return score;
}

float profile_hmm_score_set(const std::vector<HMMInputSequence>& sequences, const HMMInputData& data, const uint32_t flags)
{
    if (sequences.empty()) throw Error(NPH_ERR_INVALID, "profile_hmm_score_set: no sequences");
    HmmBatch b;
    b.add(sequences[0], data, flags);
    for (size_t i = 1; i < sequences.size(); ++i) {
        HMMInputData alt = data;
        const std::string name = sequences[i].get_alphabet()->get_name();
        auto it = data.read->alt_models[data.strand].find(name);
        if (it == data.read->alt_models[data.strand].end())
            throw Error(NPH_ERR_INVALID, "read has no pore model for alphabet " + name);   // the reference asserts alt model != NULL
        alt.pore_model = it->second;
        b.add(sequences[i], alt, flags);
    }
    std::vector<float> s = b.run(Engine::thread_default());
    float out = 0.0f;
    Engine::thread_default().check(nph_score_set_combine(s.data(), 1, (uint32_t)s.size(), &out), "nph_score_set_combine");
    return out;
}

std::vector<AlignedPair> adaptive_banded_simple_event_align(SquiggleRead& read, const PoreModel& pore_model, const std::string& sequence)
{
    AbeaBatch b;
    b.add(read, pore_model, sequence);
    return b.run(Engine::thread_default())[0];
}

SquiggleScalings estimate_scalings_using_mom(const std::string& sequence, const PoreModel& pore_model, const std::vector<float>& event_means)
{
    Engine& eng = Engine::thread_default();
    const uint32_t k = pore_model.k;
    if (sequence.size() < k || event_means.empty()) throw Error(NPH_ERR_INVALID, "empty events or sequence shorter than k");
    const uint32_t n_kmers = (uint32_t)(sequence.size() - k + 1);
    std::vector<uint32_t> ranks(n_kmers);
    kmer_ranks(*pore_model.pmalphabet, sequence.data(), sequence.size(), k, false, ranks.data());
    nph_read r{};
    r.event_off = 0; r.n_events = (uint32_t)event_means.size(); r.scale = 1.0; r.var = 1.0;
    nph_abea_job j{};
    j.rank_off = 0; j.pairs_off = 0; j.read = 0; j.n_kmers = n_kmers; j.pairs_cap = 0;
    double ss[2] = {0, 1};
    eng.check(nph_mom_batch(eng.ctx(), &r, 1, event_means.data(), event_means.size(), ranks.data(), ranks.size(), &j, 1,
                            eng.model_id(&pore_model), ss),
              "nph_mom_batch");
    SquiggleScalings out;
    out.set4(ss[0], ss[1], 0.0, 1.0);
    return out;
}

} // namespace nph
