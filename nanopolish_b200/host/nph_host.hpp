// nph_host.hpp — C++ host side above the C ABI (include/nph.h).
//
// Mirrors the reference's call surface for the hot path — same type names, members, argument meaning
// and soft-failure behaviour — so a nanopolish caller can switch by changing includes/namespaces:
//
//   HMMInputData, HMMAlignmentFlags         ref: src/common/nanopolish_common.h:53-62, src/hmm/nanopolish_profile_hmm.h:34-38
//   HMMInputSequence                        ref: src/hmm/nanopolish_hmm_input_sequence.h:20-98
//   SquiggleRead / SquiggleEvent / SquiggleScalings   ref: src/nanopolish_squiggle_read.h:53-93, 103-299
//   PoreModel / PoreModelStateParams        ref: src/pore_model/nanopolish_poremodel.h:20-110
//   Alphabet (+ nucleotide, u_to_t_rna, cpg, gpc, dam, dcm)   ref: src/common/nanopolish_alphabet.{h,cpp}
//   profile_hmm_score / profile_hmm_score_set          ref: src/hmm/nanopolish_profile_hmm.h:24-31
//   adaptive_banded_simple_event_align / estimate_scalings_using_mom   ref: src/nanopolish_raw_loader.h:16-24
//
// The free functions score a batch of one through a per-thread engine (drop-in, slow: one launch per
// call).  Real callers collect a BamProcessor batch worth of jobs in HmmBatch / AbeaBatch and run
// them with one launch; that is the intended integration (INTEGRATION.md).
//
// Nothing here computes a score on the CPU: every result comes from libnph.so, and a missing GPU
// surfaces as nph::Error.
#pragma once
#include <cmath>
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/nph.h"

namespace nph {

struct Error : std::runtime_error {
    int status;
    Error(int s, const std::string& what) : std::runtime_error(what), status(s) {}
};

// ---------------------------------------------------------------------------------------------
// Alphabets
// ---------------------------------------------------------------------------------------------
constexpr char METHYLATED_SYMBOL = 'M';

class Alphabet {
public:
    Alphabet(const char* name, const char* bases, const char* complements,
             std::vector<std::string> sites, std::vector<std::string> sites_methylated,
             std::vector<std::string> sites_methylated_complement);

    uint8_t rank(char b) const { return m_rank[(unsigned char)b]; }
    char base(uint8_t r) const { return m_bases[r]; }
    char complement(char b) const { return m_complement[rank(b)]; }
    uint32_t size() const { return (uint32_t)m_bases.size(); }
    const char* get_name() const { return m_name.c_str(); }

    size_t num_recognition_sites() const { return m_sites.size(); }
    size_t recognition_length() const { return m_sites.empty() ? 0 : m_sites[0].size(); }
    const char* get_recognition_site(size_t i) const { return m_sites[i].c_str(); }
    const char* get_recognition_site_methylated(size_t i) const { return m_sites_m[i].c_str(); }
    const char* get_recognition_site_methylated_complement(size_t i) const { return m_sites_mc[i].c_str(); }

    // lexicographic rank of str[0..k) among all k-mers of this alphabet
    uint32_t kmer_rank(const char* str, uint32_t k) const
    {
        uint32_t r = 0;
        for (uint32_t i = 0; i < k; ++i) r = r * size() + rank(str[i]);
        return r;
    }
    void lexicographic_next(std::string& str) const;
    size_t get_num_strings(size_t l) const { size_t n = 1; for (size_t i = 0; i < l; ++i) n *= size(); return n; }

    std::string reverse_complement(const std::string& str) const;
    std::string disambiguate(const std::string& str) const;
    std::string methylate(const std::string& str) const;
    std::string unmethylate(const std::string& str) const;
    bool contains_all(const char* bases) const;
    bool is_motif_match(const std::string& str, size_t i) const;

private:
    struct Match { unsigned offset = 0, length = 0; bool covers_methylated_site = false; };
    Match match_to_site(const std::string& str, size_t i, const std::string& site) const;

    std::string m_name, m_bases, m_complement;
    uint8_t m_rank[256];
    std::vector<std::string> m_sites, m_sites_m, m_sites_mc;
};

extern const Alphabet gDNAAlphabet, gMCpGAlphabet, gMethylGpCAlphabet, gMethylDamAlphabet, gMethylDcmAlphabet, gUtoTRNAAlphabet;
const Alphabet* get_alphabet_by_name(const std::string& name);   // throws nph::Error for an unknown name
const Alphabet* best_alphabet(const char* bases);

// out[i] = alphabet.kmer_rank(s + i, k) for the n = len - k + 1 k-mers of s (nothing when len < k), in one rolling pass;
// reversed stores them back to front, out[n - 1 - i]
void kmer_ranks(const Alphabet& alphabet, const char* s, size_t len, uint32_t k, bool reversed, uint32_t* out);

// ---------------------------------------------------------------------------------------------
// Pore model
// ---------------------------------------------------------------------------------------------
struct PoreModelStateParams {
    double level_mean = 0, level_stdv = 1, sd_mean = 0, sd_stdv = 0;
    double level_log_stdv = 0, sd_lambda = 0, sd_log_lambda = 0;
    PoreModelStateParams() {}
    PoreModelStateParams(double lm, double ls, double sm, double ss) : level_mean(lm), level_stdv(ls), sd_mean(sm), sd_stdv(ss)
    {
        sd_lambda = std::pow(sd_mean, 3.0) / std::pow(sd_stdv, 2.0);
        level_log_stdv = std::log(level_stdv);
        sd_log_lambda = std::log(sd_lambda);
    }
};

class PoreModel {
public:
    explicit PoreModel(uint32_t _k = 5) : k(_k), pmalphabet(&gDNAAlphabet) {}
    PoreModelStateParams get_parameters(uint32_t kmer_rank) const { return states[kmer_rank]; }
    size_t get_num_states() const { return states.size(); }

    std::string name, type;
    uint32_t k;
    const Alphabet* pmalphabet;
    std::vector<PoreModelStateParams> states;
};

// ---------------------------------------------------------------------------------------------
// SquiggleRead: the data-model part the hot path reads
// ---------------------------------------------------------------------------------------------
struct SquiggleEvent {
    float mean;
    float stdv;
    double start_time;
    float duration;
    float log_stdv;
};

struct SquiggleScalings {
    SquiggleScalings() : scale(1.0), shift(0.0), drift(0.0), var(1.0), scale_sd(1.0), var_sd(1.0) { set6(0.0, 1.0, 0.0, 1.0, 1.0, 1.0); }
    void set4(double _shift, double _scale, double _drift, double _var) { set6(_shift, _scale, _drift, _var, 1.0, 1.0); }
    void set6(double _shift, double _scale, double _drift, double _var, double _scale_sd, double _var_sd)
    {
        shift = _shift; scale = _scale; drift = _drift; var = _var; scale_sd = _scale_sd; var_sd = _var_sd;
        log_var = std::log(var);
        scaled_var = var / scale;
        log_scaled_var = std::log(scaled_var);
    }
    double scale, shift, drift, var, scale_sd, var_sd;
    double log_var, scaled_var, log_scaled_var;
};

struct GaussianParameters {
    float mean = 0.0f, stdv = 1.0f, log_stdv = 0.0f;
};

enum PoreType { PORETYPE_R7 = 0, PORETYPE_R9 = 1 };
enum SquiggleReadNucleotideType { SRNT_DNA = 0, SRNT_RNA = 1 };     // ref: src/nanopolish_squiggle_read.h:38-43

// ref: src/nanopolish_squiggle_read.h:32-46
struct IndexPair {
    int32_t start = -1, stop = -1;      // inclusive
    IndexPair() {}
    IndexPair(int32_t a, int32_t b) : start(a), stop(b) {}
};
struct EventRangeForBase { IndexPair indices[2]; };

class SquiggleRead {
public:
    SquiggleRead() { base_model[0] = base_model[1] = nullptr; events_per_base[0] = events_per_base[1] = 0.0; }

    float get_unscaled_level(uint32_t event_idx, uint32_t strand) const { return events[strand][event_idx].mean; }
    float get_time(uint32_t event_idx, uint32_t strand) const
    {
        return (float)(events[strand][event_idx].start_time - events[strand][0].start_time);
    }
    // same mixed-precision expression as the reference (float - float*double, narrowed)
    float get_drift_scaled_level(uint32_t event_idx, uint32_t strand) const
    {
        float level = get_unscaled_level(event_idx, strand);
        float time = get_time(event_idx, strand);
        return (float)(level - time * scalings[strand].drift);
    }
    GaussianParameters get_scaled_gaussian_from_pore_model_state(const PoreModel& pore_model, size_t strand_idx, size_t rank) const
    {
        const SquiggleScalings& s = scalings[strand_idx];
        const PoreModelStateParams& p = pore_model.states[rank];
        GaussianParameters gp;
        gp.mean = (float)(s.scale * p.level_mean + s.shift);
        gp.stdv = (float)(p.level_stdv * s.var);
        gp.log_stdv = (float)(p.level_log_stdv + s.log_var);
        return gp;
    }
    float get_fully_scaled_level(uint32_t event_idx, uint32_t strand) const
    {
        return (float)((get_drift_scaled_level(event_idx, strand) - scalings[strand].shift) / scalings[strand].scale);
    }
    float get_stdv(uint32_t event_idx, uint32_t strand) const { return events[strand][event_idx].stdv; }
    float get_duration(uint32_t event_idx, uint32_t strand) const { return events[strand][event_idx].duration; }
    // ref: src/nanopolish_squiggle_read.h:229-233
    int32_t flip_k_strand(int32_t k_idx, uint32_t k) const { return (int32_t)read_sequence.size() - k_idx - (int32_t)k; }
    // index of the event nearest to a k-mer of the basecalled sequence: the first event of the closest k-mer that has
    // one, looking backwards first, at most 1000 k-mers either way (-1 if none).
    // ref: src/nanopolish_squiggle_read.cpp:160-186
    int get_next_event(int start, int stop, int stride, uint32_t strand) const
    {
        for (; start != stop; start += stride) {
            const int ei = base_to_event_map[start].indices[strand].start;
            if (ei != -1) return ei;
        }
        return -1;
    }
    int get_closest_event_to(int k_idx, uint32_t strand) const
    {
        const int stop_before = k_idx - 1000 > 0 ? k_idx - 1000 : 0;
        const int last = (int)base_to_event_map.size() - 1;
        const int stop_after = k_idx + 1000 < last ? k_idx + 1000 : last;
        const int event_before = get_next_event(k_idx, stop_before, -1, strand);
        const int event_after = get_next_event(k_idx, stop_after, 1, strand);
        return event_before == -1 ? event_after : event_before;
    }
    // ref: src/nanopolish_squiggle_read.cpp:393-428
    size_t get_sample_index_at_time(size_t sample_time) const { return sample_time - sample_start_time; }
    std::pair<size_t, size_t> get_event_sample_idx(size_t strand_idx, size_t event_idx) const
    {
        const double event_start_time = events[strand_idx][event_idx].start_time;
        const double event_duration = events[strand_idx][event_idx].duration;
        const size_t start_idx = get_sample_index_at_time((size_t)(event_start_time * sample_rate));
        const size_t end_idx = get_sample_index_at_time((size_t)((event_start_time + event_duration) * sample_rate));
        return std::make_pair(start_idx, end_idx);
    }
    std::vector<float> get_scaled_samples_for_event(size_t strand_idx, size_t event_idx) const
    {
        const std::pair<size_t, size_t> sample_range = get_event_sample_idx(strand_idx, event_idx);
        std::vector<float> out;
        for (size_t i = sample_range.first; i < sample_range.second; ++i) {
            const double curr_sample_time = (sample_start_time + i) / sample_rate;
            const double s = samples.at(i);
            double scaled_s = s - scalings[strand_idx].shift;
            scaled_s -= (curr_sample_time - (sample_start_time / sample_rate)) * scalings[strand_idx].drift;
            scaled_s /= scalings[strand_idx].scale;
            out.push_back((float)scaled_s);
        }
        return out;
    }
    bool has_events_for_strand(size_t strand_idx) const { return !events[strand_idx].empty(); }
    size_t get_model_k(uint32_t strand) const { return base_model[strand]->k; }
    const PoreModel* get_base_model(uint32_t strand) const { return base_model[strand]; }
    // The reference resolves alternative-alphabet models through the PoreModelSet singleton
    // (squiggle_read.h:194-200); here the caller registers them on the read.
    const PoreModel* get_model(uint32_t strand, const std::string& alphabet) const
    {
        if (base_model[strand] && alphabet == base_model[strand]->pmalphabet->get_name()) return base_model[strand];
        auto it = alt_models[strand].find(alphabet);
        return it == alt_models[strand].end() ? nullptr : it->second;
    }

    std::string read_name;
    PoreType pore_type = PORETYPE_R9;
    SquiggleReadNucleotideType nucleotide_type = SRNT_DNA;
    uint32_t read_id = 0;
    std::string read_sequence;
    std::vector<SquiggleEvent> events[2];
    // contiguous copy of events[strand][*].mean (what the device consumes), so that batching a read is one memcpy instead of a
    // strided gather over 24-byte SquiggleEvents; valid while its size equals events[strand].size() — nph::load_from_raw fills it,
    // cache_event_means() refreshes it, code that edits event means afterwards must call it again (or clear the cache)
    std::vector<float> event_mean_cache[2];
    void cache_event_means()
    {
        for (int st = 0; st < 2; ++st) {
            event_mean_cache[st].resize(events[st].size());
            for (size_t i = 0; i < events[st].size(); ++i) event_mean_cache[st][i] = events[st][i].mean;
        }
    }
    SquiggleScalings scalings[2];
    const PoreModel* base_model[2];
    std::map<std::string, const PoreModel*> alt_models[2];   // alphabet name -> model (cpg, dam, ...)
    double events_per_base[2];
    std::vector<EventRangeForBase> base_to_event_map;       // filled by nph::load_from_raw (nph_raw.hpp)
    double sample_rate = 0.0;
    uint64_t sample_start_time = 0;                          // 0 once the raw samples are kept (squiggle_read.cpp:252)
    std::vector<float> samples;                              // the trimmed raw samples, kept on request (SRF_LOAD_RAW_SAMPLES)
};

// ---------------------------------------------------------------------------------------------
// HMM inputs
// ---------------------------------------------------------------------------------------------
struct HMMInputData {
    SquiggleRead* read = nullptr;
    const PoreModel* pore_model = nullptr;
    uint32_t event_start_idx = 0;
    uint32_t event_stop_idx = 0;
    uint8_t strand = 0;
    int8_t event_stride = 1;
    uint8_t rc = 0;
};

enum HMMAlignmentFlags { HAF_ALLOW_PRE_CLIP = 1, HAF_ALLOW_POST_CLIP = 2 };

class HMMInputSequence {
public:
    HMMInputSequence(const std::string& seq) : m_alphabet(&gDNAAlphabet), m_seq(seq) { m_rc_seq = m_alphabet->reverse_complement(seq); }
    HMMInputSequence(const std::string& fwd, const Alphabet* alphabet) : m_alphabet(alphabet), m_seq(fwd) { m_rc_seq = m_alphabet->reverse_complement(m_seq); }
    HMMInputSequence(const std::string& fwd, const std::string& rc, const Alphabet* alphabet) : m_alphabet(alphabet), m_seq(fwd), m_rc_seq(rc) {}
    HMMInputSequence(std::string&& fwd, std::string&& rc, const Alphabet* alphabet) : m_alphabet(alphabet), m_seq(std::move(fwd)), m_rc_seq(std::move(rc)) {}

    const std::string& get_sequence() const { return m_seq; }
    const Alphabet* get_alphabet() const { return m_alphabet; }
    size_t length() const { return m_seq.length(); }
    void swap() { m_seq.swap(m_rc_seq); }
    std::string get_kmer(uint32_t i, uint32_t k, bool do_rc) const
    {
        return !do_rc ? m_seq.substr(i, k) : m_rc_seq.substr(m_rc_seq.length() - i - k, k);
    }
    size_t get_num_kmer_ranks(size_t k) const { return m_alphabet->get_num_strings(k); }
    // rank of the i-th k-mer; with do_rc the rank of its reverse complement (NOT the i-th k-mer of the rc string)
    uint32_t get_kmer_rank(uint32_t i, uint32_t k, bool do_rc) const
    {
        return !do_rc ? m_alphabet->kmer_rank(m_seq.c_str() + i, k)
                      : m_alphabet->kmer_rank(m_rc_seq.c_str() + (length() - i - k), k);
    }

    // all n = length() - k + 1 ranks get_kmer_rank(0..n-1, k, do_rc) in one rolling pass (appended to out)
    void append_kmer_ranks(uint32_t k, bool do_rc, std::vector<uint32_t>& out) const;
    // the alphabet ranks of the symbols of the string the strand reads (m_seq, or m_rc_seq with do_rc): what the *_seq calls of
    // the C ABI take — k-mer i of a job is then the k codes at i, resp. at length - i - k (appended to out)
    void append_codes(bool do_rc, std::vector<uint8_t>& out) const;

private:
    const Alphabet* m_alphabet;
    std::string m_seq, m_rc_seq;
};

struct AlignedPair { int ref_pos; int read_pos; };

// ---------------------------------------------------------------------------------------------
// Engine + batches
// ---------------------------------------------------------------------------------------------
extern double hmm_indel_bias_factor;   // ref: src/hmm/nanopolish_profile_hmm_r9.cpp:19 (default 1.0)

class Engine {
public:
    explicit Engine(int device = 0);
    ~Engine();
    Engine(const Engine&) = delete;
    Engine& operator=(const Engine&) = delete;
    nph_ctx* ctx() const { return m_ctx; }
    uint32_t model_id(const PoreModel* model);       // uploads on first use
    void forget_model(const PoreModel* model) { m_models.erase(model); }   // after a model was edited in place
    static Engine& thread_default();                  // lazily created, device from $NPH_DEVICE (default 0)
    void check(int status, const char* what) const;
    // page-locked host staging owned by the engine, grown on demand and reused across calls: one buffer per use
    enum class Staging { EventalignRecords, EventMeans, StartTimes, MethylationSites, EventalignTsvIn, EventalignTsv, Count };
    void* pinned(Staging use, size_t bytes);
    // the buffer of a use as it stands (nullptr and 0 before the first pinned() for it)
    void* pinned_if_any(Staging use, size_t* bytes) const { *bytes = m_pinned[(int)use].bytes; return m_pinned[(int)use].p; }

private:
    nph_ctx* m_ctx = nullptr;
    std::unordered_map<const PoreModel*, uint32_t> m_models;
    struct Pinned { void* p = nullptr; size_t bytes = 0; };
    Pinned m_pinned[(int)Staging::Count];
};

// == snprintf(dst, ..., "%.<prec>lf", v), byte for byte, by exact integer arithmetic on the binary value (round half to
// even on the exact quotient — what glibc prints in the default rounding mode; csrc/tsv_format.cuh).  float: prec <= 5;
// double: prec <= 3.  Other precisions, magnitudes of 2^39 (float) / 2^52 (double) and above and non-finite values take
// snprintf.  Returns the length.
size_t format_fixed(char* dst, float v, int prec);
size_t format_fixed(char* dst, double v, int prec);

// Threads the host-side batch loops use (chain building, record scatter, TSV formatting): $NPH_HOST_THREADS if set,
// else min(omp_get_max_threads(), 32) — GPU nodes expose many more logical CPUs than a container's CPU quota covers
// (e.g. 128 logical CPUs under a cgroup quota of 16), and a parallel region that oversubscribes them pays for it at every
// barrier; short bursts of 32-64 threads still fit one quota period.
int host_threads();

// body(i) for every i in [0, n) on `threads` workers, handed out `chunk` indices at a time.  An exception must not leave an
// OpenMP region (that terminates the process): the message of the lowest index that threw is rethrown after the loop.
template <typename Body>
void parallel_for(size_t n, int threads, int chunk, const Body& body)
{
    long long failed = (long long)n;
    std::string what;
#pragma omp parallel for schedule(dynamic, chunk) num_threads(threads) if (threads > 1)
    for (long long i = 0; i < (long long)n; ++i) {
        try {
            body((size_t)i);
        } catch (const std::exception& e) {
#pragma omp critical(nph_parallel_for_error)
            if (i < failed) { failed = i; what = e.what(); }
        }
    }
    if (failed < (long long)n) throw Error(NPH_ERR_INVALID, what);
}

namespace detail {
// The distinct (read, strand) pairs of a batch, numbered in the order they were first seen: the nph_read index the jobs
// and records of the C ABI carry.
class ReadTable {
public:
    typedef std::pair<const SquiggleRead*, uint8_t> Key;
    uint32_t index(const SquiggleRead* read, uint8_t strand)
    {
        const Key key(read, strand);
        if (!m_reads.empty() && m_reads.back() == key) return (uint32_t)m_reads.size() - 1;   // consecutive jobs of one read: the common case
        auto it = m_index.find(key);
        if (it != m_index.end()) return it->second;
        m_index.emplace(key, (uint32_t)m_reads.size());
        m_reads.push_back(key);
        return (uint32_t)m_reads.size() - 1;
    }
    const std::vector<Key>& reads() const { return m_reads; }
    size_t size() const { return m_reads.size(); }
    void clear() { m_index.clear(); m_reads.clear(); }

private:
    std::map<Key, uint32_t> m_index;
    std::vector<Key> m_reads;
};

// The table's reads -> the flat nph_read records + event arrays the C ABI takes.  The arrays live in the engine's
// page-locked staging (no page faults after the first batch, full-speed H2D) and stay valid until the next flatten on the
// same engine; time is nullptr when no read has a drift term (the start times are then not needed).
struct FlatReads {
    std::vector<nph_read> reads;
    const float* mean = nullptr;
    const double* time = nullptr;
    size_t n_events = 0;
};
FlatReads flatten_reads(Engine& engine, const ReadTable& table);

// What profile_hmm_score / profile_hmm_align check of one job, and the job: read resolved through `reads`; rank_off and
// model_id are the caller's to fill.
nph_hmm_job make_hmm_job(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags, ReadTable& reads);
// jobs[j].model_id = engine.model_id(models[j])
void resolve_model_ids(Engine& engine, const std::vector<const PoreModel*>& models, std::vector<nph_hmm_job>& jobs);
}

// A batch of profile_hmm_score calls.  add() returns the index of the job's score in run()'s result.
// Where the k-mer ranks of one HMMInputSequence already sit in a batch (per strand), so that scoring the same sequence
// against many reads — a haplotype against a pile-up — stores and uploads them once.  One cache per sequence object and
// batch; a default-constructed cache is empty.
struct RankCache {
    uint64_t off[2] = {~(uint64_t)0, ~(uint64_t)0};     // [rc]
    uint32_t k = 0;
};

class HmmBatch {
public:
    size_t add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags = 0);
    // the same; the ranks are taken from / recorded in `cache`, which must belong to this sequence and this batch
    size_t add(const HMMInputSequence& sequence, const HMMInputData& data, uint32_t flags, RankCache& cache);
    size_t size() const { return m_jobs.size(); }
    void clear();
    std::vector<float> run(Engine& engine, double indel_bias = hmm_indel_bias_factor);
    const std::vector<nph_hmm_job>& jobs() const { return m_jobs; }
    // the k-mer ranks of the queued jobs, ranks()[job.rank_off + i] = get_kmer_rank(i, k, rc) — derived from the codes on request
    // (the batch itself ships one byte per base; for inspection and tests)
    std::vector<uint32_t> ranks() const;
    const std::vector<uint8_t>& codes() const { return m_codes; }

private:
    detail::ReadTable m_reads;
    std::vector<const PoreModel*> m_job_models;
    std::vector<nph_hmm_job> m_jobs;
    std::vector<uint8_t> m_codes;           // per distinct (sequence, strand): its symbols' alphabet ranks; jobs' rank_off index this
};

// A batch of adaptive_banded_simple_event_align calls (one per read).
class AbeaBatch {
public:
    size_t add(SquiggleRead& read, const PoreModel& pore_model, const std::string& sequence);
    size_t size() const { return m_jobs.size(); }
    void clear();
    std::vector<std::vector<AlignedPair>> run(Engine& engine);

private:
    detail::ReadTable m_reads;
    const PoreModel* m_model = nullptr;
    std::vector<nph_abea_job> m_jobs;
    std::vector<uint32_t> m_ranks;
    uint64_t m_pairs_total = 0;
};

// ---- the reference's free functions (batch of one through Engine::thread_default()) ----
float profile_hmm_score(const HMMInputSequence& sequence, const HMMInputData& data, const uint32_t flags = 0);
float profile_hmm_score(const HMMInputSequence& sequence, const std::vector<HMMInputData>& data, const uint32_t flags = 0);
float profile_hmm_score_set(const std::vector<HMMInputSequence>& sequences, const HMMInputData& data, const uint32_t flags = 0);
std::vector<AlignedPair> adaptive_banded_simple_event_align(SquiggleRead& read, const PoreModel& pore_model, const std::string& sequence);
// event_table of scrappie reduced to what the function reads: the event means
SquiggleScalings estimate_scalings_using_mom(const std::string& sequence, const PoreModel& pore_model, const std::vector<float>& event_means);

} // namespace nph
