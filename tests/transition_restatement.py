"""TransitionParameters' training, restated (src/hmm/nanopolish_transition_parameters.cpp:294-448): add_training_from_alignment
over a profile_hmm_align path, the skip-bin histogram train() reads, train() itself and print(), and model_score's segment cutting
(src/nanopolish_scorereads.cpp:116-203).  Counts are kept in the layout of nph_transition_counts (include/nph.h): 81 words,
state_transitions (3 x 6), n_matches, n_merges, n_skips, skip_total[30], skip_count[30]."""
import numpy as np

WORDS, MATCHES, MERGES, SKIPS, TOTAL, COUNT, BINS = 81, 18, 19, 20, 21, 51, 30
STATE = {"M": 0, "B": 1, "K": 2}


class Asserts(Exception):
    """where the reference asserts"""


def scaled_mean(level_mean: float, scale: float, shift: float) -> np.float32:
    """get_scaled_gaussian_from_pore_model_state's mean: scale * level_mean + shift in double, narrowed to float"""
    return np.float32(scale * level_mean + shift)


def skip_bin(l1: np.float32, l2: np.float32) -> int:
    """get_skip_bin: (size_t)(fabs(l1 - l2) / 0.5), clamped to the last bin"""
    q = abs(float(l1) - float(l2)) / 0.5
    return BINS - 1 if q >= BINS - 1 else int(q)


def add_training(counts, path, ranks, mean_of, ignore=5, trace=None):
    """add_training_from_alignment(sequence, data, path, ignore): path = [(event_idx, kmer_idx, state char)], ranks[i] =
    get_kmer_rank(i, k, rc), mean_of(rank) = the scaled mean.  trace (a list) receives ('obs', pi, from, to, bin, state) and
    ('interior', pi) records for the edge checks."""
    n = len(path)
    if n <= ignore:
        return
    n_kmers = len(ranks)
    prev = "M"
    for pi, (_, ki, s) in enumerate(path):
        if s not in STATE or prev not in STATE:
            raise Asserts("state")
        move = pi == 0 or path[pi - 1][1] != ki
        t = STATE[prev] * 6 + 2 * STATE[s] + int(move)
        counts[t] += 1
        if ignore < pi < n - ignore:
            if trace is not None:
                trace.append(("interior", pi))
            if s != "B":
                fr, to = path[pi - 1][1], ki
                if s == "K" and prev == "M":
                    to = fr + 1
                if fr >= n_kmers or to >= n_kmers:
                    raise Asserts("kmer")
                l1, l2 = mean_of(ranks[fr]), mean_of(ranks[to])
                if not (np.isfinite(l1) and np.isfinite(l2)):
                    raise Asserts("mean")
                b = skip_bin(l1, l2)
                counts[TOTAL + b] += 1
                counts[COUNT + b] += s == "K"
                if trace is not None:
                    trace.append(("obs", pi, fr, to, b, s, prev, abs(float(l1) - float(l2))))
            counts[t] += 1
        prev = s
        counts[MATCHES] += s == "M"
        counts[MERGES] += s == "E"
        counts[SKIPS] += s == "K"


def train(counts, prior=None):
    """TransitionParameters::train(): per bin skip = prior * 100, total = 100, +is_skip and +1 per observation in turn"""
    out = []
    for b in range(BINS):
        skip = (0.0 if prior is None else float(prior[b])) * 100
        for _ in range(int(counts[COUNT + b])):
            skip += 1.0
        out.append(skip / (100.0 + float(counts[TOTAL + b])))
    return out


def report(counts2, priors=(None, None)) -> str:
    """scorereads' stderr after --train-transitions"""
    s = ""
    for strand in range(2):
        s += f"Transition parameters for {strand}\n"
        s += "".join(f"skip_probabilities[{b}] = {p:.3f};\n" for b, p in enumerate(train(counts2[strand], priors[strand])))
    return s


def segments(alignment, ref_seq, ref_pos0, eps, k):
    """model_score's segments: [(event_start, event_stop, segment bases)] of alignment = [(ref_position, event_idx)], ref_seq
    the contig from ref_pos0; segments with fetched_len <= k are skipped (and returned in `skipped`)"""
    out, skipped = [], []
    a = eps
    while a < len(alignment) - eps:
        (r0, e0), (r1, e1) = alignment[a], alignment[a + eps]
        seg = ref_seq[max(0, r0 - ref_pos0):max(0, min(r1 - ref_pos0, len(ref_seq) - 1) + 1)]
        (skipped if len(seg) <= k else out).append((e0, e1, seg))
        a += eps
    return out, skipped
