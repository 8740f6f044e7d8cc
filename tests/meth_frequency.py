"""A restatement of the reference's scripts/calculate_methylation_frequency.py, the checker of nph_methfreq_* (written from the
script's rules, not from its code; tests/test_meth_frequency_oracle.py pins it to the script's own output).

Per row of the methylation_calls.tsv inputs, in order: llr = float(log_lik_ratio); the row is skipped when abs(llr) <
threshold * num_motifs; it is methylated when llr > 0.  Without split (or for one-motif groups) it adds num_motifs calls to
(chromosome, start, end); with split, every "CG" of its sequence (overlapping ones too) adds one call to (chromosome, start +
pos - first_pos, same) with group size 1 and sequence "split-group".  A key keeps the group size and sequence of the row that
created it.  Output: the header, then the keys in Python's tuple order, "%.3f" of the double methylated / called.
"""
from __future__ import annotations

HEADER = "\t".join(["chromosome", "start", "end", "num_motifs_in_group", "called_sites", "called_sites_methylated",
                    "methylated_frequency", "group_sequence"]) + "\n"
CALLS_HEADER = "\t".join(["chromosome", "strand", "start", "end", "read_name", "log_lik_ratio", "log_lik_methylated",
                          "log_lik_unmethylated", "num_calling_strands", "num_motifs", "sequence"]) + "\n"


def _cg_positions(seq: str):
    return [i for i in range(len(seq) - 1) if seq[i] == "C" and seq[i + 1] == "G"]


def frequency_table(tsv_texts: list, call_threshold: float = 2.0, split_groups: bool = False) -> str:
    """the script's stdout for the input files whose contents are tsv_texts (each with its header line)"""
    sites = {}            # key -> [group size, sequence, called, methylated]

    def add(key, n, methylated, seq):
        s = sites.setdefault(key, [n, seq, 0, 0])
        s[2] += n
        if methylated:
            s[3] += n

    for text in tsv_texts:
        lines = text.split("\n")
        cols = lines[0].split("\t")
        for line in lines[1:]:
            if not line:
                continue
            row = dict(zip(cols, line.split("\t")))
            n = int(row["num_motifs"])
            llr = float(row["log_lik_ratio"])
            if abs(llr) < call_threshold * n:
                continue
            c, s, e, seq = row["chromosome"], int(row["start"]), int(row["end"]), row["sequence"]
            if split_groups and n > 1:
                pos = _cg_positions(seq)
                for p in pos:
                    add((c, s + p - pos[0], s + p - pos[0]), 1, llr > 0, "split-group")
            else:
                add((c, s, e), n, llr > 0, seq)
    out = [HEADER]
    for key in sorted(sites):
        n, seq, called, meth = sites[key]
        out.append("%s\t%s\t%s\t%d\t%d\t%d\t%.3f\t%s\n" % (key[0], key[1], key[2], n, called, meth, float(meth) / called, seq))
    return "".join(out)
