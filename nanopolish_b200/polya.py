"""nanopolish polya's output: the header and one TSV row per primary record (src/nanopolish_polya_estimator.cpp:765-766,
:823-826, :877), from the results of Engine.polya_batch.  There is one row per read, so the rows are formatted here on the
host with the reference's format string; Python's %-formatting rounds doubles like glibc's printf, and prints the infinite
read rate of a read whose median k-mer duration is 0 as "inf", as glibc does.

Secondary records (BAM_FSECONDARY) produce no row; the caller drops them before the batch.
"""
from __future__ import annotations

HEADER = "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\tpolya_length\tqc_tag\n"
QC_TAGS = ("PASS", "NOREGION", "ADAPTER", "SUFFCLIP", "READ_FAILED_LOAD")
READ_FAILED_LOAD = 4
BAM_FSECONDARY = 0x100


def _size_t_plus_one(v: int) -> float:
    # region_indices.x + 1 in size_t, then converted to double
    return float((int(v) + 1) % (1 << 64))


def row(name: str, contig: str, pos: int, res) -> str:
    """The row of one record; res is one POLYA_RES_DT element."""
    if int(res["qc"]) == READ_FAILED_LOAD:
        return "%s\t%s\t%d\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n" % (name, contig, pos)
    return "%s\t%s\t%d\t%.1f\t%.1f\t%.1f\t%.1f\t%.2f\t%.2f\t%s\n" % (
        name, contig, pos, _size_t_plus_one(res["start"]), _size_t_plus_one(res["leader"]), _size_t_plus_one(res["adapter"]),
        _size_t_plus_one(res["polya"]), float(res["read_rate"]), float(res["polya_length"]), QC_TAGS[int(res["qc"])])


def rows(names, contigs, positions, results) -> str:
    return "".join(row(n, c, int(p), r) for n, c, p, r in zip(names, contigs, positions, results))
