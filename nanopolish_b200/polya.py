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


def _row(name: str, contig: str, pos: int, seg, extra=()) -> str:
    """The row of one record from its POLYA_RES_DT segmentation, with the extra columns before qc_tag; a read that failed to
    load gets the 10-column row without them."""
    if int(seg["qc"]) == READ_FAILED_LOAD:
        return "%s\t%s\t%d\t-1.0\t-1.0\t-1.0\t-1.0\t-1.00\t-1.00\tREAD_FAILED_LOAD\n" % (name, contig, pos)
    numbers = "%s\t%s\t%d\t%.1f\t%.1f\t%.1f\t%.1f\t%.2f\t%.2f" % (
        name, contig, pos, _size_t_plus_one(seg["start"]), _size_t_plus_one(seg["leader"]), _size_t_plus_one(seg["adapter"]),
        _size_t_plus_one(seg["polya"]), float(seg["read_rate"]), float(seg["polya_length"]))
    return "\t".join([numbers, *extra, QC_TAGS[int(seg["qc"])]]) + "\n"


def row(name: str, contig: str, pos: int, res) -> str:
    """The row of one record; res is one POLYA_RES_DT element."""
    return _row(name, contig, pos, res)


def rows(names, contigs, positions, results) -> str:
    return "".join(row(n, c, int(p), r) for n, c, p, r in zip(names, contigs, positions, results))
