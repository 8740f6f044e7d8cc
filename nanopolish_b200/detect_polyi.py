"""nanopolish detect-polyi's output: the header and one TSV row per primary record (src/nanopolish_detect_polyi.cpp:1040-1041,
:1105-1108, :1159), from the results of Engine.detect_polyi_batch.  The row is polya's with a `detected` column before
`qc_tag`; a read that failed to load gets polya's 10-column row, without `detected`, as the reference prints it.

Secondary records (BAM_FSECONDARY) produce no row; the caller drops them before the batch.
"""
from __future__ import annotations

from .polya import QC_TAGS, READ_FAILED_LOAD, _row  # noqa: F401 (QC_TAGS, READ_FAILED_LOAD: public here too)

HEADER = ("readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\tpolya_length\t"
          "detected\tqc_tag\n")
DETECTED_TAGS = ("NONE", "POLYA-ONLY", "POLYI-ONLY", "A+I")     # NPH_POLYI_*


def row(name: str, contig: str, pos: int, res) -> str:
    """The row of one record; res is one POLYI_RES_DT element."""
    return _row(name, contig, pos, res["seg"], (DETECTED_TAGS[int(res["detected"])],))


def rows(names, contigs, positions, results) -> str:
    return "".join(row(n, c, int(p), r) for n, c, p, r in zip(names, contigs, positions, results))
