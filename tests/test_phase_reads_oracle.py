"""The compiled reference's own phase_single_read (src/nanopolish_phase_reads.cpp:178-347, run unmodified by
oracle/phase_reads_harness.cpp) against the restatement in tests/phase_restatement.py with oracle forward scores: the SAM line of
every record, byte for byte, on reads of both strands with gapped and soft-clipped CIGARs and IUPAC / lower-case contig bases,
variant lists with SNPs, REF mismatches, lower-case REFs, non-SNPs, two variants at one position and ties, records whose range is
empty (a line of the plain reference, every quality '?') and records with no variant at or after them (no line)."""
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import phase_cases as pc


@pytest.fixture(scope="module")
def ref_phase():
    if not os.path.exists(pc.REF_PHASE):
        pytest.skip("oracle/_ref/libnpref_phase.so not built (it needs the reference sources)")
    return pc.RefPhase()


def test_sam_lines_equal_reference(ref_phase, port_oracle):
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(8, 2000, model, seed=515)
    cl = pc.cases(rs)
    hs = ref_phase.register(rs, cl)
    rng = np.random.default_rng(3)
    n_lines = n_called = 0
    for i, c in enumerate(cl):
        var = pc.plant(c, rng)
        for v in (var, [x for x in var if x[0] > c["ref_pos"] + len(c["upper"])], []):   # planted; empty range; nothing at or after
            want = pc.restated(port_oracle, rs, model, i, c, v)
            got = ref_phase.line(hs[i], c, v)
            assert got == want
            if got:
                n_lines += 1
                n_called += sum(q != "?" for q in got.split("\t")[10].strip())
        assert pc.restated(port_oracle, rs, model, i, c, []) is None
    assert n_lines == 16 and n_called > 20
