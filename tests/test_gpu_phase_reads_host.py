"""The C++ host mirror nph::PhaseReads (host/nph_phase_reads.hpp, through the nphh_phase_reads shim and one nph_phase_reads_batch
call): its SAM records, byte for byte, against the compiled reference's own phase_single_read (oracle/phase_reads_harness.cpp) where
that library is built, and against the restatement (tests/phase_restatement.py) always — every record-level rule (no record when no
variant lies at or after the read, a record of the plain reference when the range is empty), last-variant-wins, the SEQ round trip
through the 4-bit codes, and one line against a literal string."""
import ctypes as C
import os

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import phase_cases as pc
from tests.test_host_mirror import HOST_SO, _register, _register_reads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def host():
    lib = C.CDLL(HOST_SO)
    lib.nphh_last_error.restype = C.c_char_p
    return lib


def test_mirror_sam_equals_reference(host, port_oracle):
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(8, 2000, model, seed=515)
    cl = pc.cases(rs)
    # one contig stretch per read, so one sorted variant list serves the batch
    shift = 0
    for c in cl:
        pad = "A" * shift
        c["contig"] = pad + c["contig"]; c["ref_pos"] += shift
        c["pairs"] = [(p + shift, e) for p, e in c["pairs"]]
        shift += len(c["contig"]) + 10
    rng = np.random.default_rng(3)
    var = sorted([v for c in cl[:-2] for v in pc.plant(c, rng)[:-1]], key=lambda v: v[0])      # the last two reads: no variant at or after them
    var = [v for v in var if v[0] < cl[-2]["ref_pos"]]
    var.append((cl[-3]["ref_pos"] + len(cl[-3]["upper"]) + 2, "A", "C"))                       # read -3: an empty range, not at the end
    var = [v for v in var if not (cl[-3]["ref_pos"] <= v[0] < cl[-3]["ref_pos"] + len(cl[-3]["upper"]))]
    mh = _register(host, model)
    rh = _register_reads(host, rs, mh)
    got = pc.mirror_sam(host, rh, cl, var)
    want = [pc.restated(port_oracle, rs, model, i, c, var) for i, c in enumerate(cl)]
    assert want[-1] is None and want[-2] is None and set(want[-3].split("\t")[10].strip()) == {"?"}
    assert got == "".join(w for w in want if w)
    if os.path.exists(pc.REF_PHASE):
        ref = pc.RefPhase()
        hs = ref.register(rs, cl)
        for i, c in enumerate(cl):
            assert ref.line(hs[i], c, var) == want[i]
    assert sum(q != "?" for w in want if w for q in w.split("\t")[10].strip()) > 10


def test_mirror_literal_line(host):
    model = synth.load_model("nucleotide")
    rs = synth.gen_reads(1, 400, model, seed=1)
    mh = _register(host, model)
    rh = _register_reads(host, rs, mh)
    case = dict(name="lit", flag=16, mapq=7, ref_pos=2, upper="ACGTNRYX=acgt0", pairs=[])
    got = pc.mirror_sam(host, rh, [case], [(1000, "A", "C")])
    assert got == "lit\t16\tchr1\t3\t7\t14M\t*\t0\t0\tACGTNRYN=ACGTA\t??????????????\n"
