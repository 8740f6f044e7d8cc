"""Pin the port oracle's tail caller (npo_polya_trace in oracle/np_oracle.c) to the compiled reference's poly(A) and
detect-polyi (oracle/_ref/libnpref_polya.so and libnpref_polyi.so) on every edge case of tests/tail_cases.py: the segmentation,
the read rate and length bit for bit, the QC, the Bernoulli pair, the detection tag and the TSV row.  The port is also pinned to
the slow Python restatements in polya_cases / polyi_cases on short reads, the builders' claims are checked on its traces, and
the coverage tables go to the test log.

The reference's answers live in tests/golden/ref_tail_edges.pkl.xz (a ref_calls.CaseRecord: asked live where both libraries
exist and compared with the record, replayed elsewhere).  NPH_REF_CASES_RECORD=<dir> pytest tests/test_tail_edges_oracle.py
writes a new record to <dir>."""
import os
import re

import numpy as np
import pytest

from tests import polya_cases as pc
from tests import polyi_cases as qc
from tests import ref_calls
from tests import tail_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLYA_CU = os.path.join(ROOT, "nanopolish_b200", "csrc", "polya.cu")

reference = ref_calls.case_fixture(tc.GOLDEN, ref=tc.live_refs)


@pytest.fixture(scope="module")
def cases(port_oracle):
    return tc.all_cases(port_oracle)


def test_kernel_constants():
    """the tile, CTA, flat-tile and QC constants tail_cases.py restates are polya.cu's"""
    src = open(POLYA_CU).read()
    assert re.search(r"constexpr int kTile = (\d+);", src).group(1) == str(tc.TILE)
    assert re.search(r"constexpr int kEmitWarps = (\d+);", src).group(1) == str(tc.EMIT_WARPS)
    assert "constexpr int kThreads = 32 * (1 + kEmitWarps);" in src
    assert "constexpr uint32_t kFlat = N_ST * kTile;" in src
    assert "enum { ST_S = 0, ST_L, ST_A, ST_P, ST_C, ST_T, N_ST };" in src and tc.N_ST == 6
    assert "for (uint32_t i = tid; i < nk; i += kThreads)" in src          # the selection's stride over k-mers
    assert "if (tid == 0) s_rank = nk / 2;" in src
    assert f"if (m >= {tc.MIN_TAIL})" in src
    assert f"if (n_adapter < {tc.MIN_REGION} || n_polya < {tc.MIN_REGION}) qc = NPH_POLYA_NOREGION;" in src
    assert f"else if (adapter_length > {tc.MAX_ADAPTER}) qc = NPH_POLYA_ADAPTER;" in src
    assert f"else if (jb.suffix_clip > {tc.MAX_CLIP}) qc = NPH_POLYA_SUFFCLIP;" in src
    assert "emissions<kPolyi>(x[i == 0 ? n - 1 : i], s_g, e);" in src


def test_port_matches_the_python_restatement(port_oracle):
    """npo_polya_trace against polya_cases.restate_segment / restate_rate and polyi_cases.restate_segment / restate_bernoulli"""
    rng = np.random.default_rng(31)
    reads = [pc.synth_read(rng, f"r{i}", int(n)) for i, n in enumerate((2, 3, 5, 257, 600, 1500))]
    reads += [qc.synth_polyi_read(rng, f"q{i}", int(n)) for i, n in enumerate((900, 1700, 2600))]
    for r in reads:
        for polyi in (False, True):
            t = port_oracle.tail_trace(r, polyi)
            m = qc if polyi else pc
            assert tuple(int(v) for v in t["seg"]) == tuple(int(v) for v in m.restate_segment(r.samples, r.scale, r.shift, r.var)), r.name
            assert t["read_rate"] == pc.restate_rate(r), r.name
            if polyi:
                start, stop = int(t["seg"][2]) + 1, int(t["seg"][3])
                assert (t["polyi_last"], t["polya_first"]) == qc.restate_bernoulli(r, start, stop), r.name


@pytest.mark.parametrize("mode", tc.MODES)
def test_edges_match_reference(reference, port_oracle, cases, mode):
    cs = [c for c in cases if c.mode == mode]
    got = reference.answers(mode, [tc.fingerprint(c) for c in cs], lambda i: reference.live.answer(cs[i]))
    bad = [(c.name, tc.port_answer(port_oracle, c), g) for c, g in zip(cs, got) if tc.port_answer(port_oracle, c) != g]
    assert not bad, f"{len(bad)} of {len(cs)} cases: the port differs from the reference, first: {bad[:2]}"
    assert len(cs) > 100


def test_builders_reach_every_edge(port_oracle, cases):
    cover, _ = tc.check_tail_edges(port_oracle, cases)
    print()
    for fam, c in cover.items():
        print(tc.coverage_table(c, fam))
    for mode in tc.MODES:
        found = tc.finite_tie_search(port_oracle, mode, n_try=3000)
        print(f"{mode}: finite ties the backtrack read on quantised constant / periodic signals:",
              ", ".join(tc.RULES[k] for k in sorted(found)) or "none",
              "| not reached:", ", ".join(r for k, r in enumerate(tc.RULES) if k not in found))


def test_latest_bernoulli_switch():
    """The first A of the Bernoulli path is at least 7 steps before the tail's end, whatever the bits: a path that switches at
    step s stays in A for d = m - s steps, and it beats staying in I only if logf(0.1) + d * (eA - eI) > d * logf(0.9), where
    eA - eI is largest on a 1 bit (logf(0.92154) - logf(0.72304)).  So the kernel's `i + 1 < m` guard never decides, and the
    latest switch tail_cases reaches is m - 7.  Also, row 0's A score is -inf, so step 1's pointer into A is always I and the
    earliest switch is 2."""
    f = np.float32
    lg = lambda v: f(qc._logf(f(v)))
    gain = f(lg(0.92154) - lg(0.72304))
    for d in range(1, 7):
        assert f(lg(0.10) + f(d) * gain) < f(f(d) * lg(0.90)), d
    assert f(lg(0.10) + f(7) * gain) > f(f(7) * lg(0.90))
