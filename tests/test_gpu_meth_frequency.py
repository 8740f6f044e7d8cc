"""The per-site methylation frequency table on the device (nph_methfreq_*, csrc/meth_frequency.cu) through the C ABI.

The checker is tests/meth_frequency.py, the restatement of the reference's calculate_methylation_frequency.py (pinned to the script's
own output in tests/test_meth_frequency_oracle.py), applied to the rows the device itself writes for the same batches
(nph_methylation_tsv, pinned byte for byte to the compiled reference in tests/test_gpu_methylation.py).  So the table folded on the
device must be, byte for byte, what the script prints for the concatenated methylation_calls.tsv of the batches."""
import numpy as np
import pytest

from nanopolish_b200 import synth
from nanopolish_b200._lib import NphError
from tests import meth_frequency as mf

pytestmark = pytest.mark.gpu
K = 6
NPH_ERR_INVALID, NPH_ERR_STATE = -3, -5
CONTIGS = ["chr2", "chr10", "chr1"]          # contig ids 0, 1, 2: id order is not name order


@pytest.fixture(scope="module")
def eng():
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    e.model_upload(synth.load_model("nucleotide"))
    e.model_upload(synth.load_model("cpg"))
    yield e
    e.close()


def _batch(seed, n_reads, ref_start):
    rs = synth.gen_reads(n_reads, 2500, synth.load_model("nucleotide"), seed=seed, cpg_keep=0.3)
    ref, pairs, recs = synth.methylation_records(rs, model_id=1, ref_start=ref_start, rc_every=2)
    return rs, ref, pairs, recs


@pytest.fixture(scope="module")
def batches():
    """six batches over three contigs; the reads of a contig start at nearby positions, so keys repeat within and across batches"""
    return [(b % 3, _batch(4100 + 1000 * b, 250, 10_000 + 17 * (b // 3))) for b in range(6)]


def _run(eng, batch, params=None):
    """score the batch; its methylation_calls.tsv as the script reads it (header + the device's rows)"""
    contig_id, (rs, ref, pairs, recs) = batch
    eng.reads_load(rs.reads, rs.ev_mean, rs.ev_start_time)
    eng.methylation_load(ref, pairs, recs, params if params is not None else synth.meth_params("cpg", K))
    eng.methylation_run()
    names = ["read_%d" % i for i in range(recs.shape[0])]
    return mf.CALLS_HEADER + eng.methylation_tsv(CONTIGS[contig_id], names, recs["rc"]).decode()


def _fold(eng, batches, t, split):
    eng.methylation_frequency_reset(t, split)
    texts = []
    for b in batches:
        texts.append(_run(eng, b))
        eng.methylation_frequency_add(b[0])
    return texts


def _rows(texts):
    for text in texts:
        for line in text.split("\n")[1:]:
            if line:
                f = line.split("\t")
                yield f[0], int(f[2]), int(f[3]), f[5], int(f[9]), f[10]


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("t", [0.0, 2.0])
def test_table_equals_the_script_on_the_device_rows(eng, batches, t, split):
    texts = _fold(eng, batches, t, split)
    got = eng.methylation_frequency_tsv(CONTIGS).decode()
    want = mf.frequency_table(texts, t, split)
    assert got == want
    n_keys, n_calls, n_ambiguous = eng.methylation_frequency_counts()
    assert n_keys == want.count("\n") - 1 > 1000
    rows = list(_rows(texts))
    assert n_ambiguous == sum(1 for r in rows if abs(float(r[3])) < t * r[4])
    assert (n_ambiguous == 0) == (t == 0.0) and n_calls > 0


def test_workload_is_not_vacuous(eng, batches):
    """the batches hold a key seen with two different sequences, a split key that meets a single-site key, and rows printed as
    0.00 / -0.00 (D == 0)"""
    rows = list(_rows([_run(eng, b) for b in batches]))
    seqs = {}
    for c, s, e, llr, n, seq in rows:
        seqs.setdefault((c, s, e), set()).add(seq)
    assert any(len(v) > 1 for v in seqs.values())
    singles = {(c, s, e) for c, s, e, _, n, _ in rows if n == 1}
    split = set()
    for c, s, e, _, n, seq in rows:
        if n > 1:
            pos = [i for i in range(len(seq) - 1) if seq[i:i + 2] == "CG"]
            split.update((c, s + p - pos[0], s + p - pos[0]) for p in pos)
    assert split & singles
    assert any(r[3] in ("0.00", "-0.00") for r in rows)


def test_threshold_on_a_row(eng, batches):
    """the threshold equal to |llr| of a one-motif row: that row sits exactly on the boundary and counts"""
    texts = [_run(eng, b) for b in batches[:2]]
    row = next(r for r in _rows(texts) if r[4] == 1 and r[3] not in ("0.00", "-0.00"))
    t = abs(float(row[3]))
    texts = _fold(eng, batches[:2], t, False)
    want = mf.frequency_table(texts, t, False)
    assert eng.methylation_frequency_tsv(CONTIGS).decode() == want
    assert "\t%d\t%d\t" % (row[1], row[2]) in want


def test_growth_mid_run_output_and_reset(eng, batches):
    """a one-read first batch (the table starts at 1 024 slots, grown past half full), output between folds, reset"""
    small = (1, _batch(77, 1, 10_000))
    eng.methylation_frequency_reset(2.0, True)
    texts = [_run(eng, small)]
    eng.methylation_frequency_add(small[0])
    first_keys = eng.methylation_frequency_counts()[0]
    for b in batches[:3]:
        texts.append(_run(eng, b)); eng.methylation_frequency_add(b[0])
    mid = eng.methylation_frequency_tsv(CONTIGS)
    assert mid.decode() == mf.frequency_table(texts, 2.0, True)
    assert eng.methylation_frequency_tsv(CONTIGS) == mid
    for b in batches[3:]:
        texts.append(_run(eng, b)); eng.methylation_frequency_add(b[0])
    got = eng.methylation_frequency_tsv(CONTIGS).decode()
    assert got == mf.frequency_table(texts, 2.0, True)
    n_keys = eng.methylation_frequency_counts()[0]
    assert first_keys < 512 < n_keys
    # the same folds into a table that starts large enough give the same bytes
    eng.methylation_frequency_reset(2.0, True)
    for b in batches:
        _run(eng, b); eng.methylation_frequency_add(b[0])
    _run(eng, small); eng.methylation_frequency_add(small[0])
    texts2 = texts[1:] + texts[:1]
    assert eng.methylation_frequency_tsv(CONTIGS).decode() == mf.frequency_table(texts2, 2.0, True)
    eng.methylation_frequency_reset()
    assert eng.methylation_frequency_counts() == (0, 0, 0)
    assert eng.methylation_frequency_tsv(CONTIGS).decode() == mf.HEADER


def test_refusals(eng, batches):
    from nanopolish_b200.engine import Engine
    fresh = Engine(0)
    try:
        with pytest.raises(NphError) as ex:
            fresh.methylation_frequency_add(0)
        assert ex.value.status == NPH_ERR_STATE
    finally:
        fresh.close()
    texts = _fold(eng, batches[:2], 2.0, False)
    want = mf.frequency_table(texts, 2.0, False)
    with pytest.raises(NphError) as ex:
        eng.methylation_frequency_tsv(CONTIGS, cap=100)
    assert ex.value.status == NPH_ERR_INVALID
    assert eng.methylation_frequency_tsv(CONTIGS, cap=len(want)).decode() == want
    for names in (CONTIGS[:1], ["chr2", "chr10", "chr2"]):         # contig id 1 has no name; a name twice
        with pytest.raises(NphError) as ex:
            eng.methylation_frequency_tsv(names)
        assert ex.value.status == NPH_ERR_INVALID
    # a batch whose window parameters let a group start fewer than k - 1 bases into its record: its sequence column is undefined
    contig_id, (rs, ref, pairs, recs) = batches[2]
    ref, recs = ref.copy(), recs.copy()
    recs[0]["ref_off"] += 6; recs[0]["ref_len"] -= 6; recs[0]["ref_start_pos"] += 6      # the event alignment starts at offset 0
    o = int(recs[0]["ref_off"])
    ref[o:o + 8] = np.frombuffer(b"AAAACGAA", np.uint8)                                   # a site at offset 4
    params = synth.meth_params("cpg", K, min_separation=0, min_flank=3, min_event_span=0)
    before = eng.methylation_frequency_counts()
    with pytest.raises(NphError) as ex:
        _run(eng, (contig_id, (rs, ref, pairs, recs)), params)            # nph_methylation_tsv refuses the batch
    assert ex.value.status == NPH_ERR_INVALID
    with pytest.raises(NphError) as ex:
        eng.methylation_frequency_add(contig_id)
    assert ex.value.status == NPH_ERR_INVALID
    assert eng.methylation_frequency_counts() == before
    assert eng.methylation_frequency_tsv(CONTIGS).decode() == want


def test_frequency_number_formatting_on_device():
    """fixed_of<3> == printf("%.3f") of every m / n, n <= 5000, and fixed_of<2> unchanged, on the device"""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "checks", "check_tsv_format")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "device: 0 bad" in r.stdout
