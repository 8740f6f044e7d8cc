"""phase-reads on the device — nph_phase_reads_batch (csrc/phase_reads.cu) through the C ABI.

The checker is tests/phase_restatement.py: a plain-Python restatement of phase_single_read's variant loop
(src/nanopolish_phase_reads.cpp:246-318) whose windows are scored by the oracle.  The device must return the same sites per
record, in list order, with bit-identical scores, the same call and quality character, and the same scored-event count.  Crafted
records hit every rule of the loop; a synthetic batch of 2 000 reads on both strands has SNPs every 30-1 000 bases (overlapping
windows), planted REF mismatches, non-SNPs, N / IUPAC reference bytes and records without variants."""
import numpy as np
import pytest

from nanopolish_b200 import _lib, synth
from tests import phase_restatement as pr

pytestmark = pytest.mark.gpu
K = 6


@pytest.fixture(scope="module")
def model():
    return synth.load_model("nucleotide")


@pytest.fixture(scope="module")
def eng(model):
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    e.model_upload(model)
    yield e
    e.close()


def _check(eng, port_oracle, model, rs, ref, pairs, recs, variants, var_range):
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    off, calls, scored = eng.phase_reads_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, recs, variants, var_range)
    sites, jobs, ranks, _ = pr.enumerate_batch(ref, pairs, recs, variants, var_range, K)
    scores = port_oracle.hmm_score_batch(rs.reads, rs.ev_mean, rs.ev_start_time, [model], ranks, jobs)[0] if jobs.shape[0] else np.zeros(0, np.float32)
    want_off, want = pr.expected_calls(sites, scores, variants, recs.shape[0])
    assert np.array_equal(off, want_off)
    assert np.array_equal(calls["record"], want["record"]) and np.array_equal(calls["variant"], want["variant"])
    assert np.array_equal(calls["ref_score"].view(np.uint32), want["ref_score"].view(np.uint32))
    assert np.array_equal(calls["alt_score"].view(np.uint32), want["alt_score"].view(np.uint32))
    assert np.array_equal(calls["call"], want["call"]) and np.array_equal(calls["qual"], want["qual"])
    E = np.abs(jobs["event_stop"].astype(np.int64) - jobs["event_start"].astype(np.int64)) + 1
    assert scored == int(E.sum())
    return calls, jobs


def _var(p, ref_base, alt_base, is_snp=1):
    return (p, ref_base, alt_base, is_snp, 0)


def _crafted(model):
    """six records on one contig stretch each: forward, reverse, forward with a stall, reverse with e1 == e2, a record whose range is
    empty but not at the end of the list, and a record with N / IUPAC bases in a scored window."""
    rs = synth.gen_reads(6, 1800, model, seed=31)
    ref, pairs, recs, _, _ = synth.phase_batch(rs, seed=1, rc_every=2, p_iupac=0.0)
    ref = ref.copy()
    var = []

    def base(r, p):
        R = recs[r]
        return bytes(ref[int(R["ref_off"]) + p - int(R["ref_start_pos"]):][:1])

    def rec_pairs(r):
        R = recs[r]
        return pairs[int(R["pair_off"]):int(R["pair_off"]) + int(R["n_pairs"])]

    other = {b"A": b"C", b"C": b"G", b"G": b"T", b"T": b"A"}
    # record 0 (forward): windows whose edge lies on the first / last aligned base and one base beyond each; a non-SNP; a REF
    # mismatch; a lowercase REF; two variants at one position; a tie (alt == ref)
    p0 = rec_pairs(0)
    f, l = int(p0["ref_pos"][0]), int(p0["ref_pos"][-1])
    for p in (f + 29, f + 30):
        var.append(_var(p, base(0, p), other[base(0, p)]))
    mid = (f + l) // 2
    var += [_var(mid - 200, base(0, mid - 200), b"T", 0), _var(mid - 150, other[base(0, mid - 150)], base(0, mid - 150)),
            _var(mid - 100, base(0, mid - 100).lower(), other[base(0, mid - 100)]),
            _var(mid, base(0, mid), other[base(0, mid)]), _var(mid, base(0, mid), other[other[base(0, mid)]]),
            _var(mid + 100, base(0, mid + 100), base(0, mid + 100))]
    for p in (l - 30, l - 29):
        var.append(_var(p, base(0, p), other[base(0, p)]))
    # record 1 (reverse): first / last aligned base windows
    p1 = rec_pairs(1)
    f1, l1 = int(p1["ref_pos"][0]), int(p1["ref_pos"][-1])
    var += [_var(f1 + 30, base(1, f1 + 30), other[base(1, f1 + 30)]), _var((f1 + l1) // 2, base(1, (f1 + l1) // 2), other[base(1, (f1 + l1) // 2)]),
            _var(l1 - 30, base(1, l1 - 30), other[base(1, l1 - 30)])]
    # record 2 (forward): a stall window, 1 300 events over 61 bases (> 20 per base, still scored)
    p2 = rec_pairs(2)
    s = int(p2["ref_pos"][0]) + 100
    tail = p2["ref_pos"] >= s + 30
    p2["read_pos"][tail] = np.minimum(p2["read_pos"][tail] + 1300, rs.reads[2]["n_events"] - 1)
    var.append(_var(s, base(2, s), other[base(2, s)]))
    # record 3 (reverse): a window with e1 == e2
    p3 = rec_pairs(3)
    q = (int(p3["ref_pos"][0]) + int(p3["ref_pos"][-1])) // 2
    inside = (p3["ref_pos"] >= q - 30) & (p3["ref_pos"] <= q + 30)
    p3["read_pos"][inside] = p3["read_pos"][inside][0]
    var.append(_var(q, base(3, q), other[base(3, q)]))
    # record 4: no variant in its range (a later record has some)
    # record 5 (reverse): N and IUPAC bytes in a scored window, and an N at a centre whose variant's REF is N
    p5 = rec_pairs(5)
    c = (int(p5["ref_pos"][0]) + int(p5["ref_pos"][-1])) // 2
    o = int(recs[5]["ref_off"]) + c - int(recs[5]["ref_start_pos"])
    ref[o - 20] = ord("N"); ref[o + 7] = ord("R"); ref[o + 25] = ord("Y")
    ref[o + 150] = ord("N")
    var += [_var(c, base(5, c), other[base(5, c)]), _var(c + 150, b"N", b"A")]
    variants = np.array(var, synth.PHASE_VARIANT_DT)
    variants = variants[np.argsort(variants["ref_position"], kind="stable")]
    return rs, ref, pairs, recs, variants, pr.var_ranges(variants["ref_position"], recs)


def test_crafted_records(eng, port_oracle, model):
    rs, ref, pairs, recs, variants, vr = _crafted(model)
    assert vr[4][0] == vr[4][1] and vr[4][0] < variants.shape[0]
    calls, jobs = _check(eng, port_oracle, model, rs, ref, pairs, recs, variants, vr)
    assert (jobs["stride"] == -1).any() and ((jobs["event_start"] == jobs["event_stop"]) & (jobs["rc"] == 1)).any()
    assert (np.abs(jobs["event_stop"].astype(np.int64) - jobs["event_start"]) > 20 * 60).any()
    assert (calls["ref_score"] == calls["alt_score"]).any() and (calls["qual"] == 63).any()
    vs = variants[calls["variant"]]
    assert (vs["ref_base"] == b"N").any() and (vs["is_snp"] == 1).all()


def test_synthetic_batch(eng, port_oracle, model):
    rs = synth.gen_reads(2000, 3000, model, seed=5)
    ref, pairs, recs, variants, vr = synth.phase_batch(rs, seed=7, step=(30, 1000), p_mismatch=0.1, p_non_snp=0.1, p_no_variants=0.1, p_iupac=0.003)
    calls, jobs = _check(eng, port_oracle, model, rs, ref, pairs, recs, variants, vr)
    assert calls.shape[0] > 2000 and (recs["rc"] == 1).any() and (vr[:, 0] == vr[:, 1]).any()
    assert (calls["call"] == variants[calls["variant"]]["alt_base"]).any() and (calls["call"] == variants[calls["variant"]]["ref_base"]).any()


def test_abi_layout():
    assert synth.PHASE_VARIANT_DT.itemsize == 8 and synth.PHASE_CALL_DT.itemsize == 20
    assert [synth.PHASE_VARIANT_DT.fields[f][1] for f in ("ref_position", "ref_base", "alt_base", "is_snp", "reserved")] == [0, 4, 5, 6, 7]
    assert [synth.PHASE_CALL_DT.fields[f][1] for f in ("record", "variant", "ref_score", "alt_score", "call", "qual", "reserved")] == [0, 4, 8, 12, 16, 17, 18]


def test_refusals(eng, model):
    rs = synth.gen_reads(4, 1200, model, seed=9)
    ref, pairs, recs, variants, vr = synth.phase_batch(rs, seed=3, step=(30, 200), p_mismatch=0.0, p_non_snp=0.0, p_no_variants=0.0)
    deltas, first = synth.compact_event_alignment(recs, pairs, ref.shape[0])
    run = lambda **kw: eng.phase_reads_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, kw.get("recs", recs), variants,
                                             kw.get("vr", vr), calls_cap=kw.get("cap"))
    off, calls, _ = run()
    n = calls.shape[0]
    assert n > 4
    with pytest.raises(_lib.NphError, match=f"calls_cap too small: {n} calls"):
        run(cap=n - 1)
    bad = vr.copy(); bad[1] = (bad[1][1] + 1, bad[1][1])
    with pytest.raises(_lib.NphError, match="variant range"):
        run(vr=bad)
    bad = vr.copy(); bad[2][1] = variants.shape[0] + 1
    with pytest.raises(_lib.NphError, match="variant range"):
        run(vr=bad)
    r = recs.copy(); r[0]["model_id"] = 5
    with pytest.raises(_lib.NphError, match="out of range"):
        run(recs=r)
    r = recs.copy(); r[1]["ref_len"] = ref.shape[0] + 1
    with pytest.raises(_lib.NphError, match="out of range"):
        run(recs=r)
    r = recs.copy(); r[1]["read"] = rs.reads.shape[0]
    with pytest.raises(_lib.NphError, match="out of range"):
        run(recs=r)
    from nanopolish_b200.engine import Engine
    e = Engine(0)
    try:
        e.model_upload(synth.load_model("cpg"))
        r = recs.copy(); r["model_id"] = 0
        with pytest.raises(_lib.NphError, match="not a nucleotide model"):
            e.phase_reads_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, deltas, first, r, variants, vr)
    finally:
        e.close()
    # a job the scorer refuses: an event index beyond its read
    d2 = deltas.copy(); f2 = first.copy(); f2[0] = int(rs.reads[0]["n_events"]) + 5
    with pytest.raises(_lib.NphError, match="validation"):
        eng.phase_reads_batch(rs.reads, rs.ev_mean, rs.ev_start_time, ref, d2, f2, recs, variants, vr)
