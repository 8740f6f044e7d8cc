"""nanopolish polya and detect-polyi end to end through the C++ host mirror (nph::load_from_raw, then nph::PolyaBatch or
nph::DetectPolyiBatch): direct-RNA raw reads are loaded on the device, then a batch of BAM-like records (primary and secondary,
last CIGAR operations of every kind, a read missing from the index, a read whose load fails) goes through one nph_polya_batch
or nph_detect_polyi_batch call and comes back as polya_main's or detect_polyi_main's TSV.  The expected rows come from the same
chain through the oracle (oracle/prep_chain.py) and the reference's own poly(A) or detect-polyi code."""
import ctypes as C

import numpy as np
import pytest

from nanopolish_b200 import synth
from tests import host_mirror as hm
from tests import polya_cases as pc
from tests import polyi_cases as qc

pytestmark = pytest.mark.gpu
# (C shim, header line, the reference's class)
MODES = {
    "polya": ("nphh_polya", "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\tread_rate\t"
              "polya_length\tqc_tag\n", pc.RefPolya),
    "detect_polyi": ("nphh_detect_polyi", "readname\tcontig\tposition\tleader_start\tadapter_start\tpolya_start\ttranscript_start\t"
                     "read_rate\tpolya_length\tdetected\tqc_tag\n", qc.RefPolyi),
}
host = hm.fixture()


def test_polya_after_load_from_raw_like_a_caller(host, port_oracle):
    _after_load_from_raw_like_a_caller(host, port_oracle, "polya")


def test_detect_polyi_after_load_from_raw_like_a_caller(host, port_oracle):
    _after_load_from_raw_like_a_caller(host, port_oracle, "detect_polyi")


def _after_load_from_raw_like_a_caller(host, port_oracle, mode):
    from oracle.prep_chain import oracle_chain
    shim, header, ref_class = MODES[mode]
    ref = ref_class()
    m6 = synth.load_model("nucleotide")
    sd5 = m6.level_stdv.reshape(1024, 4).mean(1)
    rna = synth.PoreModel("derived.u_to_t_rna.5mer", 5, "nucleotide", m6.level_mean.reshape(1024, 4).mean(1), sd5, np.log(sd5))
    raw, rr, seqs = synth.gen_raw(5, 40000, rna, seed=433, mean_dwell=40.0, return_seqs=True)
    signals = [np.ascontiguousarray(raw[int(r["sample_off"]):int(r["sample_off"]) + int(r["n_samples"])][::-1]) for r in rr]
    # a flat signal trims to nothing: its load fails and its events stay empty
    signals.append(np.full(20000, np.float32(80.0), np.float32))
    seqs = list(seqs) + [seqs[0]]
    n = len(signals)
    rate = 3012.0
    want = oracle_chain(port_oracle, rna, signals, seqs, sample_rate=rate, rna=True)

    p = hm.p
    mean5, sd, lsd = (np.ascontiguousarray(a) for a in (rna.level_mean, rna.level_stdv, rna.level_log_stdv))
    mh = host.nphh_model_create(b"u_to_t_rna", 5, 1024, p(mean5), p(sd), p(lsd))
    assert mh >= 0, host.nphh_last_error()
    soff = np.zeros(n + 1, np.uint64); soff[1:] = np.cumsum([s.shape[0] for s in signals])
    qoff = np.zeros(n + 1, np.uint64); qoff[1:] = np.cumsum([c.shape[0] for c in seqs])
    seqbuf = b"".join(synth._CODE2DNA[c].tobytes() for c in seqs).replace(b"T", b"U")
    eoff = np.zeros(n, np.uint64); eoff[1:] = np.cumsum([s.shape[0] // 2 + 8 for s in signals])[:-1]
    room = int(eoff[-1]) + signals[-1].shape[0] // 2 + 8
    n_events = np.zeros(n, np.uint32); scal = np.zeros((n, 5)); stats = np.zeros(5, np.uint64)
    mean = np.zeros(room, np.float32); stdv = np.zeros(room, np.float32); start = np.zeros(room, np.float64); dur = np.zeros(room, np.float32)
    flat = np.ascontiguousarray(np.concatenate(signals))
    host.nphh_set_rna(1)
    try:
        first = host.nphh_load_from_raw(mh, n, p(flat), p(soff), seqbuf, p(qoff), C.c_double(rate), p(n_events), p(scal), p(eoff), p(mean),
                                        p(stdv), p(start), p(dur), None, p(stats))
    finally:
        host.nphh_set_rna(0)
    assert first >= 0, host.nphh_last_error()
    assert n_events[-1] == 0

    # records: every read once as a primary record, read 0 again as a secondary one, and a read missing from the index
    ops = [0, 4, 5, 1, 2, 0]            # last CIGAR operation: M, S, H, I, D, M
    clips = [12, 201, 200, 250, 3, 7]
    recs = []
    for i in range(n):
        recs.append((f"read{i}", "chrR", 1000 + i, 0, [(40 << 4) | 4, (900 << 4) | 0, (clips[i] << 4) | ops[i]], first + i))
    recs.insert(2, ("read0", "chrR", 5000, 0x100, [(900 << 4) | 0], first))
    recs.append(("missing", "chrR", 7, 0, [(900 << 4) | 0, (210 << 4) | 4], -1))
    m = len(recs)
    names = (C.c_char_p * m)(*[r[0].encode() for r in recs])
    contigs = (C.c_char_p * m)(*[r[1].encode() for r in recs])
    pos = np.array([r[2] for r in recs], np.int32)
    flag = np.array([r[3] for r in recs], np.uint16)
    cig = np.array([c for r in recs for c in r[4]], np.uint32)
    coff = np.zeros(m + 1, np.uint64); coff[1:] = np.cumsum([len(r[4]) for r in recs])
    handle = np.array([r[5] for r in recs], np.int32)
    sig_of = lambda r: signals[r[5] - first] if r[5] >= 0 else np.zeros(0, np.float32)
    samples = np.ascontiguousarray(np.concatenate([sig_of(r) for r in recs]))
    so = np.zeros(m + 1, np.uint64); so[1:] = np.cumsum([sig_of(r).shape[0] for r in recs])
    srate = np.full(m, rate)
    cap = 1 << 16
    buf = C.create_string_buffer(cap); need = C.c_size_t()
    got = getattr(host, shim)(m, names, contigs, p(pos), p(flag), p(cig), p(coff), p(handle), p(samples), p(so), p(srate), buf, cap, C.byref(need))
    assert got > 0, host.nphh_last_error()
    got = buf.raw[:got].decode()

    rows = [header]
    for name, contig, ps, fl, cigar, h in recs:
        if fl & 0x100:
            continue
        if h < 0:
            rows.append(ref.read(pc.PolyaRead(name, np.zeros(0, np.float32), rate, 1, 0, 1, None, None, None, contig=contig, pos=ps, loaded=False))[-1])
            continue
        w = want[h - first]
        loaded = w["events"] is not None and w.get("cal") is not None and int(w["cal"]["status"]) == 0
        r = pc.PolyaRead(name, signals[h - first], rate, float(w["cal"]["scale"]) if loaded else 1.0, float(w["cal"]["shift"]) if loaded else 0.0,
                         float(w["cal"]["var"]) if loaded else 1.0, w.get("duration"),
                         w["b2e"]["start"].astype(np.int32) if loaded else None, w["b2e"]["stop"].astype(np.int32) if loaded else None,
                         suffix_clip=cigar[-1] >> 4, contig=contig, pos=ps, loaded=loaded)
        rows.append(ref.read(r)[-1])
    assert sum(1 for w in want[:-1] if w["events"] is not None and int(w["cal"]["status"]) == 0) >= 4
    assert got == "".join(rows)
    # the secondary record has no row; the flat read and the missing one fail to load
    assert got.count("\n") == 1 + n + 1 and got.count("READ_FAILED_LOAD") == 2
