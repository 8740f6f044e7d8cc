"""TEST INFRASTRUCTURE ONLY.  The load_from_raw chain through the ORACLE: trim -> detect_events -> SquiggleEvent conversion
-> MoM -> ABEA -> base_to_event_map / recalibration, in the order src/nanopolish_squiggle_read.cpp:226-336 runs them."""
import numpy as np

from nanopolish_b200 import synth


def squiggle_events(ev, sample_rate):
    """events -> (duration f32, start_time f64) as squiggle_read.cpp:243-250 computes them (sequential double sum)."""
    dur = (ev["length"].astype(np.float64) / sample_rate).astype(np.float32)
    t = np.concatenate([[0.0], np.cumsum(dur.astype(np.float64))[:-1]]) if ev.shape[0] else np.zeros(0)   # cumsum folds left to right
    return dur, t


def oracle_chain(port, model, signals, seqs, sample_rate=4000.0, rna=False, params=None):
    """Returns per read a dict: events (EVENT_DT), duration, start_time, and — when the read got that far — mom, cal
    (CALIBRATION_DT record), b2e, n_pairs.  rna: scrappie's RNA detector parameters, the MoM estimate on the events in
    acquisition order, then the events turned around to 5'->3' before ABEA (squiggle_read.cpp:204-213,237-240,262-265).
    params: an EVENT_PARAMS_DT record to use instead, whose reverse_events says whether the events are turned around."""
    prm = synth.event_params(rna) if params is None else params
    rna = bool(prm[0]["reverse_events"])
    out = []
    for x, codes in zip(signals, seqs):
        r = {"events": None}
        ok, s, e = port.trim_raw(x)
        out.append(r)
        r["range"] = (s, e) if ok else (0, 0)
        if not ok:
            continue
        ev = port.detect_events(np.ascontiguousarray(x[s:e]), prm)
        r["events"] = ev
        r["duration"], r["start_time"] = squiggle_events(ev, sample_rate)
        reads = np.zeros(1, synth.READ_DT)
        reads[0] = (0, ev.shape[0], 0, 1.0, 0.0, 0.0, 1.0, 0.0, 0.0)
        rs = synth.ReadSet(reads, np.ascontiguousarray(ev["mean"]), r["start_time"], [codes], [None], [None], model.k)
        jobs, ranks, total = synth.abea_jobs(rs)
        sh, sc = port.mom(rs.reads, rs.ev_mean, model, ranks, jobs[0])
        if rna:
            ev = r["events"] = np.ascontiguousarray(ev[::-1])
            r["duration"], r["start_time"] = np.ascontiguousarray(r["duration"][::-1]), np.ascontiguousarray(r["start_time"][::-1])
            rs = synth.ReadSet(reads, np.ascontiguousarray(ev["mean"]), r["start_time"], [codes], [None], [None], model.k)
        reads[0]["shift"], reads[0]["scale"] = sh, sc
        r["mom"] = (sh, sc)
        pairs, res, _ = port.abea_batch(rs.reads, rs.ev_mean, rs.ev_start_time, model, ranks, jobs, total)
        r["n_pairs"] = int(res[0]["n_pairs"])
        r["b2e"], r["cal"] = port.recalibrate(rs.reads, rs.ev_mean, model, ranks, jobs[0], pairs, r["n_pairs"])
    return out
