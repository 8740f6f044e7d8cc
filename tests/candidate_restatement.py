"""A plain-Python walk of AlignmentDB::get_variants_in_region (src/alignment/nanopolish_alignment_db.cpp:259-368): per record, in
record order, the depth range and the walk from lower_bound(start) to lower_bound(stop), then the merge on (position, ref_seq,
alt_seq).  A record without a pair at or after start adds nothing (the reference dereferences end() there)."""
import bisect


def instances(region_ref: str, region_start: int, bases: bytes, aligned, start: int, stop: int):
    """(depth range or None, [(ref_position, ref_seq, alt_seq)]) of one record; aligned: (ref_pos, read_pos) pairs"""
    ap = [(int(a), int(b)) for a, b in aligned]
    if not ap:
        return None, []
    refs = [a for a, _ in ap]
    si, ei = bisect.bisect_left(refs, start), bisect.bisect_left(refs, stop)
    if si == len(ap):
        return None, []
    ds = max(ap[si][0], start)
    de = min(ap[-1][0] if ei == len(ap) else ap[ei][0], stop)
    rb = lambda p: region_ref[p[0] - region_start]
    qb = lambda p: chr(bases[p[1]])
    out = []
    i = si
    while i != ei:
        mismatch = rb(ap[i]) != qb(ap[i])
        nx = i + 1
        gap = nx != ei and (ap[nx][0] != ap[i][0] + 1 or ap[nx][1] != ap[i][1] + 1)
        if gap:
            while nx != ei and rb(ap[nx]) != qb(ap[nx]):
                nx += 1
        if nx != ei and (mismatch or gap) and ap[nx][0] < stop - 1:
            out.append((ap[i][0], region_ref[ap[i][0] - region_start:ap[nx][0] - region_start], bases[ap[i][1]:ap[nx][1]].decode("latin-1")))
        i = nx
    return (ds, de), out


def distinct(region_ref: str, region_start: int, bases_list, aligned_list, start: int, stop: int):
    """{(ref_position, ref_seq, alt_seq): (count, depth)} over every record"""
    assert stop >= start
    depth = [0] * (stop - start + 1)
    counts = {}
    for b, a in zip(bases_list, aligned_list):
        rng, inst = instances(region_ref, region_start, b, a, start, stop)
        if rng is not None:
            for p in range(rng[0], rng[1]):
                depth[p - start] += 1
        for v in inst:
            counts[v] = counts.get(v, 0) + 1
    return {v: (c, depth[v[0] - start]) for v, c in counts.items()}


def kept(dist: dict, min_frequency: float, min_depth: int):
    """the variants the reference's filter keeps, in its std::map key order ("contig:pos:ref:alt" compared bytewise; the contig
    is common), with their INFO counts"""
    out = []
    for (p, r, a), (c, d) in sorted(dist.items(), key=lambda kv: f"{kv[0][0]}:{kv[0][1]}:{kv[0][2]}".encode("latin-1")):
        if (c / d if d else (float("inf") if c else float("nan"))) >= min_frequency and d >= min_depth:
            out.append((p, r, a, c, d))
    return out
