"""A numpy statement of the parallel decision rule k_device_paths.cu applies to curved rings (vb_fragment_from_device_curves),
for the CPU tests to hold against the host PathEncoder before any GPU run. Per ring of points P and kinds K (0 on-curve, 1
off-curve; a valid ring starts and ends on-curve with at most two off-curve points in a row):

- every on-curve point e after the first ends a segment whose start is the on-curve point before it, e - degree;
- the first kept segment is the lowest one with a point EPS-far from P[0] (the start-tangent tests, no sequential dependency);
- a later segment is kept when the EPS span of its start and its points exceeds EPS in x or y (the span against its own
  start, not the last kept end point);
- the ring is walked in order, with the span against the last kept end point, when some segment after the first kept one
  fails the span test while ending unequal in value to its start (`walk`).

`encode` writes the tag bytes and path-data words these decisions give, in the kernels' order, for a fill or a stroke."""
import numpy as np

EPS = 1e-12
TAG_LINE, TAG_QUAD, TAG_PATH, SUBPATH_END = 0x09, 0x0A, 0x10, 0x04
f32 = np.float32


def neq(p, q):
    d = np.abs(np.asarray(p, f32) - np.asarray(q, f32))
    return bool(d[0] > EPS or d[1] > EPS)


def span_keeps(at, pts):
    """is_zero_length_segment, negated: the span of `at` and `pts` ((k, 2) float32) exceeds EPS in x or y."""
    a = np.vstack([np.asarray(at, f32)[None], pts])
    s = a.max(0) - a.min(0)
    return bool(s[0] > EPS or s[1] > EPS)


def ring_rule(P, K):
    """(keep per on-curve end point {e: bool}, first, last, degree per end point, walk) of one ring by the parallel rule; first
    is None for a ring that keeps nothing."""
    P = np.asarray(P, f32).reshape(-1, 2)
    on = np.flatnonzero(np.asarray(K) == 0)
    ends = on[1:]
    deg = {int(e): int(e - s) for s, e in zip(on[:-1], on[1:])}
    # each point after the first belongs to the segment of the next on-curve point at or after it
    seg_end = on[np.searchsorted(on, np.arange(1, len(P)))]
    tangent = np.array([neq(P[j], P[0]) for j in range(1, len(P))], bool)
    firsts = seg_end[tangent]
    if firsts.size == 0:
        return {}, None, None, deg, False
    first = int(firsts.min())
    span = {int(e): span_keeps(P[e - deg[e]], P[e - deg[e] + 1:e + 1]) for e in ends}
    odd = {e: not span[e] and not (P[e] == P[e - deg[e]]).all() for e in span}
    walk = any(odd[e] for e in odd if e > first)
    keep = {e: e == first or (e > first and span[e]) for e in span}
    if walk:  # the encoders' order: the span against the last kept end point
        at = P[first]
        for e in ends:
            if e > first:
                keep[int(e)] = span_keeps(at, P[e - deg[e] + 1:e + 1])
                if keep[int(e)]:
                    at = P[e]
    last = max(e for e in keep if keep[e])
    return keep, first, last, deg, walk


def start_tangent_end(P, first, degree):
    P = np.asarray(P, f32).reshape(-1, 2)
    p0, e = P[0], P[first]
    third = f32(1.0) / f32(3.0)
    if degree == 1:
        return p0 + third * (e - p0)
    if degree == 2:
        c = P[first - 1]
        return c + third * (p0 - c) if neq(c, p0) else c + third * (e - c)
    c1, c2 = P[first - 2], P[first - 1]
    return c1 if neq(c1, p0) else (c2 if neq(c2, p0) else e)


def encode(pts, kinds, roff, poff, stroke, closed):
    """(tag bytes, path-data words as float32, walked rings) of the rule for every path, without the TRANSFORM and STYLE
    tags: what the kernels write after them."""
    pts = np.asarray(pts, f32).reshape(-1, 2)
    tags, data, walked = [], [], []
    closes = closed or not stroke
    n_paths = len(poff) - 1
    for i in range(n_paths):
        path_kept = False
        for r in range(poff[i], poff[i + 1]):
            b0, b1 = int(roff[r]), int(roff[r + 1])
            if b0 == b1:
                continue
            P, K = pts[b0:b1], np.asarray(kinds[b0:b1])
            keep, first, last, deg, walk = ring_rule(P, K)
            if walk:
                walked.append(r)
            if first is None:
                continue
            path_kept = True
            ste = start_tangent_end(P, first, deg[first])
            p0, pl = P[0], P[last]
            tail = []
            if closes and (p0.view(np.uint32) != pl.view(np.uint32)).any():
                tail.append((TAG_LINE, [p0]))
            if stroke:
                if closes:
                    if neq(ste, p0):
                        tail.append((TAG_LINE, [ste]))
                elif span_keeps(pl, np.stack([p0, ste])):
                    tail.append((TAG_QUAD, [p0, ste]))
            ring_tags = []
            data.extend(P[0])
            for j in range(1, len(P)):
                e = j if K[j] == 0 else j + (1 if K[j + 1] == 0 else 2)
                if keep[e]:
                    data.extend(P[j])
                    if j == e:
                        ring_tags.append(TAG_LINE + deg[e] - 1)
            for t, ps in tail:
                ring_tags.append(t)
                for p in ps:
                    data.extend(p)
            ring_tags[-1] |= SUBPATH_END
            tags += ring_tags
        if path_kept:
            tags.append(TAG_PATH)
    return tags, np.array(data, f32), walked


def elements(pts, kinds, b0, b1):
    """The element list of one ring: M, then L / Q / C per on-curve point after the first (without the Z)."""
    els = [("M", float(pts[b0][0]), float(pts[b0][1]))]
    ctl = []
    for j in range(b0 + 1, b1):
        if kinds[j]:
            ctl += [float(pts[j][0]), float(pts[j][1])]
            continue
        els.append(("LQC"[len(ctl) // 2], *ctl, float(pts[j][0]), float(pts[j][1])))
        ctl = []
    return els


def points_of(els):
    """(points, kinds, ring_offsets) of an element list of M / L / Q / C / Z (shapes.path_elements): one ring per M. A Z adds
    nothing; a curved closing segment already ends on a repeat of the first point."""
    pts, kinds, roff = [], [], [0]
    for el in els:
        k = el[0]
        if k == "M":
            if len(pts) > roff[-1]:
                roff.append(len(pts))
            pts.append(el[1:3])
            kinds.append(0)
        elif k in "LQC":
            v = el[1:]
            for m in range(0, len(v), 2):
                pts.append(v[m:m + 2])
                kinds.append(0 if m == len(v) - 2 else 1)
    if len(pts) > roff[-1]:
        roff.append(len(pts))
    return np.array(pts, np.float64).reshape(-1, 2), np.array(kinds, np.uint8), np.array(roff, np.int32)
