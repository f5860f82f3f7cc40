"""What flatten must produce, stated from geometry rather than from the shader arithmetic.

flatten turns every path segment (line, quad, cubic; f32 control points, an f32 affine transform and a style) into a
soup of straight lines. Everything here works in float64 from the f32 inputs of the encoded scene (`decode` reads the
path tags, path data, transforms and styles of an `Encoding`), evaluates the exact curves densely, and checks the lines
an implementation emitted (the oracle's or the GPU's `lines`) against them:

* Fills (device space; flatten transforms the control points first). With e the case's tolerance:
  - every emitted line lies within e of the exact curve, and the exact curve within e of the emitted lines (so no piece
    is missing or cut short);
  - at sample points farther than e from the curve, the winding number of the path's lines equals the exact curve's.
* Strokes (local space: a stroke is built around the untransformed centreline and then transformed, so under a
  non-uniform transform its device width varies; the emitted lines are taken back through the inverse affine, and a
  device tolerance e becomes e / s_min locally, s_min the transform's smaller singular value). With d the distance to
  the centreline and w the width:
  - every point of the exact boundary (d = w/2) lies within e of the emitted lines, so a chord that sags into a join or
    cap arc, or a piece cut short, shows; and no emitted point lies more than e outside the stroke (d > w/2 + e);
  - points with d > w/2 + e have winding number 0, points with d < w/2 - e a non-zero one (the disc-sweep rule; round
    joins and caps are exact under it);
  - the rule says nothing about the region around a join vertex or an open end of a non-round style, nor around a cusp:
    there discs of radius (w/2) max(miter limit, sqrt 2) + e are "don't care";
  - for strokes whose segments are all straight, the exact outline is a union of convex pieces, and is checked directly
    instead, both by the distances above (to the boundary of the union) and by winding numbers at every point farther
    than e from that boundary: per segment the rectangle of its butt sweep, per join the bevel triangle or the miter
    kite (up to the limit, a bevel past it) or a disc (round), per open end the half square (square cap), a disc
    (round) or nothing (butt).
* Count bound. The fewest chords that keep within tol = 0.25 px of a curve number about the integral of
  sqrt(|kappa| / (8 tol)) ds; per path the lines may be at most COUNT_FACTOR times that sum plus COUNT_PER_PIECE per
  segment side, join and cap (plus what its arcs need). A cubic that runs into flatten's SUBDIV_LIMIT emits at least
  65,536 lines, far past this.
* `classify_path` restates the formulas of flatten's Euler-spiral subdivision (in float64; arc line counts with flatten's
  f32 rounding) to report what each segment
  reached: the `robust` branch of each Euler segment (low k1, low dist_scaled, or the espc_int_approx branch and which
  of its BREAK1/2/3 pieces), the lines per Euler segment (and whether the clamp of 100 was hit), arc line counts, and
  whether a line-to fast path applies. It shows where a case falls; it never predicts the lines that are checked.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
from scipy.spatial import cKDTree

TOL = 0.25  # flatten's tolerance, device px
COUNT_FACTOR = 3.0
COUNT_PER_PIECE = 4
SQRT2 = math.sqrt(2.0)

STYLE_FLAGS_STYLE = 0x80000000
JOIN_MASK, JOIN_BEVEL, JOIN_MITER, JOIN_ROUND = 0x30000000, 0, 0x10000000, 0x20000000
CAP_BUTT, CAP_SQUARE, CAP_ROUND = 0, 1, 2


# ---- the encoded scene ---------------------------------------------------------------------------------------------------
@dataclass
class Subpath:
    segs: list = field(default_factory=list)  # (k, 2) float64 control points, k = 2 (line), 3 (quad), 4 (cubic)
    closed: bool = False


@dataclass
class PathGeom:
    index: int
    xf: tuple  # (a, b, c, d, e, f) column-major, as float64 of the f32 values
    is_stroke: bool
    width: float = 0.0
    join: int = 0
    start_cap: int = 0
    end_cap: int = 0
    miter_limit: float = 0.0
    subpaths: list = field(default_factory=list)

    @property
    def lin(self):
        a, b, c, d = self.xf[:4]
        return np.array([[a, c], [b, d]])

    def to_device(self, p):
        return p @ self.lin.T + np.array(self.xf[4:])

    def to_local(self, p):
        return (p - np.array(self.xf[4:])) @ np.linalg.inv(self.lin).T

    def singular_values(self):
        s = np.linalg.svd(self.lin, compute_uv=False)
        return float(s.min()), float(s.max())


def decode(enc) -> list:
    """The paths of an Encoding, from its tag stream: segment k of a subpath reads its p0 at the data cursor (in points),
    and the cursor moves by the segment's point count, plus one (the next move-to) at the end of a subpath. Strokes end
    every subpath with a cap marker: a quad (open) or a line (closed)."""
    from vello_b200.encoding import TAG_PATH, TAG_STYLE, TAG_SUBPATH_END_BIT, TAG_TRANSFORM, f16_to_f32
    data = np.asarray(enc.path_data, np.float32).astype(np.float64).reshape(-1, 2)
    paths, cur = [], None
    t_ix = s_ix = -1
    cursor = 0
    for tag in enc.path_tags:
        if tag == TAG_TRANSFORM:
            t_ix += 1
            continue
        if tag == TAG_STYLE:
            s_ix += 1
            continue
        if tag == TAG_PATH:
            if cur is not None:
                paths.append(cur)
            cur = None
            continue
        kind = tag & 3
        if not kind:
            continue
        assert tag & 8, "i16 path data is not produced by the encoder"
        if cur is None:
            flags, width = enc.styles[s_ix]
            xf = tuple(float(np.float32(v)) for v in enc.transforms[t_ix])
            stroke = bool(flags & STYLE_FLAGS_STYLE)
            cur = PathGeom(len(paths), xf, stroke)
            if stroke:
                cur.width = float(np.float32(width))
                cur.join = flags & JOIN_MASK
                cur.start_cap = (flags >> 26) & 3
                cur.end_cap = (flags >> 24) & 3
                cur.miter_limit = float(f16_to_f32(flags & 0xFFFF))
            cur.subpaths.append(Subpath())
        pts = data[cursor: cursor + kind + 1].copy()
        sp = cur.subpaths[-1]
        end = bool(tag & TAG_SUBPATH_END_BIT)
        if cur.is_stroke and end:
            sp.closed = kind == 1  # the cap marker: not a segment of the centreline
        elif not (pts == pts[0]).all():
            sp.segs.append(pts)
        cursor += kind + (1 if end else 0)
        if end:
            cur.subpaths.append(Subpath())
    if cur is not None:
        paths.append(cur)
    for p in paths:
        p.subpaths = [s for s in p.subpaths if s.segs]
    return paths


# ---- exact curves --------------------------------------------------------------------------------------------------------
def bez(pts, t):
    """Points of a Bezier of any degree at parameters t (de Casteljau in float64)."""
    q = np.asarray(pts, np.float64)[None]
    t = np.asarray(t, np.float64)[:, None, None]
    while q.shape[1] > 1:
        q = q[:, :-1] * (1 - t) + q[:, 1:] * t
    return np.broadcast_to(q[:, 0], (len(t), 2)).copy()


def bez_deriv(pts, t):
    n = len(pts) - 1
    return n * bez(np.diff(pts, axis=0), t)


def _n_samples(pts, spacing):
    ctrl = float(np.hypot(*np.diff(pts, axis=0).T).sum())
    return int(min(max(ctrl / spacing, 16), 4000))


def sample(pts, spacing):
    """Dense points of one segment, about `spacing` apart (at most 4,001: on the largest curves here, circles of radius
    10^6 px, the chords between them still lie within 2e-3 px of the curve), and their parameters."""
    t = np.linspace(0.0, 1.0, _n_samples(pts, spacing) + 1)
    return bez(pts, t), t


class SegSet:
    """Exact distances from points to a set of straight segments a-b. The segments are cut into pieces no longer than L
    (their median length, or longer to stay under `max_pieces`), with a k-d tree over the pieces' midpoints. The 8
    nearest pieces give an upper bound U of the distance; the nearest piece's midpoint lies within U + L/2, so every piece
    whose midpoint lies that close is then measured too. With `upto`, distances up to it are exact and larger ones are
    upper bounds (which are all that is needed of points far from the set). `widen=False` keeps the 8 nearest pieces
    only: for the dense, evenly cut samples of the exact curves, where they always hold the nearest piece, this saves
    the wider search; emitted lines, long and short mixed, always get it."""

    def __init__(self, a, b, max_pieces=3_000_000, widen=True):
        self.widen = widen
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        ln = np.hypot(*(b - a).T) if len(a) else np.zeros(0)
        piece = max(float(np.median(ln)) if len(ln) else 1.0, float(ln.sum()) / max_pieces, 1e-12)
        k = np.maximum(1, np.ceil(ln / piece)).astype(np.int64)
        idx = np.repeat(np.arange(len(a)), k)
        j = np.arange(len(idx)) - np.repeat(np.cumsum(k) - k, k)
        f0, f1 = (j / k[idx])[:, None], ((j + 1) / k[idx])[:, None]
        self.a = a[idx] + (b[idx] - a[idx]) * f0
        self.b = a[idx] + (b[idx] - a[idx]) * f1
        self.half = 0.5 * float(np.hypot(*(self.b - self.a).T).max()) if len(idx) else 0.0
        self.tree = cKDTree(0.5 * (self.a + self.b)) if len(idx) else None

    def _to(self, p, ix):
        a, b = self.a[ix], self.b[ix]
        d = b - a
        ll = (d * d).sum(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.clip(np.where(ll > 0, ((p[:, None] - a) * d).sum(-1) / ll, 0.0), 0.0, 1.0)
        q = a + u[..., None] * d
        return np.sqrt(((q - p[:, None]) ** 2).sum(-1))

    def dist(self, p, upto=np.inf):
        p = np.asarray(p, np.float64).reshape(-1, 2)
        n = len(self.a) if self.tree is not None else 0
        if not n or not len(p):
            return np.full(len(p), np.inf)
        k = min(8, n)
        _, ix = self.tree.query(p, k=k)
        out = self._to(p, ix.reshape(len(p), k)).min(1)
        # a piece whose midpoint lies r away is at least r - half away: widen the search until that cannot beat `out`
        todo, K = (np.arange(len(p)) if self.widen else np.zeros(0, np.int64)), 8
        while len(todo) and K < n:
            K = min(4 * K, n, 512)
            dd, ix = self.tree.query(p[todo], k=K)
            dd, ix = dd.reshape(len(todo), K), ix.reshape(len(todo), K)
            out[todo] = np.minimum(out[todo], self._to(p[todo], ix).min(1))
            todo = todo[(dd[:, -1] - self.half < np.minimum(out[todo], upto)) & (K < n)]
            if K == 512:
                break
        if len(todo) and self.widen:  # still more candidates: take them all
            i = todo
            lists = self.tree.query_ball_point(p[i], np.minimum(out[i], upto) + self.half)
            cnt = np.array([len(c) for c in lists], np.int64)
            if cnt.sum():
                c = np.concatenate([np.asarray(c, np.int64) for c in lists])
                who = np.repeat(i, cnt)
                d = self._to(p[who], c[:, None])[:, 0]
                np.minimum.at(out, who, d)
        return out


def winding(a, b, p):
    """Winding numbers of the closed line soup a-b at points p, by row crossings: per point, the lines crossing its row
    left of it, signed -1 for a line going down (as in the fine stage)."""
    a, b, p = np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(p, np.float64)
    out = np.zeros(len(p), np.int64)
    if not len(a) or not len(p):
        return out
    order = np.argsort(p[:, 1], kind="stable")
    ys = p[order, 1]
    ylo, yhi = np.minimum(a[:, 1], b[:, 1]), np.maximum(a[:, 1], b[:, 1])
    # rows y with ylo <= y < yhi: exactly those where (y0 <= y) != (y1 <= y)
    i0, i1 = np.searchsorted(ys, ylo, "left"), np.searchsorted(ys, yhi, "left")
    cnt = i1 - i0
    step = 20_000_000
    li = np.nonzero(cnt)[0]
    csum = np.cumsum(cnt[li])
    start = 0
    while start < len(li):
        stop = int(np.searchsorted(csum, (csum[start - 1] if start else 0) + step, "right"))
        stop = max(stop, start + 1)
        ls = li[start:stop]
        c = cnt[ls]
        line = np.repeat(ls, c)
        pt = np.repeat(i0[ls] - np.cumsum(c) + c, c) + np.arange(int(c.sum()))
        y = ys[pt]
        x0, y0, x1, y1 = a[line, 0], a[line, 1], b[line, 0], b[line, 1]
        xc = x0 + (y - y0) / (y1 - y0) * (x1 - x0)
        hit = xc < p[order[pt], 0]
        out += np.bincount(order[pt][hit], weights=np.where(y1[hit] > y0[hit], -1, 1), minlength=len(p)).astype(np.int64)
        start = stop
    return out


def path_lines(lines, pi):
    mine = lines[lines["path_ix"] == pi]
    return mine["p0"].astype(np.float64), mine["p1"].astype(np.float64)


# ---- fills ---------------------------------------------------------------------------------------------------------------
def fill_curve(path, spacing=0.05):
    """Device-space dense polylines of every subpath (each closed by the encoder), as segment end point arrays."""
    A, B = [], []
    for sp in path.subpaths:
        for s in sp.segs:
            q, _ = sample(path.to_device(s), spacing)
            A.append(q[:-1])
            B.append(q[1:])
    return np.concatenate(A), np.concatenate(B)


def _grid(lo, hi, n, rng):
    gx = lo[0] + (hi[0] - lo[0]) * (np.arange(n) + rng.uniform(0.1, 0.9, n)) / n
    gy = lo[1] + (hi[1] - lo[1]) * (np.arange(n) + rng.uniform(0.1, 0.9, n)) / n
    return np.stack(np.meshgrid(gx, gy), -1).reshape(-1, 2)


def _near_band(a, b, offsets, n_max=6000):
    """Points at the given normal offsets from a subsample of the polyline a-b's vertices."""
    sel = np.unique(np.linspace(0, len(a) - 1, min(n_max, len(a))).astype(np.int64))
    d = b[sel] - a[sel]
    ln = np.hypot(*d.T)
    ok = ln > 0
    nrm = np.stack([-d[ok, 1], d[ok, 0]], 1) / ln[ok, None]
    base = 0.5 * (a[sel][ok] + b[sel][ok])
    return np.concatenate([base + o * nrm for o in offsets]) if len(base) else np.zeros((0, 2))


def check_fill(path, lines, eps, grid=160, seed=0):
    """Assert the fill contract for one path; returns the measured distances (lines to curve, curve to lines) and the
    number of winding samples checked."""
    a, b = path_lines(lines, path.index)
    assert len(a), f"path {path.index}: no lines"
    ca, cb = fill_curve(path)
    curve = SegSet(ca, cb, widen=False)
    emitted = SegSet(a, b)
    # lines -> curve, at 5 points of every line; curve -> lines at every curve sample
    f = np.array([0.0, 0.25, 0.5, 0.75, 1.0])[None, :, None]
    on_lines = (a[:, None] + (b - a)[:, None] * f).reshape(-1, 2)
    d_lc = curve.dist(on_lines, upto=2 * eps)
    d_cl = emitted.dist(np.concatenate([ca, cb[-1:]]), upto=2 * eps)
    worst_lc, worst_cl = float(d_lc.max()), float(d_cl.max())
    k = int(np.argmax(d_lc))
    assert worst_lc <= eps, f"path {path.index}: an emitted point {on_lines[k]} is {worst_lc:.4g} px from the curve (eps {eps})"
    k = int(np.argmax(d_cl))
    assert worst_cl <= eps, f"path {path.index}: the curve at {ca[min(k, len(ca) - 1)]} is {worst_cl:.4g} px from every line (eps {eps})"
    rng = np.random.default_rng(seed)
    lo, hi = np.minimum(ca.min(0), a.min(0)) - 4 * eps - 1, np.maximum(ca.max(0), a.max(0)) + 4 * eps + 1
    pts = np.concatenate([_grid(lo, hi, grid, rng), _near_band(ca, cb, (-3 * eps, -1.5 * eps, 1.5 * eps, 3 * eps))])
    far = curve.dist(pts, upto=2 * eps) > eps
    pts = pts[far]
    got, want = winding(a, b, pts), winding(ca, cb, pts)
    bad = got != want
    if bad.any():
        k = int(np.argmax(bad))
        raise AssertionError(f"path {path.index}: {int(bad.sum())} of {len(pts)} samples farther than {eps} px from the curve "
                             f"have another winding number, first at {pts[k]}: lines {int(got[k])}, curve {int(want[k])}")
    return dict(lines_to_curve=worst_lc, curve_to_lines=worst_cl, samples=len(pts))


# ---- strokes -------------------------------------------------------------------------------------------------------------
def _unit(v):
    return v / np.hypot(*v)


def _start_tangent(s):
    for k in range(1, len(s)):
        if (s[k] != s[0]).any():
            return _unit(s[k] - s[0])
    return np.array([1.0, 0.0])


def _end_tangent(s):
    for k in range(len(s) - 2, -1, -1):
        if (s[k] != s[-1]).any():
            return _unit(s[-1] - s[k])
    return np.array([1.0, 0.0])


def _cusps(s, scale):
    """Parameters of a cubic where its speed nearly vanishes (a cusp), as points."""
    if len(s) < 4:
        return []
    t = np.linspace(0.0, 1.0, 4001)
    v = np.hypot(*bez_deriv(s, t).T)
    thr = 1e-3 * max(scale, 1e-300)
    out = []
    for k in np.nonzero((v < thr))[0]:
        if 0 < t[k] < 1 and v[k] <= v[max(k - 1, 0)] and v[k] <= v[min(k + 1, len(t) - 1)]:
            out.append(bez(s, t[k:k + 1])[0])
    return out


def _convex_sd(poly, p):
    """max over the edges of a convex polygon (either orientation) of the signed distance to the edge line: < 0 inside
    (and then minus the exact depth), > 0 outside (and then at most the exact distance)."""
    poly = np.asarray(poly, np.float64)
    e = np.roll(poly, -1, 0) - poly
    area = (poly[:, 0] * np.roll(poly[:, 1], -1) - np.roll(poly[:, 0], -1) * poly[:, 1]).sum()
    nrm = np.stack([e[:, 1], -e[:, 0]], 1) * (1 if area > 0 else -1)
    ln = np.hypot(*nrm.T)
    keep = ln > 0
    nrm = nrm[keep] / ln[keep, None]
    return ((p[:, None] - poly[keep][None]) * nrm[None]).sum(-1).max(1)


def _miter_ok(t0, t1, limit):
    """flatten.wgsl's miter condition, exactly: 2 |t0||t1| < (|t0||t1| + t0.t1) limit^2, with a turn."""
    cr, d = t0[0] * t1[1] - t0[1] * t1[0], t0 @ t1
    hyp = math.hypot(cr, d)
    return 2 * hyp < (hyp + d) * limit * limit and abs(cr) > 1e-12


def outline_pieces(path):
    """For a stroke whose segments are all straight: its outline as (convex polygons, discs (centre, radius))."""
    h = 0.5 * path.width
    polys, discs = [], []
    for sp in path.subpaths:
        segs = [(s[0], s[-1]) for s in sp.segs]
        for a, b in segs:
            n = _unit(b - a)
            n = np.array([-n[1], n[0]]) * h
            polys.append([a + n, b + n, b - n, a - n])
        verts = list(range(len(segs) if sp.closed else len(segs) - 1))
        for k in verts:
            (a0, v), (_, b1) = segs[k], segs[(k + 1) % len(segs)]
            t0, t1 = _unit(v - a0), _unit(b1 - v)
            n0, n1 = np.array([-t0[1], t0[0]]) * h, np.array([-t1[1], t1[0]]) * h
            if path.join == JOIN_ROUND:
                discs.append((v, h))
                continue
            polys.append([v, v + n0, v + n1])
            polys.append([v, v - n0, v - n1])
            if path.join == JOIN_MITER and _miter_ok(t0, t1, path.miter_limit):
                cr = t0[0] * t1[1] - t0[1] * t1[0]
                s = -1.0 if cr > 0 else 1.0  # the outer side
                # the corner where the two offset lines meet
                p0, p1 = v + s * n0, v + s * n1
                m = np.linalg.solve(np.stack([t0, -t1], 1), p1 - p0)
                polys.append([v, p0, p0 + m[0] * t0, p1])
        if not sp.closed:
            for pt, tan, cap in ((segs[0][0], -_unit(segs[0][1] - segs[0][0]), path.start_cap),
                                 (segs[-1][1], _unit(segs[-1][1] - segs[-1][0]), path.end_cap)):
                n = np.array([-tan[1], tan[0]]) * h
                if cap == CAP_SQUARE:
                    polys.append([pt + n, pt + n + h * tan, pt - n + h * tan, pt - n])
                elif cap == CAP_ROUND:
                    discs.append((pt, h))
    return polys, discs


def check_stroke(path, lines, eps, grid=128, seed=0, exact_outline=None):
    """Assert the stroke contract for one path (module docstring) with device tolerance `eps`; returns what was
    measured, in local px times s_min (the units of `eps`): `boundary_to_lines`, the largest distance from a point of the
    exact boundary to the emitted lines, and `lines_outside`, how far the farthest emitted point lies outside the stroke;
    and the sample counts."""
    a_dev, b_dev = path_lines(lines, path.index)
    assert len(a_dev), f"path {path.index}: no lines"
    a, b = path.to_local(a_dev), path.to_local(b_dev)
    s_min, s_max = path.singular_values()
    e = eps / s_min
    h = 0.5 * path.width
    spacing = min(0.05 / s_max, max(h, 1e-9) / 4)
    A, B, care_c = [], [], []
    R = h * max(path.miter_limit if path.join == JOIN_MITER else 0.0, SQRT2) + e
    ends = []
    for sp in path.subpaths:
        for s in sp.segs:
            q, _ = sample(s, spacing)
            A.append(q[:-1])
            B.append(q[1:])
            care_c += _cusps(s, float(np.abs(np.diff(s, axis=0)).max()))
        if path.join != JOIN_ROUND:
            vs = [s[-1] for s in sp.segs[:-1]] + ([sp.segs[-1][-1]] if sp.closed else [])
            care_c += vs
        if not sp.closed:
            ends += [(sp.segs[0][0], path.start_cap), (sp.segs[-1][-1], path.end_cap)]
    care_c += [p for p, cap in ends if cap != CAP_ROUND]
    ca, cb = np.concatenate(A), np.concatenate(B)
    centre = SegSet(ca, cb, widen=False)
    straight = all(len(s) == 2 for sp in path.subpaths for s in sp.segs)
    if exact_outline is None:
        exact_outline = straight
    rng = np.random.default_rng(seed)
    lo, hi = ca.min(0) - R - 2 * e, ca.max(0) + R + 2 * e
    offs = [0.0] + [sg * (h + k * e) for sg in (-1, 1) for k in (-3, -1.5, 1.5, 3)]
    pts = [_grid(lo, hi, grid, rng), _near_band(ca, cb, offs)]
    for c in care_c:  # polar grids around every don't-care centre: the join / cap shapes are checked there
        r = np.linspace(0.05, 1.0, 24)[:, None] * (R + 2 * e)
        th = np.linspace(0, 2 * np.pi, 96, endpoint=False)[None] + 0.013
        pts.append(np.stack([c[0] + r * np.cos(th), c[1] + r * np.sin(th)], -1).reshape(-1, 2))
    # rings just inside and outside w/2 around every vertex and end: where round joins and caps put their arcs
    n_th = int(min(4000, max(96, 2 * np.pi * h / (4 * spacing))))
    th = np.linspace(0, 2 * np.pi, n_th, endpoint=False)[None] + 0.007
    r = np.array([h - 3 * e, h - 1.5 * e, h + 1.5 * e, h + 3 * e])[:, None]
    for sp in path.subpaths:
        for c in [sp.segs[0][0]] + [s[-1] for s in sp.segs]:
            pts.append(np.stack([c[0] + r * np.cos(th), c[1] + r * np.sin(th)], -1).reshape(-1, 2))
    pts = np.concatenate(pts)
    wind = winding(a, b, pts)
    rep = dict(samples=len(pts))
    polys, discs = outline_pieces(path) if exact_outline else ([], [])
    if exact_outline:
        sd = np.full(len(pts), np.inf)
        for poly in polys:
            sd = np.minimum(sd, _convex_sd(poly, pts))
        for c, r in discs:
            sd = np.minimum(sd, np.hypot(*(pts - c).T) - r)
        inside, outside = sd < -e, sd > e
        rep["checked"] = int((inside | outside).sum())
    else:
        d = centre.dist(pts, upto=h + 2 * e)
        care = np.ones(len(pts), bool)
        if care_c:
            cc = np.asarray(care_c)
            care = cKDTree(cc).query(pts)[0] > R
        inside, outside = care & (d < h - e), care & (d > h + e)
        rep["checked"] = int((inside | outside).sum())
    # distances: the exact boundary must lie within e of the lines (a chord that sags into a join or cap arc, or a piece
    # cut short, shows here), and no emitted point may lie more than e outside the stroke
    emitted = SegSet(a, b)
    f = np.array([0.0, 0.25, 0.5, 0.75])[None, :, None]
    on = (a[:, None] + (b - a)[:, None] * f).reshape(-1, 2)
    if exact_outline:
        edge = []
        for poly in polys:
            q = np.asarray(poly, np.float64)
            for u, v in zip(q, np.roll(q, -1, 0)):
                k = int(min(4000, max(8, np.hypot(*(v - u)) / spacing)))
                edge.append(u + (v - u) * (np.arange(k) / k)[:, None])
        for c, r in discs:
            k = int(min(20000, max(96, 2 * np.pi * r / spacing)))
            t = np.arange(k) * (2 * np.pi / k)
            edge.append(np.stack([c[0] + r * np.cos(t), c[1] + r * np.sin(t)], 1))
        edge = np.concatenate(edge)

        def sd_union(q):
            out = np.full(len(q), np.inf)
            for poly in polys:
                out = np.minimum(out, _convex_sd(poly, q))
            for c, r in discs:
                out = np.minimum(out, np.hypot(*(q - c).T) - r)
            return out
        # on the union's boundary: some point a hair away is outside every piece (a point on a shared edge, such as a
        # join vertex on the end of a segment's rectangle, is interior)
        step = 1e-3 * e
        out_near = np.zeros(len(edge), bool)
        for th in np.arange(8) * (np.pi / 4) + 0.1:
            out_near |= sd_union(edge + step * np.array([np.cos(th), np.sin(th)])) > 0
        edge = edge[out_near]
        outside_by = sd_union(on)
    else:
        edge = _near_band(ca, cb, (-h, h), n_max=20000)
        if path.join == JOIN_ROUND or CAP_ROUND in (path.start_cap, path.end_cap):
            t = np.linspace(0, 2 * np.pi, n_th, endpoint=False) + 0.003
            ring = np.stack([h * np.cos(t), h * np.sin(t)], 1)
            edge = np.concatenate([edge] + [c + ring for sp in path.subpaths for c in [sp.segs[0][0]] + [s[-1] for s in sp.segs]])
        edge = edge[centre.dist(edge, upto=2 * h) >= h * (1 - 1e-9) - 1e-9]  # on the boundary of the disc sweep
        outside_by = centre.dist(on, upto=h + 2 * e) - h
        if care_c:
            tree = cKDTree(np.asarray(care_c))
            edge = edge[tree.query(edge)[0] > R]
            outside_by = outside_by[tree.query(on)[0] > R]
    gap = emitted.dist(edge, upto=2 * e) if len(edge) else np.zeros(1)
    rep["boundary_to_lines"] = float(gap.max()) * s_min
    rep["lines_outside"] = float(max(outside_by.max(), 0.0)) * s_min if len(outside_by) else 0.0
    k = int(np.argmax(gap))
    assert gap.max() <= e, f"path {path.index}: the stroke's boundary at local {edge[k]} is {gap.max():.4g} local px from " \
                           f"every line (band {e:.3g})"
    assert rep["lines_outside"] <= eps, f"path {path.index}: an emitted point lies {rep['lines_outside']:.4g} px outside the stroke"
    bad_in = inside & (wind == 0)
    bad_out = outside & (wind != 0)
    for bad, what in ((bad_in, "inside the stroke have winding 0"), (bad_out, "outside the stroke have a winding number")):
        if bad.any():
            k = int(np.argmax(bad))
            raise AssertionError(f"path {path.index}: {int(bad.sum())} of {len(pts)} samples {what}, first at local "
                                 f"{pts[k]} (band {e:.3g} local px, {'exact outline' if exact_outline else 'disc sweep'})")
    return rep


# ---- count bound ---------------------------------------------------------------------------------------------------------
def _min_chords(q):
    """sum over a dense polyline q of sqrt(|d theta| ds / (8 tol)): the integral of sqrt(|kappa| / (8 tol)) ds."""
    d = np.diff(q, axis=0)
    ln = np.hypot(*d.T)
    keep = ln > 0
    d, ln = d[keep], ln[keep]
    if len(d) < 2:
        return 0.0
    th = np.arctan2(d[:, 1], d[:, 0])
    dth = np.abs((np.diff(th) + np.pi) % (2 * np.pi) - np.pi)
    ds = 0.5 * (ln[1:] + ln[:-1])
    return float(np.sqrt(dth * ds / (8 * TOL)).sum())


def _arc_lines(angle, r_dev):
    """Lines of an arc of `angle` at device radius r_dev: ceil(angle / theta), theta = 2 acos(1 - tol / r), with
    1 - tol / r, the angle and the quotient rounded to f32 as flatten rounds them (at r = 10^6 px the f32 rounding of
    1 - tol / r alone takes the half turn from 2,222 lines to 2,276)."""
    f = np.float32
    x = f(1) - f(f(TOL) / f(max(r_dev, TOL)))
    theta = max(f(1e-4), f(2) * f(math.acos(float(x))))
    return max(1, math.ceil(float(f(f(angle) / theta))))


def count_bound(path):
    """The most lines a path may have (module docstring)."""
    total, pieces = 0.0, 0
    arcs = 0
    if not path.is_stroke:
        for sp in path.subpaths:
            for s in sp.segs:
                q, _ = sample(path.to_device(s), 0.05)
                total += _min_chords(q)
                pieces += 1
        return COUNT_FACTOR * total + COUNT_PER_PIECE * pieces
    h = 0.5 * path.width
    _, s_max = path.singular_values()
    for sp in path.subpaths:
        for s in sp.segs:
            q, t = sample(s, 0.05 / s_max)
            tan = bez_deriv(s, t)
            ln = np.hypot(*tan.T)
            ok = ln > 0
            nrm = np.zeros_like(tan)
            nrm[ok] = np.stack([-tan[ok, 1], tan[ok, 0]], 1) / ln[ok, None]
            for sg in (1, -1):
                total += _min_chords(path.to_device(q + sg * h * nrm))
            pieces += 2 + 1  # two sides and a join or a cap
        n_ends = len(sp.segs) + (0 if sp.closed else 1)
        arcs += n_ends * _arc_lines(math.pi, s_max * h)
    return COUNT_FACTOR * total + COUNT_PER_PIECE * pieces + (arcs if path.join == JOIN_ROUND or
                                                                   CAP_ROUND in (path.start_cap, path.end_cap) else 0)


# ---- classifier ----------------------------------------------------------------------------------------------------------
BREAK1, BREAK2, BREAK3 = 0.8, 1.25, 2.1


def _espc_piece(x):
    y = abs(x)
    return "sin" if y < BREAK1 else "pow" if y < BREAK2 else "quad1" if y < BREAK3 else "quad2"


def _cubic_params(p0, p1, q0, q1, dt):
    chord = p1 - p0
    c2 = chord @ chord
    if c2 < 1e-12:
        return 0.0, 0.0, 1e-6, math.sqrt((9 / 32) * (q0 @ q0 + q1 @ q1)) * dt
    scale = dt / c2
    h0 = np.array([q0 @ chord, q0[1] * chord[0] - q0[0] * chord[1]])
    h1 = np.array([q1 @ chord, q1[0] * chord[1] - q1[1] * chord[0]])
    th0, th1 = math.atan2(h0[1], h0[0]), math.atan2(h1[1], h1[0])
    d0, d1 = math.hypot(*h0) * scale, math.hypot(*h1) * scale
    s0, c0, s1, c1 = math.sin(th0), math.cos(th0), math.sin(th1), math.cos(th1)
    err = 2.0
    if c0 * c1 >= 0:
        e0, e1 = (2 / 3) / max(1 + c0, 1e-9), (2 / 3) / max(1 + c1, 1e-9)
        s01 = c0 * s1 + c1 * s0
        amin = 0.15 * (2 * e0 * s0 + 2 * e1 * s1 - e0 * e1 * s01)
        a = 0.15 * (2 * d0 * s0 + 2 * d1 * s1 - d0 * d1 * s01)
        symm, asymm = abs(th0 + th1), abs(th0 - th1)
        dist = math.hypot(d0 - e0, d1 - e1)
        err = (4.625e-6 * symm ** 3 + 7.5e-3 * asymm) * symm ** 2 + 1.55 * abs(a - amin) + (5e-3 * symm + 7e-2 * asymm) * dist
    return th0, th1, math.sqrt(c2), err * math.sqrt(c2)


def _euler_params(th0, th1):
    k0, dth = th0 + th1, th1 - th0
    d2, k2 = dth * dth, (th0 + th1) ** 2
    a = 6.0 - d2 / 70 - d2 * d2 / 10780 + d2 ** 3 * 2.769178184818219e-07
    b = -0.1 + d2 / 4200 + d2 * d2 * 1.6959677820260655e-05
    c = -1 / 1400 + d2 * 6.84915970574303e-05 - k2 * 7.936475029053326e-06
    a += (b + c * k2) * k2
    ch = 1.0 - d2 / 40 + d2 * d2 * 0.00034226190482569864 - d2 ** 3 * 1.9349474568904524e-06
    b_ = -1 / 24 + d2 * 0.0024702380951963226 - d2 * d2 * 3.7297408997537985e-05
    c_ = 1 / 1920 - d2 * 4.87350869747975e-05 - k2 * 3.1001936068463107e-06
    ch += (b_ + c_ * k2) * k2
    return k0, dth * a, ch


def _espc_int(x):
    y = abs(x)
    if y < BREAK1:
        a = math.sin(1.0976991822760038 * y) / 1.0976991822760038
    elif y < BREAK2:
        a = (math.sqrt(8) / 3) * (y - 1) * math.sqrt(abs(y - 1)) + math.pi / 4
    else:
        qa, qb, qc = (0.6406, -0.81, 0.9148117935952064) if y < BREAK3 else (0.5, -0.156, 0.16145779359520596)
        a = (qa * y + qb) * y + qc
    return math.copysign(a, x) if x else 0.0


def _euler_segments(c, offset, scale):
    """flatten's subdivision of one cubic c (in the space it flattens in) into Euler segments: per segment its branch,
    espc pieces, unclamped line count and clamped count."""
    def ev(t):
        return bez(c, np.array([t]))[0], bez_deriv(c, np.array([t]))[0] / 3.0
    out = []
    t0_u, dt, last_t = 0, 1.0, 0.0
    last_p, last_q = c[0], c[1] - c[0]
    deriv = False
    if last_q @ last_q < 1e-12:
        last_q = ev(1e-6)[1]
        deriv = True
    while t0_u * dt != 1.0 and len(out) < 70000:
        t1 = t0_u * dt + dt
        p1, q1 = ev(t1)
        if q1 @ q1 < 1e-12:
            deriv = True
            pn, qn = ev(t1 - 1e-6)
            q1 = qn
            if t1 < 1.0:
                p1, t1 = pn, t1 - 1e-6
        th0, th1, chord_len, err = _cubic_params(last_p, p1, last_q, q1, t1 - last_t)
        if err * scale <= TOL or dt <= 1.0 / 65536:
            k0_, k1, ch = _euler_params(th0, th1)
            k0 = k0_ - 0.5 * k1
            dist_scaled = offset / chord_len * ch
            mult = math.sqrt(0.125 * scale * chord_len / (ch * TOL))
            rec = dict(subdiv_limit=dt <= 1.0 / 65536 and err * scale > TOL, deriv_thresh=deriv,
                       tiny_chord=float((p1 - last_p) @ (p1 - last_p)) < 1e-12)
            if abs(k1) < 1e-3:
                rec["branch"] = "k1"
                n_frac = math.sqrt(abs(k0_ * (k0_ * dist_scaled + 1)))
            elif abs(dist_scaled) < 1e-3:
                rec["branch"] = "dist"
                integral = (k1 + k0) * math.sqrt(abs(k1 + k0)) - k0 * math.sqrt(abs(k0))
                n_frac = (2 / 3) * integral / k1
            else:
                a = -2 * dist_scaled * k1
                b = -1 - 2 * dist_scaled * k0
                rec["branch"] = "espc"
                rec["pieces"] = (_espc_piece(b), _espc_piece(a + b))
                k_peak = k0 - k1 * b / a
                n_frac = (_espc_int(a + b) - _espc_int(b)) * math.sqrt(abs(k_peak * (k_peak * dist_scaled + 1))) / a
            want = math.ceil(n_frac * mult) if math.isfinite(n_frac * mult) else 10 ** 9
            rec["n_want"], rec["n"] = want, min(max(want, 1), 100)
            rec["clamped"] = want > 100
            out.append(rec)
            last_p, last_q, last_t = p1, q1, t1
            t0_u += 1
            while t0_u % 2 == 0:
                t0_u //= 2
                dt *= 2
        else:
            t0_u *= 2
            dt *= 0.5
    return out


def _as_cubic(s):
    if len(s) == 2:
        return np.array([s[0], s[0] + (s[1] - s[0]) / 3, s[1] + (s[0] - s[1]) / 3, s[1]])
    if len(s) == 3:
        return np.array([s[0], s[1] + (s[0] - s[1]) / 3, s[1] + (s[2] - s[1]) / 3, s[2]])
    return s


def classify_path(path):
    """What the path's segments reach in flatten (module docstring): a dict of
    euler: list of per-Euler-segment records (branch, pieces, n_want, n, clamped, subdiv_limit, deriv_thresh: a
    derivative below DERIV_THRESH was replaced, tiny_chord: a chord below DERIV_THRESH),
    arcs: line counts of the arcs of round joins and caps, fast: how many segments take a line-to fast path,
    flags: a set of segment kinds (seg:line|quad|cubic), joins (join:bevel|miter|miter-bevel|round, miter-bevel being a
    miter join past its limit), caps (cap:butt|square|round), "closed", "tangent_fallback" (a segment shorter than
    TANGENT_THRESH, whose tangent flatten replaces), "mirror" (det < 0) and "non_uniform" (unequal singular values)."""
    out = dict(euler=[], arcs=[], fast=0, flags=set())
    flags = out["flags"]
    s_min, s_max = path.singular_values()
    if np.linalg.det(path.lin) < 0:
        flags.add("mirror")
    if s_max > s_min * (1 + 1e-6):
        flags.add("non_uniform")
    names = {JOIN_BEVEL: "bevel", JOIN_MITER: "miter", JOIN_ROUND: "round"}
    caps = {CAP_BUTT: "butt", CAP_SQUARE: "square", CAP_ROUND: "round"}
    h = 0.5 * path.width
    for sp in path.subpaths:
        if path.is_stroke:
            if sp.closed:
                flags.add("closed")
            else:
                flags |= {"cap:" + caps[path.start_cap], "cap:" + caps[path.end_cap]}
        for k, s in enumerate(sp.segs):
            flags.add("seg:" + {2: "line", 3: "quad", 4: "cubic"}[len(s)])
            if path.is_stroke and float(((s[1:] - s[0]) ** 2).sum(1).max()) < 1e-12:
                flags.add("tangent_fallback")
            if path.is_stroke and (k + 1 < len(sp.segs) or sp.closed):
                t0, t1 = _end_tangent(s), _start_tangent(sp.segs[(k + 1) % len(sp.segs)])
                jn = names[path.join]
                flags.add("join:" + ("miter-bevel" if jn == "miter" and not _miter_ok(t0, t1, path.miter_limit) else jn))
            if not path.is_stroke:
                dev = path.to_device(s)
                if len(s) == 2 and np.abs(dev).max() < 65536:
                    out["fast"] += 1
                    continue
                out["euler"] += _euler_segments(_as_cubic(dev), 0.0, 1.0)
                continue
            if len(s) == 2 and _stroke_line_fast(path, s):
                out["fast"] += 1
            else:
                for sg in (1, -1):
                    out["euler"] += _euler_segments(_as_cubic(s), sg * h, s_max)
            last = k == len(sp.segs) - 1
            if last and not sp.closed:
                if path.end_cap == CAP_ROUND:
                    out["arcs"].append(_arc_lines(3.1415927, float(np.hypot(*(path.lin @ (_end_tangent(s) * h))))))
            else:
                nxt = sp.segs[(k + 1) % len(sp.segs)]
                t0, t1 = _end_tangent(s), _start_tangent(nxt)
                if path.join == JOIN_ROUND:
                    ang = abs(math.atan2(t0[0] * t1[1] - t0[1] * t1[0], t0 @ t1))
                    out["arcs"].append(_arc_lines(ang, float(np.hypot(*(path.lin @ (np.array([-t0[1], t0[0]]) * h))))))
        if not sp.closed and path.start_cap == CAP_ROUND:
            t = _start_tangent(sp.segs[0])
            out["arcs"].append(_arc_lines(3.1415927, float(np.hypot(*(path.lin @ (t * h))))))
    return out


def _stroke_line_fast(path, s):
    """k_flatten's guard of its stroked line-to fast path (evaluated in float64)."""
    chord = s[1] - s[0]
    c2 = float(chord @ chord)
    mag = float(np.abs(s).max())
    s1 = float(np.abs(path.lin).sum())
    u = mag * 2.0 ** -22
    off = 0.5 * path.width
    return off > 0 and mag * s1 < 16384.0 and c2 >= 256 * u * u and c2 >= u * off and 1e-10 <= c2 < 1e30
