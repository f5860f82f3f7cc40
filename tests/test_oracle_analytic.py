"""Analytic ground truth for the oracle (and, through the GPU parity tests, for the CUDA path), independent of the restated
shader code: what the pixels SHOULD be by geometry and by the W3C compositing definitions.

The reference's golden images pin fills, one circle, linear gradients and nearest images only (DESIGN.md section 4). These
tests tie the rows the goldens do not reach -- partial MSAA coverage, sloped edges, strokes, clips, the 16 mix modes and 14
Porter-Duff operators, radial and sweep gradients, luminance masks -- to first principles:

* area AA of a simple polygon == the exact area of polygon n pixel (sloped edges: 1.5 LSB; axis-aligned edges inside a pixel
  go through fine.wgsl's `xmin - 1e-6` division, whose f32 rounding is worth up to 7 % of a pixel: a property of the
  reference's formula, asserted loosely);
* MSAA8 / MSAA16: the sample patterns are n-rooks, so an axis-aligned edge at k/n of a pixel covers exactly k/n; sloped
  edges are the LUT-quantised half planes, asserted within 2 samples of the exact area;
* a stroke's total coverage == width x length (+ the caps' area);
* a clipped fill == clip coverage x fill coverage;
* every blend mode == the W3C `Compositing and Blending Level 1` formula evaluated in float64 by blend_ref.py (restated
  from the specification text, not from blend.wgsl), within 2 LSB at a few colour pairs (test_blend_ref.py checks every
  branch of the same formulas exactly, over 65536 pairs per mode);
* radial / sweep gradients == the ramp colour at the analytically computed parameter.
"""
import math

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16
from vello_b200.encoding import (BLACK, COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_NORMAL, STYLE_CAP_BUTT, STYLE_CAP_ROUND,
                                 STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, TRANSPARENT, Color, Gradient, Scene, Stroke, resolve)
from vello_b200.shapes import Affine, BezPath, Line, Rect

from .blend_ref import MIXES, w3c_composite

WHITE = Color.from_rgba8(255, 255, 255)


def render(oracle, scene, w, h, aa, base=BLACK):
    return oracle.render(resolve(scene.encoding), w, h, base.premul_rgba8_u32(), aa)


def coverage(oracle, shape, w, h, aa, rule=FILL_NON_ZERO):
    """White `shape` on black: the red channel / 255 is the coverage the rasteriser assigned to each pixel."""
    s = Scene()
    s.fill(rule, Affine.IDENTITY, WHITE, None, shape)
    return render(oracle, s, w, h, aa)[..., 0].astype(np.float64) / 255.0


# ---- exact polygon-pixel intersection areas (Sutherland-Hodgman against the four pixel edges) ------------------------------
def _clip_poly(poly, axis, bound, keep_less):
    out = []
    n = len(poly)
    for i in range(n):
        a, b = poly[i], poly[(i + 1) % n]
        ina = (a[axis] <= bound) if keep_less else (a[axis] >= bound)
        inb = (b[axis] <= bound) if keep_less else (b[axis] >= bound)
        if ina:
            out.append(a)
        if ina != inb:
            t = (bound - a[axis]) / (b[axis] - a[axis])
            out.append((a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1])))
    return out


def _area(poly):
    return 0.5 * abs(sum(poly[i][0] * poly[(i + 1) % len(poly)][1] - poly[(i + 1) % len(poly)][0] * poly[i][1] for i in range(len(poly))))


def exact_coverage(poly, w, h):
    cov = np.zeros((h, w))
    xs = [p[0] for p in poly]
    ys = [p[1] for p in poly]
    for y in range(max(0, int(math.floor(min(ys)))), min(h, int(math.ceil(max(ys))))):
        for x in range(max(0, int(math.floor(min(xs)))), min(w, int(math.ceil(max(xs))))):
            p = _clip_poly(poly, 0, x, False)
            p = _clip_poly(p, 0, x + 1, True) if p else p
            p = _clip_poly(p, 1, y, False) if p else p
            p = _clip_poly(p, 1, y + 1, True) if p else p
            cov[y, x] = _area(p) if len(p) >= 3 else 0.0
    return cov


def poly_path(poly):
    p = BezPath()
    p.move_to(*poly[0])
    for q in poly[1:]:
        p.line_to(*q)
    p.close_path()
    return p


def random_convex(rng, cx, cy, r, n):
    ang = np.sort(rng.uniform(0, 2 * math.pi, n))
    rad = rng.uniform(0.6 * r, r, n)
    return [(float(cx + rad[i] * math.cos(ang[i])), float(cy + rad[i] * math.sin(ang[i]))) for i in range(n)]


# ---- coverage ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_area_aa_of_sloped_polygons_is_the_exact_area(oracle, seed):
    rng = np.random.default_rng(seed)
    poly = random_convex(rng, 24.3, 23.1, 19.0, int(rng.integers(3, 9)))
    got = coverage(oracle, poly_path(poly), 48, 48, AA_AREA)
    want = exact_coverage(poly, 48, 48)
    assert np.abs(got - want).max() <= 1.5 / 255 + 1e-6, np.abs(got - want).max()


def test_area_aa_of_a_concave_even_odd_star(oracle):
    # a pentagram under the even-odd rule: the inner pentagon is a hole; compare the TOTAL area (pixelwise the self-
    # intersections make area AA approximate: two edges of one path in one pixel)
    pts = [(24 + 20 * math.sin(2 * math.pi * k * 2 / 5), 24 - 20 * math.cos(2 * math.pi * k * 2 / 5)) for k in range(5)]
    eo = coverage(oracle, poly_path(pts), 48, 48, AA_AREA, FILL_EVEN_ODD).sum()
    nz = coverage(oracle, poly_path(pts), 48, 48, AA_AREA, FILL_NON_ZERO).sum()
    r = 20.0
    outer = 5 * r * r * math.sin(math.radians(36)) * math.sin(math.radians(18)) / math.sin(math.radians(126))  # area of the {5/2} star's hull of points
    inner_r = r * math.sin(math.radians(18)) / math.sin(math.radians(126))
    pentagon = 2.5 * inner_r * inner_r * math.sin(math.radians(72))
    assert abs(nz - outer) / outer < 0.01
    assert abs(eo - (outer - pentagon)) / outer < 0.01


def test_area_aa_of_axis_aligned_edges(oracle):
    got = coverage(oracle, Rect(3.25, 2.5, 10.75, 9.125), 16, 16, AA_AREA)
    xs = np.arange(16)
    cx = np.clip(np.minimum(xs + 1, 10.75) - np.maximum(xs, 3.25), 0, 1)
    cy = np.clip(np.minimum(xs + 1, 9.125) - np.maximum(xs, 2.5), 0, 1)
    # the vertical edges go through `(..) / (xmax - xmin)` with xmin = x - 1e-6 in f32 (fine.wgsl:1046-1052)
    assert np.abs(got - np.outer(cy, cx)).max() <= 0.07
    assert np.abs(got - np.outer(cy, cx))[:, 4:10].max() <= 1.0 / 255  # columns without a vertical edge: exact


@pytest.mark.parametrize("aa,n", [(AA_MSAA8, 8), (AA_MSAA16, 16)])
def test_msaa_patterns_are_n_rooks(oracle, aa, n):
    """An axis-aligned edge at k/n of a pixel covers exactly k of the n samples, horizontally and vertically."""
    for k in range(n + 1):
        f = k / n
        got = coverage(oracle, Rect(2.0 + f, 1.0, 9.0, 7.0), 12, 8, aa)
        assert got[3, 2] == pytest.approx(round(255 * (1 - f)) / 255, abs=1e-9), (k, got[3, 2])
        assert (got[3, 3:9] == 1.0).all() and got[3, 1] == 0.0
        got = coverage(oracle, Rect(2.0, 1.0 + f, 9.0, 7.0), 12, 8, aa)
        assert got[1, 4] == pytest.approx(round(255 * (1 - f)) / 255, abs=1e-9), (k, got[1, 4])


@pytest.mark.parametrize("aa,n", [(AA_MSAA8, 8), (AA_MSAA16, 16)])
@pytest.mark.parametrize("seed", range(3))
def test_msaa_of_sloped_polygons_is_near_the_exact_area(oracle, aa, n, seed):
    rng = np.random.default_rng(100 + seed)
    poly = random_convex(rng, 24.3, 23.1, 19.0, int(rng.integers(3, 9)))
    got = coverage(oracle, poly_path(poly), 48, 48, aa)
    want = exact_coverage(poly, 48, 48)
    # every value is a whole number of samples
    assert np.abs(got * 255 - np.round(np.round(got * n) / n * 255)).max() <= 0.5
    assert np.abs(got - want).max() <= 2.0 / n + 1e-3
    assert abs(got.sum() - want.sum()) / want.sum() < 0.01


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
def test_stroke_coverage_is_width_times_length(oracle, aa):
    def total(stroke, shape):
        s = Scene()
        s.stroke(stroke, Affine.IDENTITY, WHITE, None, shape)
        return render(oracle, s, 64, 64, aa)[..., 0].astype(np.float64).sum() / 255.0
    line = Line(10.3, 12.6, 50.8, 41.2)
    length = math.hypot(50.8 - 10.3, 41.2 - 12.6)
    w = 5.0
    tol = 0.012 if aa == AA_AREA else 0.02
    assert abs(total(Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), line) - w * length) / (w * length) < tol
    sq = w * length + w * w
    assert abs(total(Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_SQUARE, end_cap=STYLE_CAP_SQUARE), line) - sq) / sq < tol
    rd = w * length + math.pi * (w / 2) ** 2
    assert abs(total(Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_ROUND, end_cap=STYLE_CAP_ROUND), line) - rd) / rd < tol


def test_clip_is_the_product_of_coverages(oracle):
    clip, rect = Rect(4.5, 3.25, 20.5, 14.75), Rect(8.0, 1.0, 30.0, 12.5)
    s = Scene()
    s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, clip)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, WHITE, None, rect)
    s.pop_layer()
    got = render(oracle, s, 32, 16, AA_MSAA16)[..., 0].astype(np.float64) / 255
    a = coverage(oracle, clip, 32, 16, AA_MSAA16)
    b = coverage(oracle, rect, 32, 16, AA_MSAA16)
    assert np.abs(got - a * b).max() <= 1.5 / 255


# ---- W3C compositing and blending: the float64 restatement of the specification lives in blend_ref.py -------------------
def _blend_scene(mix, compose, backdrop: Color, source: Color, layer_alpha=1.0):
    s = Scene()
    r = Rect(0.0, 0.0, 16.0, 16.0)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, backdrop, None, r)
    s.push_layer(FILL_NON_ZERO, mix, compose, layer_alpha, Affine.IDENTITY, r)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, source, None, r)
    s.pop_layer()
    return s


def _unpremul8(px):
    return px.astype(np.float64) / 255.0


BLEND_COLOURS = [(Color.from_rgba8(200, 90, 40, 255), Color.from_rgba8(30, 160, 220, 255)),
                 (Color.from_rgba8(200, 90, 40, 255), Color.from_rgba8(30, 160, 220, 140)),
                 (Color.from_rgba8(64, 220, 130, 180), Color.from_rgba8(240, 70, 200, 110)),
                 (Color.from_rgba8(20, 40, 230, 90), Color.from_rgba8(250, 240, 30, 255))]


def _channels(c: Color):
    return [c.r, c.g, c.b], c.a


@pytest.mark.parametrize("mix", range(16))
def test_mix_modes_match_the_w3c_formulas(oracle, mix):
    for backdrop, source in BLEND_COLOURS:
        img = render(oracle, _blend_scene(mix, COMPOSE_SRC_OVER, backdrop, source), 16, 16, AA_AREA, TRANSPARENT)
        cb, ab = _channels(backdrop)
        cs, as_ = _channels(source)
        want = w3c_composite(mix, COMPOSE_SRC_OVER, cb, ab, cs, as_)
        got = _unpremul8(img[8, 8])
        a = want[3]
        want_stored = [want[i] / a if a > 0 else 0.0 for i in range(3)] + [a]  # the target stores separated alpha
        assert np.abs(got - np.clip(want_stored, 0, 1)).max() <= 2.5 / 255, (MIXES[mix], got * 255, np.array(want_stored) * 255)
        assert (img == img[8, 8]).all()  # flat everywhere


@pytest.mark.parametrize("compose", range(14))
@pytest.mark.parametrize("mix", [0, 1, 15])
def test_compose_operators_match_porter_duff(oracle, compose, mix):
    for backdrop, source in BLEND_COLOURS:
        img = render(oracle, _blend_scene(mix, compose, backdrop, source), 16, 16, AA_AREA, TRANSPARENT)
        cb, ab = _channels(backdrop)
        cs, as_ = _channels(source)
        want = w3c_composite(mix, compose, cb, ab, cs, as_)
        a = want[3]
        got = _unpremul8(img[8, 8])
        assert abs(got[3] - a) <= 2.0 / 255, (compose, got[3] * 255, a * 255)
        if a > 0.02:  # colour of a (nearly) transparent pixel is not meaningful after the division
            tol = 2.5 / 255 / max(a, 0.25)
            assert np.abs(got[:3] - np.clip([want[i] / a for i in range(3)], 0, 1)).max() <= tol, (compose, mix, got * 255, want)


def test_layer_alpha_and_luminance_mask(oracle):
    backdrop, source = Color.from_rgba8(200, 90, 40, 255), Color.from_rgba8(30, 160, 220, 255)
    img = render(oracle, _blend_scene(MIX_NORMAL, COMPOSE_SRC_OVER, backdrop, source, 0.4), 16, 16, AA_AREA, TRANSPARENT)
    want = [0.4 * s + 0.6 * b for s, b in zip((30, 160, 220), (200, 90, 40))]
    assert np.abs(img[8, 8, :3].astype(np.float64) - want).max() <= 1.5 and img[8, 8, 3] == 255
    # luminance mask (scene.rs:208-236): the backdrop is multiplied by the layer's luminance (sRGB coefficients) x alpha
    s = Scene()
    r = Rect(0.0, 0.0, 16.0, 16.0)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, backdrop, None, r)
    s.push_luminance_mask_layer(FILL_NON_ZERO, 1.0, Affine.IDENTITY, r)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, source, None, r)
    s.pop_layer()
    img = render(oracle, s, 16, 16, AA_AREA, TRANSPARENT)
    lum = 0.2125 * 30 / 255 + 0.7154 * 160 / 255 + 0.0721 * 220 / 255
    # premultiplied backdrop x lum, stored with separated alpha: colour unchanged, alpha = lum
    assert abs(int(img[8, 8, 3]) - 255 * lum) <= 1.5
    assert np.abs(img[8, 8, :3].astype(np.float64) - (200, 90, 40)).max() <= 2.0


# ---- gradients ------------------------------------------------------------------------------------------------------------------
def _lerp_colour(c0, c1, t):
    return np.array([c0[i] + (c1[i] - c0[i]) * t for i in range(3)])


def test_radial_and_sweep_gradients_follow_their_parameter(oracle):
    c0, c1 = (255, 32, 16), (16, 64, 255)
    stops = [(0.0, Color.from_rgba8(*c0)), (1.0, Color.from_rgba8(*c1))]
    r = Rect(0.0, 0.0, 64.0, 64.0)
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.radial((32.0, 32.0), 0.0, (32.0, 32.0), 30.0, stops), None, r)
    img = render(oracle, s, 64, 64, AA_AREA).astype(np.float64)
    ys, xs = np.mgrid[0:64, 0:64]
    t = np.clip(np.hypot(xs - 32.0, ys - 32.0) / 30.0, 0, 1)  # gradients are evaluated at the pixel's integer coordinates (fine.wgsl:1283)
    want = np.stack([c0[i] + (c1[i] - c0[i]) * t for i in range(3)], axis=-1)
    assert np.abs(img[..., :3] - want).max() <= 2.0
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.sweep((32.0, 32.0), 0.0, 2 * math.pi, stops), None, r)
    img = render(oracle, s, 64, 64, AA_AREA).astype(np.float64)
    ang = np.arctan2(ys - 32.0, xs - 32.0)
    t = np.where(ang < 0, ang + 2 * math.pi, ang) / (2 * math.pi)
    want = np.stack([c0[i] + (c1[i] - c0[i]) * t for i in range(3)], axis=-1)
    far = np.hypot(xs - 32.0, ys - 32.0) > 3  # the parameter is discontinuous at the centre and along the seam
    seam = (np.abs(ys - 32.0) < 1.5) & (xs >= 32)
    ok = far & ~seam
    # the shader's atan2 is a degree-7 polynomial (fine.wgsl:1346-1366): 1e-3 of a turn
    assert np.abs(img[..., :3] - want)[ok].max() <= 2.5


# ---- joins, curves ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("join", ["bevel", "miter", "round"])
@pytest.mark.parametrize("phi_deg", [35.0, 90.0, 130.0])
def test_join_area(oracle, join, phi_deg):
    """Two segments meeting at exterior angle phi, butt caps. Union area = w (L1 + L2) - inner overlap + join wedge, with the
    inner overlap a kite of (w/2)^2 tan(phi/2) and the wedge a triangle (bevel), a sector (round) or the same kite (miter)."""
    from vello_b200.encoding import STYLE_JOIN_MITER, STYLE_JOIN_ROUND
    w, l1, l2 = 8.0, 60.0, 55.0
    phi = math.radians(phi_deg)
    p0 = (20.0, 100.0)
    p1 = (p0[0] + l1, p0[1])
    p2 = (p1[0] + l2 * math.cos(phi), p1[1] - l2 * math.sin(phi))
    path = BezPath([("M",) + p0, ("L",) + p1, ("L",) + p2])
    jn = {"bevel": STYLE_JOIN_BEVEL, "miter": STYLE_JOIN_MITER, "round": STYLE_JOIN_ROUND}[join]
    s = Scene()
    s.stroke(Stroke(w, join=jn, miter_limit=10.0, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), Affine.IDENTITY, WHITE, None, path)
    got = render(oracle, s, 160, 160, AA_AREA)[..., 0].astype(np.float64).sum() / 255
    h = w / 2
    kite = h * h * math.tan(phi / 2)
    wedge = {"bevel": 0.5 * h * h * math.sin(phi), "round": 0.5 * h * h * phi, "miter": kite}[join]
    want = w * (l1 + l2) - kite + wedge
    assert abs(got - want) / want < 0.004, (got, want)


def _cubic_area(p0, p1, p2, p3):
    """Signed area contribution  1/2 * integral (x dy - y dx)  of one cubic Bezier (closed form, from the Bernstein products)."""
    x0, y0 = p0; x1, y1 = p1; x2, y2 = p2; x3, y3 = p3
    return (x0 * (6 * y1 + 3 * y2 + y3) + 3 * x1 * (-2 * y0 + y2 + y3) + 3 * x2 * (-y0 - y1 + 2 * y3) - x3 * (y0 + 3 * y1 + 6 * y2)) / 20.0


def test_flattened_curves_keep_their_area(oracle):
    """flatten's Euler-spiral subdivision replaces a curve by chords no further than the tolerance (0.25 px) from the spiral, so
    for arcs (which the spiral fits exactly) the rendered area differs from the closed form by at most 2/3 x perimeter x
    tolerance (a chord of sagitta e cuts off 2/3 e x its length) and the chords lie inside; for general cubics the spiral fit
    may use another `tol`, and every point of every emitted line stays within 2 tol of the true curve."""
    from vello_b200.shapes import Circle, Ellipse
    tol = 0.25
    got = coverage(oracle, Circle(40.3, 39.6, 30.0), 80, 80, AA_AREA).sum()
    loss = math.pi * 900.0 - got
    assert -1.0 <= loss <= (2.0 / 3.0) * 2 * math.pi * 30.0 * tol, loss
    a_, b_ = 33.0, 14.0
    got = coverage(oracle, Ellipse(40.3, 39.6, a_, b_, 0.6), 80, 80, AA_AREA).sum()
    perim = math.pi * (3 * (a_ + b_) - math.sqrt((3 * a_ + b_) * (a_ + 3 * b_)))  # Ramanujan
    loss = math.pi * a_ * b_ - got
    assert -1.0 <= loss <= (2.0 / 3.0) * perim * tol, loss
    rng = np.random.default_rng(5)
    for _ in range(4):
        # a closed loop of 4 cubics around a centre (simple, no self-intersection: control points stay in their angular sector)
        k = 4
        ang = np.linspace(0, 2 * math.pi, k + 1)
        pts = []
        for i in range(k):
            a0, a1 = ang[i], ang[i + 1]
            r = rng.uniform(22, 34, 4)
            aa = [a0, a0 + (a1 - a0) / 3, a0 + 2 * (a1 - a0) / 3, a1]
            pts.append([(50 + r[j] * math.cos(aa[j]), 50 + r[j] * math.sin(aa[j])) for j in range(4)])
        for i in range(k):  # make it closed and continuous
            pts[i][3] = pts[(i + 1) % k][0]
        path = BezPath([("M",) + pts[0][0]] + [("C",) + pts[i][1] + pts[i][2] + pts[i][3] for i in range(k)] + [("Z",)])
        want = abs(sum(_cubic_area(*pts[i]) for i in range(k)))
        ts = np.linspace(0, 1, 2001)
        curve = []
        for q in pts:
            bern = ((1 - ts) ** 3, 3 * (1 - ts) ** 2 * ts, 3 * (1 - ts) * ts ** 2, ts ** 3)
            curve.append(np.stack([sum(c * q[j][0] for j, c in enumerate(bern)), sum(c * q[j][1] for j, c in enumerate(bern))], -1))
        curve = np.concatenate(curve)
        perim = float(np.hypot(np.diff(curve[:, 0]), np.diff(curve[:, 1])).sum())
        got = coverage(oracle, path, 100, 100, AA_AREA).sum()
        # a general cubic has two error terms of `tol` each: the Euler-spiral fit (flatten.wgsl:420-450) and the chords
        assert abs(got - want) <= (2.0 / 3.0) * perim * 2 * tol, (got, want, perim)
        lines = oracle.buffer("lines")[:int(oracle.buffer("bump")["lines"][0])]
        assert 8 <= len(lines) <= 64
        for ln in lines:
            for f in (0.0, 0.25, 0.5, 0.75):
                m = ln["p0"] * (1 - f) + ln["p1"] * f
                assert np.sqrt(((curve - m) ** 2).sum(1).min()) <= 2 * tol + 0.01


# ---- images ----------------------------------------------------------------------------------------------------------------------
def _img(rng, h, w):
    d = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    d[..., 3] = 255
    return d


def test_image_nearest_is_texel_replication(oracle):
    from vello_b200.encoding import Image, QUALITY_LOW
    rng = np.random.default_rng(9)
    d = _img(rng, 5, 7)
    s = Scene()
    s.draw_image(Image(d, quality=QUALITY_LOW), Affine.scale(4.0))
    got = render(oracle, s, 28, 20, AA_AREA)
    assert np.array_equal(got, np.repeat(np.repeat(d, 4, axis=0), 4, axis=1))


def _mitchell(x, b=1.0 / 3.0, c=1.0 / 3.0):
    """Mitchell-Netravali reconstruction filter (Mitchell & Netravali 1988), the kernel fine.wgsl's bicubic uses with B = C = 1/3."""
    x = abs(x)
    if x < 1:
        return ((12 - 9 * b - 6 * c) * x ** 3 + (-18 + 12 * b + 6 * c) * x ** 2 + (6 - 2 * b)) / 6
    if x < 2:
        return ((-b - 6 * c) * x ** 3 + (6 * b + 30 * c) * x ** 2 + (-12 * b - 48 * c) * x + (8 * b + 24 * c)) / 6
    return 0.0


def test_image_bilinear_and_bicubic_reconstruction(oracle):
    from vello_b200.encoding import Image, QUALITY_HIGH, QUALITY_MEDIUM
    rng = np.random.default_rng(10)
    d = _img(rng, 6, 8)
    f = d.astype(np.float64)
    scale = 3.0
    H, W = int(6 * scale), int(8 * scale)

    def texel(ix, iy):  # pad extend
        return f[min(max(iy, 0), 5), min(max(ix, 0), 7)]

    for quality in (QUALITY_MEDIUM, QUALITY_HIGH):
        s = Scene()
        s.draw_image(Image(d, quality=quality), Affine.scale(scale))
        got = render(oracle, s, W, H, AA_AREA).astype(np.float64)
        want = np.zeros((H, W, 4))
        for y in range(H):
            for x in range(W):
                u, v = (x + 0.5) / scale, (y + 0.5) / scale  # image-space position of the pixel centre
                if quality == QUALITY_MEDIUM:
                    uu, vv = u - 0.5, v - 0.5
                    x0, y0 = math.floor(uu), math.floor(vv)
                    fx, fy = uu - x0, vv - y0
                    want[y, x] = ((1 - fy) * ((1 - fx) * texel(x0, y0) + fx * texel(x0 + 1, y0))
                                  + fy * ((1 - fx) * texel(x0, y0 + 1) + fx * texel(x0 + 1, y0 + 1)))
                else:
                    uu, vv = u - 0.5, v - 0.5
                    x0, y0 = math.floor(uu), math.floor(vv)
                    acc = np.zeros(4)
                    for j in range(-1, 3):
                        for i in range(-1, 3):
                            acc += _mitchell(uu - (x0 + i)) * _mitchell(vv - (y0 + j)) * texel(x0 + i, y0 + j)
                    want[y, x] = np.clip(acc, 0, 255)
        tol = 1.5 if quality == QUALITY_MEDIUM else 2.5
        assert np.abs(got - want).max() <= tol, (quality, np.abs(got - want).max())


# ---- gradient extend modes and the two-point radial kinds ------------------------------------------------------------------------------
def test_linear_gradient_extend_modes(oracle):
    from vello_b200.encoding import EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT
    c0, c1 = np.array([255.0, 32.0, 16.0]), np.array([16.0, 64.0, 255.0])
    stops = [(0.0, Color.from_rgba8(255, 32, 16)), (1.0, Color.from_rgba8(16, 64, 255))]
    xs = np.arange(128, dtype=np.float64)
    t = (xs - 40.0) / 24.0  # gradient line from x = 40 to x = 64, evaluated at integer pixel coordinates
    for ext, tt in ((EXTEND_PAD, np.clip(t, 0, 1)), (EXTEND_REPEAT, t - np.floor(t)), (EXTEND_REFLECT, np.abs(t - 2 * np.round(0.5 * t)))):
        s = Scene()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((40.0, 0.0), (64.0, 0.0), stops, ext), None, Rect(0.0, 0.0, 128.0, 8.0))
        got = render(oracle, s, 128, 8, AA_AREA)[4, :, :3].astype(np.float64)
        want = c0[None, :] + (c1 - c0)[None, :] * tt[:, None]
        # at the wrap of `repeat` the 512-entry ramp index jumps: skip the pixels within one ramp step of a discontinuity
        ok = np.ones(128, bool) if ext != EXTEND_REPEAT else (np.abs(tt - 0.5) < 0.49)
        assert np.abs(got - want)[ok].max() <= 2.0, (ext, np.abs(got - want)[ok].max())


@pytest.mark.parametrize("c0,r0,c1,r1", [((40.0, 48.0), 6.0, (56.0, 48.0), 40.0),    # one circle inside the other
                                         ((30.0, 48.0), 10.0, (70.0, 48.0), 10.0),   # strip (equal radii)
                                         ((30.0, 48.0), 4.0, (64.0, 50.0), 22.0)])   # cone, circles apart
def test_two_point_radial_gradient(oracle, c0, r0, c1, r1):
    """Two-point conical gradient (the HTML canvas / PDF definition): the colour at p is the stop at the LARGEST t with
    |p - c(t)| = r(t), r(t) >= 0, c(t) = c0 + t (c1 - c0), r(t) = r0 + t (r1 - r0); pixels with no solution stay unpainted."""
    col0, col1 = np.array([250.0, 40.0, 20.0]), np.array([10.0, 90.0, 240.0])
    stops = [(0.0, Color.from_rgba8(250, 40, 20)), (1.0, Color.from_rgba8(10, 90, 240))]
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.radial(c0, r0, c1, r1, stops), None, Rect(0.0, 0.0, 96.0, 96.0))
    got = render(oracle, s, 96, 96, AA_AREA, TRANSPARENT).astype(np.float64)
    cdx, cdy, dr = c1[0] - c0[0], c1[1] - c0[1], r1 - r0
    a = cdx * cdx + cdy * cdy - dr * dr
    checked = 0
    for y in range(0, 96, 3):
        for x in range(0, 96, 3):
            px, py = x - c0[0], y - c0[1]
            b = px * cdx + py * cdy + r0 * dr
            c = px * px + py * py - r0 * r0
            ts = []
            if abs(a) < 1e-9:
                if abs(b) > 1e-9:
                    ts = [c / (2 * b)]
            else:
                disc = b * b - a * c
                if disc >= 0:
                    ts = [(b + math.sqrt(disc)) / a, (b - math.sqrt(disc)) / a]
            ts = [t for t in ts if r0 + t * dr >= 0]
            if not ts:
                if abs(a) >= 1e-9 and b * b - a * c < -40.0:  # clearly outside the cone: nothing is painted
                    assert got[y, x, 3] == 0, (x, y)
                continue
            t = max(ts)
            # stay away from the parameter's discontinuities (cone boundary, the focal point) where one pixel decides
            if abs(a) >= 1e-9 and b * b - a * c < 40.0:
                continue
            want = col0 + (col1 - col0) * min(max(t, 0.0), 1.0)
            assert got[y, x, 3] == 255 and np.abs(got[y, x, :3] - want).max() <= 3.0, (x, y, t, got[y, x], want)
            checked += 1
    assert checked > 150


# ---- blurred rounded rectangle ---------------------------------------------------------------------------------------------------------
def test_blurred_rounded_rect_is_a_gaussian_blur_of_the_shape(oracle):
    """scene.rs:256-314 / fine.wgsl:1290-1330 approximate (closed form, no convolution) the Gaussian blur of a rounded
    rectangle. Ground truth: the 4x supersampled rounded rectangle convolved with a Gaussian by scipy. The approximation is
    documented as visually close, not exact: 4 % of full scale, and the total light within 1 %. The edge profile of the
    reference is erf(x / std_dev) (fine.wgsl:1217), i.e. the Gaussian of the comparison has sigma = std_dev / sqrt(2)."""
    from scipy.ndimage import gaussian_filter
    w, h, radius, sigma = 60.0, 36.0, 9.0, 5.0
    size = 128
    s = Scene()
    s.draw_blurred_rounded_rect(Affine.translate(64.0, 64.0), Rect(-w / 2, -h / 2, w / 2, h / 2), WHITE, radius, sigma)
    got = render(oracle, s, size, size, AA_AREA)[..., 0].astype(np.float64) / 255
    ss = 4
    ys, xs = (np.mgrid[0:size * ss, 0:size * ss] + 0.5) / ss
    qx, qy = np.abs(xs - 64.0) - (w / 2 - radius), np.abs(ys - 64.0) - (h / 2 - radius)
    d = np.hypot(np.maximum(qx, 0), np.maximum(qy, 0)) + np.minimum(np.maximum(qx, qy), 0) - radius
    mask = (d <= 0).astype(np.float64)
    blurred = gaussian_filter(mask, sigma / math.sqrt(2.0) * ss, mode="constant")
    # the shader evaluates at integer pixel coordinates: sample the truth there (supersample index x * ss)
    want = blurred[::ss, ::ss]
    want = 0.25 * (blurred[np.ix_(np.arange(size) * ss, np.arange(size) * ss)] + blurred[np.ix_(np.maximum(np.arange(size) * ss - 1, 0), np.arange(size) * ss)]
                   + blurred[np.ix_(np.arange(size) * ss, np.maximum(np.arange(size) * ss - 1, 0))]
                   + blurred[np.ix_(np.maximum(np.arange(size) * ss - 1, 0), np.maximum(np.arange(size) * ss - 1, 0))])
    inside = (np.abs(xs[::ss, ::ss] - 64.0) < w / 2 + 2.5 * sigma - 1) & (np.abs(ys[::ss, ::ss] - 64.0) < h / 2 + 2.5 * sigma - 1)
    assert np.abs(got - want)[inside].max() < 0.04, np.abs(got - want)[inside].max()
    assert abs(got[inside].sum() - want[inside].sum()) / want[inside].sum() < 0.01


# ---- invariances ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
def test_whole_pixel_translation_invariance_across_tiles_and_bins(oracle, aa):
    """The same shapes moved by whole pixels across 16-pixel tile and 256-pixel bin boundaries give the same pixels, moved:
    nothing in binning / tiling / backdrop propagation may depend on where the tile grid falls."""
    rng = np.random.default_rng(21)
    polys = [random_convex(rng, 40 + 30 * k, 45 + 11 * k, 26.0, 5 + k) for k in range(3)]

    def scene(dx, dy):
        s = Scene()
        for k, poly in enumerate(polys):
            shifted = [(x + dx, y + dy) for x, y in poly]
            s.fill(FILL_NON_ZERO if k != 1 else FILL_EVEN_ODD, Affine.IDENTITY, Color.from_rgba8(60 + 90 * k, 200 - 70 * k, 40 + 100 * k, 200), None, poly_path(shifted))
        s.stroke(Stroke(3.0), Affine.translate(dx, dy), Color.from_rgba8(250, 250, 20), None, Line(12.0, 15.0, 120.0, 70.0))
        return s
    ref = render(oracle, scene(0, 0), 160, 110, aa)
    for dx, dy in ((16, 0), (7, 13), (243, 201), (256, 256), (301, 199)):
        img = render(oracle, scene(dx, dy), 160 + dx, 110 + dy, aa)
        d = np.abs(img[dy:dy + 110, dx:dx + 160].astype(np.int32) - ref.astype(np.int32))
        if aa == AA_AREA:
            assert d.max() <= 1, (dx, dy, d.max())
        else:
            # a vertex at 280.3 is a different f32 than 24.3 + 256: an edge that grazes a sample point may flip that ONE sample
            flipped = int((d.max(axis=2) > 0).sum())
            assert d.max() <= 17 and flipped <= 8, (dx, dy, d.max(), flipped)
        outside = img.copy()
        outside[dy:dy + 110, dx:dx + 160] = 0
        assert (outside[..., :3] == 0).all()  # nothing leaks outside the moved bounding box (black base)


def test_shapes_hanging_over_the_frame_are_cut_not_distorted(oracle):
    rng = np.random.default_rng(22)
    poly = random_convex(rng, 40.0, 40.0, 36.0, 7)
    full = coverage(oracle, poly_path(poly), 96, 96, AA_MSAA16)
    for (ox, oy, w, h) in ((20, 0, 50, 96), (0, 30, 96, 40), (25, 25, 30, 30)):
        moved = [(x - ox, y - oy) for x, y in poly]
        part = coverage(oracle, poly_path(moved), w, h, AA_MSAA16)
        assert np.array_equal(part, full[oy:oy + h, ox:ox + w])


def test_even_odd_ring_is_the_difference_of_the_areas(oracle):
    outer = [(10.3, 8.7), (70.2, 12.4), (64.9, 61.3), (14.6, 57.8)]
    inner = [(28.1, 24.2), (50.7, 26.9), (47.3, 44.4), (30.9, 41.0)]
    p = BezPath()
    for poly in (outer, inner):
        p.move_to(*poly[0])
        for q in poly[1:]:
            p.line_to(*q)
        p.close_path()
    got = coverage(oracle, p, 80, 72, AA_AREA, FILL_EVEN_ODD)
    want = exact_coverage(outer, 80, 72) - exact_coverage(inner, 80, 72)
    assert np.abs(got - want).max() <= 1.5 / 255
    # nonzero with the inner contour reversed is the same ring; with the same orientation it is the full outer polygon
    rev = BezPath(list(poly_path(outer).els) + list(poly_path(inner[::-1]).els))
    same = BezPath(list(poly_path(outer).els) + list(poly_path(inner).els))
    assert np.abs(coverage(oracle, rev, 80, 72, AA_AREA) - want).max() <= 1.5 / 255
    assert np.abs(coverage(oracle, same, 80, 72, AA_AREA) - exact_coverage(outer, 80, 72)).max() <= 1.5 / 255


def test_affine_transform_of_a_fill_is_the_transformed_polygon(oracle):
    rng = np.random.default_rng(23)
    poly = random_convex(rng, 0.0, 0.0, 10.0, 6)
    a = Affine.translate(50.3, 41.7) * Affine.rotate(0.7) * Affine.scale(2.5)
    s = Scene()
    s.fill(FILL_NON_ZERO, a, WHITE, None, poly_path(poly))
    got = render(oracle, s, 100, 90, AA_AREA)[..., 0].astype(np.float64) / 255
    c, sn = math.cos(0.7), math.sin(0.7)
    moved = [(50.3 + 2.5 * (c * x - sn * y), 41.7 + 2.5 * (sn * x + c * y)) for x, y in poly]
    assert np.abs(got - exact_coverage(moved, 100, 90)).max() <= 1.5 / 255


# ---- whole scenes: the painter's algorithm over exact coverages ------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_random_scene_is_the_painters_algorithm_over_exact_areas(oracle, seed):
    """Twelve overlapping translucent polygons, a clip layer with alpha in the middle of the list: every pixel must equal
    src-over compositing (premultiplied, float64 here) of the shapes' exact polygon-pixel areas, in order."""
    rng = np.random.default_rng(300 + seed)
    W = H = 72
    s = Scene()
    acc = np.zeros((H, W, 4))
    acc[..., 3] = 1.0  # opaque black base

    def over(dst, colour, cov):
        src_a = colour[3] * cov
        for c in range(3):
            dst[..., c] = dst[..., c] * (1 - src_a) + colour[c] * src_a
        dst[..., 3] = dst[..., 3] * (1 - src_a) + src_a

    def add(target_scene, target_acc):
        poly = random_convex(rng, rng.uniform(15, 57), rng.uniform(15, 57), rng.uniform(8, 26), int(rng.integers(3, 8)))
        rgba = [int(v) for v in rng.integers(0, 256, 3)] + [int(rng.integers(60, 256))]
        target_scene.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(*rgba), None, poly_path(poly))
        over(target_acc, [v / 255 for v in rgba], exact_coverage(poly, W, H))

    for _ in range(5):
        add(s, acc)
    # a layer: clip polygon, alpha 0.6, three shapes inside; composited as one group (src-over, normal)
    clip = random_convex(rng, 36.0, 36.0, 27.0, 6)
    s.push_layer(FILL_NON_ZERO, MIX_NORMAL, COMPOSE_SRC_OVER, 0.6, Affine.IDENTITY, poly_path(clip))
    layer = np.zeros((H, W, 4))
    for _ in range(3):
        add(s, layer)
    s.pop_layer()
    k = 0.6 * exact_coverage(clip, W, H)
    for c in range(3):
        acc[..., c] = acc[..., c] * (1 - layer[..., 3] * k) + layer[..., c] * k  # layer[] is premultiplied already
    acc[..., 3] = acc[..., 3] * (1 - layer[..., 3] * k) + layer[..., 3] * k
    for _ in range(4):
        add(s, acc)
    got = render(oracle, s, W, H, AA_AREA).astype(np.float64)
    assert (got[..., 3] == 255).all()
    assert np.abs(got[..., :3] - 255 * acc[..., :3]).max() <= 2.5, np.abs(got[..., :3] - 255 * acc[..., :3]).max()


# ---- more stroke / image / layer semantics --------------------------------------------------------------------------------------------------
def test_miter_limit_falls_back_to_bevel(oracle):
    """kurbo / SVG: a miter join whose length exceeds miter_limit x half-width... ratio 1 / sin(theta / 2) (theta = interior
    angle) is drawn as a bevel. Interior angle 20 degrees has ratio 5.76: a bevel under limit 4, a miter under limit 10."""
    from vello_b200.encoding import STYLE_JOIN_MITER
    w, l1, l2 = 6.0, 70.0, 70.0
    phi = math.radians(160.0)  # exterior (turning) angle
    p0 = (20.0, 60.0)
    p1 = (p0[0] + l1, p0[1])
    p2 = (p1[0] + l2 * math.cos(phi), p1[1] - l2 * math.sin(phi))
    path = BezPath([("M",) + p0, ("L",) + p1, ("L",) + p2])
    h = w / 2
    kite = h * h * math.tan(phi / 2)
    # the two rectangles overlap along most of their length here (narrow angle): count the union by the exact formula for the
    # difference between the two renderings instead: miter - bevel = kite - triangle
    def area(limit):
        s = Scene()
        s.stroke(Stroke(w, join=STYLE_JOIN_MITER, miter_limit=limit, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), Affine.IDENTITY, WHITE, None, path)
        return render(oracle, s, 128, 128, AA_AREA)[..., 0].astype(np.float64).sum() / 255
    bevel_only = Scene()
    bevel_only.stroke(Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), Affine.IDENTITY, WHITE, None, path)
    bevel = render(oracle, bevel_only, 128, 128, AA_AREA)[..., 0].astype(np.float64).sum() / 255
    assert abs(area(4.0) - bevel) < 0.05                       # limit exceeded: identical to a bevel join
    want_extra = kite - 0.5 * h * h * math.sin(phi)
    assert abs((area(10.0) - bevel) - want_extra) / want_extra < 0.03


def test_dashed_stroke_area_is_width_times_the_on_length(oracle):
    length, w = 100.0, 4.0
    for pattern, offset in (((7.0, 3.0), 0.0), ((5.0, 2.0, 1.0), 0.0), ((6.0, 6.0), 4.0)):
        pat = list(pattern) * (2 if len(pattern) % 2 else 1)  # an odd pattern repeats with the roles swapped
        period = sum(pat)
        on = 0.0
        pos, i, t = offset % period, 0, 0.0  # kurbo: the pattern is entered `dash_offset` along
        # walk the pattern from the offset
        acc = 0.0
        while acc + pat[i] <= pos:
            acc += pat[i]
            i = (i + 1) % len(pat)
        rem = acc + pat[i] - pos
        while t < length:
            step = min(rem, length - t)
            if i % 2 == 0:
                on += step
            t += step
            i = (i + 1) % len(pat)
            rem = pat[i]
        s = Scene()
        st = Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT, dash_pattern=tuple(pattern), dash_offset=offset)
        s.stroke(st, Affine.IDENTITY, WHITE, None, Line(10.0, 20.3, 10.0 + length, 20.3))
        got = render(oracle, s, 128, 40, AA_AREA)[..., 0].astype(np.float64).sum() / 255
        assert abs(got - w * on) / (w * on) < 0.02, (pattern, offset, got, w * on)  # area AA's vertical-edge term: see above


def test_image_alpha_format_and_alpha_type(oracle):
    from vello_b200.encoding import ALPHA_PREMULTIPLIED, ALPHA_STRAIGHT, FORMAT_BGRA8, FORMAT_RGBA8, Image, QUALITY_LOW
    px = np.array([[[200, 100, 50, 128]]], dtype=np.uint8)
    def one(**kw):
        s = Scene()
        s.draw_image(Image(np.repeat(np.repeat(px, 4, 0), 4, 1), quality=QUALITY_LOW, **kw), Affine.IDENTITY)
        return render(oracle, s, 4, 4, AA_AREA, TRANSPARENT)[1, 1].astype(np.float64)
    a = 128 / 255
    # straight alpha: stored separated -> the colour comes back, alpha = a
    assert np.abs(one(format=FORMAT_RGBA8, alpha_type=ALPHA_STRAIGHT) - (200, 100, 50, 128)).max() <= 1.0
    # BGRA: the channels swap
    assert np.abs(one(format=FORMAT_BGRA8, alpha_type=ALPHA_STRAIGHT) - (50, 100, 200, 128)).max() <= 1.0
    # premultiplied input: the stored texel IS colour x alpha; un-premultiplying on store divides it out
    assert np.abs(one(format=FORMAT_RGBA8, alpha_type=ALPHA_PREMULTIPLIED) - (min(255, 200 / a), min(255, 100 / a), 50 / a, 128)).max() <= 1.5
    # the brush alpha multiplies everything
    got = one(format=FORMAT_RGBA8, alpha_type=ALPHA_STRAIGHT, alpha=0.5)
    assert abs(got[3] - 64) <= 1.0 and np.abs(got[:3] - (200, 100, 50)).max() <= 2.0


def test_deeply_nested_layers_multiply_their_alphas(oracle):
    """Seven nested layers (more than the four blend-stack levels kept in registers: the deeper ones spill to memory,
    fine.wgsl:1097-1130), each with alpha 0.8 and its own clip: the innermost fill arrives with 0.8^7."""
    s = Scene()
    depth = 7
    for k in range(depth):
        s.push_layer(FILL_NON_ZERO, MIX_NORMAL, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Rect(2.0 + k, 2.0 + k, 60.0 - k, 60.0 - k))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, WHITE, None, Rect(0.0, 0.0, 64.0, 64.0))
    for _ in range(depth):
        s.pop_layer()
    got = render(oracle, s, 64, 64, AA_AREA)[..., 0].astype(np.float64)
    assert abs(got[32, 32] - 255 * 0.8 ** depth) <= 3.0  # one 8-bit store per level on the way out
    # the clips nest: only the innermost rectangle (8 .. 54) is painted
    assert got[1, 1] == 0 and got[5, 32] == 0 and got[32, 56] == 0
    assert got[9, 32] == pytest.approx(got[32, 32], abs=1.0) and got[53, 9] == pytest.approx(got[32, 32], abs=1.0)


def test_arc_stroke_is_width_times_arc_length(oracle):
    from vello_b200.shapes import Arc
    r, w = 30.0, 4.0
    for start, sweep in ((0.3, 2.0), (1.0, -4.5), (-2.0, 5.9)):
        s = Scene()
        s.stroke(Stroke(w, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), Affine.IDENTITY, WHITE, None, Arc(48.0, 47.0, r, r, start, sweep))
        got = render(oracle, s, 96, 96, AA_AREA)[..., 0].astype(np.float64).sum() / 255
        want = w * r * abs(sweep)  # the annular sector: 1/2 (R^2 - r^2) |sweep| = w r |sweep|
        assert abs(got - want) / want < 0.015, (start, sweep, got, want)  # two flattened offset curves, 0.25 px each


def test_rounded_rect_and_svg_arc_areas(oracle):
    from vello_b200.shapes import RoundedRect
    w, h, r = 61.0, 37.0, 11.5
    got = coverage(oracle, RoundedRect(9.3, 14.2, 9.3 + w, 14.2 + h, r), 96, 72, AA_AREA).sum()
    want = w * h - (4 - math.pi) * r * r
    assert -1.0 <= want - got <= (2.0 / 3.0) * 2 * math.pi * r * 0.25 + 1.0  # the four corners: chords within flatten's 0.25 px
    # SVG elliptical arcs (kurbo svg.rs + SVG implementation notes F.6): half an ellipse closed by its diameter, and a
    # "pac-man": the large arc of a circle closed through the centre
    half = BezPath.from_svg("M 20 50 A 35 20 0 0 1 90 50 Z")
    got = coverage(oracle, half, 110, 90, AA_AREA).sum()
    assert -1.0 <= 0.5 * math.pi * 35 * 20 - got <= (2.0 / 3.0) * math.pi * 35 * 0.25 + 1.0
    a = math.radians(40.0)
    x0, y0 = 50 + 30 * math.cos(a), 50 - 30 * math.sin(a)
    x1, y1 = 50 + 30 * math.cos(a), 50 + 30 * math.sin(a)
    pac = BezPath.from_svg(f"M 50 50 L {x0} {y0} A 30 30 0 1 0 {x1} {y1} Z")  # large-arc, sweep 0: counter-clockwise on screen
    got = coverage(oracle, pac, 100, 100, AA_AREA).sum()
    want = math.pi * 900 * (360 - 80) / 360
    assert -1.0 <= want - got <= (2.0 / 3.0) * 2 * math.pi * 30 * 0.25 + 1.0


def test_multi_stop_gradient_and_alpha_interpolation_spaces(oracle):
    """Three opaque stops at unequal offsets == the piecewise lerp; two stops with different alphas under the two
    interpolation alpha spaces of peniko (`InterpolationAlphaSpace`): premultiplied lerps colour x alpha, separate lerps
    the straight components."""
    r = Rect(0.0, 0.0, 128.0, 4.0)
    cols = [np.array([250.0, 30.0, 10.0]), np.array([20.0, 230.0, 40.0]), np.array([30.0, 50.0, 245.0])]
    offs = [0.0, 0.3, 1.0]
    stops = [(o, Color.from_rgba8(*[int(v) for v in c])) for o, c in zip(offs, cols)]
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((8.0, 0.0), (120.0, 0.0), stops), None, r)
    got = render(oracle, s, 128, 4, AA_AREA)[2, :, :3].astype(np.float64)
    t = np.clip((np.arange(128) - 8.0) / 112.0, 0, 1)
    want = np.where((t < 0.3)[:, None], cols[0] + (cols[1] - cols[0]) * (t / 0.3)[:, None], cols[1] + (cols[2] - cols[1]) * ((t - 0.3) / 0.7)[:, None])
    assert np.abs(got - want).max() <= 2.5
    c0, a0, c1, a1 = np.array([255.0, 40.0, 0.0]), 1.0, np.array([0.0, 80.0, 255.0]), 0.2
    stops = [(0.0, Color.from_rgba8(255, 40, 0, 255)), (1.0, Color.from_rgba8(0, 80, 255, 51))]
    t = np.clip((np.arange(128) - 8.0) / 112.0, 0, 1)[:, None]
    for premul in (True, False):
        s = Scene()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((8.0, 0.0), (120.0, 0.0), stops, premul_interp=premul), None, r)
        got = render(oracle, s, 128, 4, AA_AREA, TRANSPARENT)[2].astype(np.float64)
        alpha = a0 + (a1 - a0) * t
        if premul:
            colour = ((c0 * a0) + (c1 * a1 - c0 * a0) * t) / alpha
        else:
            colour = c0 + (c1 - c0) * t
        assert np.abs(got[:, 3:4] - 255 * alpha).max() <= 1.5
        # the stored colour is premultiplied 8-bit ramp texel / alpha: at alpha 0.2 one LSB of the texel is 5 of the quotient
        assert (np.abs(got[:, :3] - colour) * alpha).max() <= 2.0, premul
