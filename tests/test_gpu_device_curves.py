"""Curved fragments from device arrays (Renderer.upload_device_paths(point_kinds=...), vb_fragment_from_device_curves): the
fragment built on the device from points, kinds (0 on-curve, 1 off-curve), offsets and colours must be word for word the
fragment `upload_fragment` makes of the Scene that fills or strokes each path with its colour, its shape being, per ring,
M p_first, then L / Q / C per on-curve point after the first (by the off-curve points in front of it), and Z (fills always,
strokes when closed). Every case composes both fragments and compares the composed scene's words, layout and draw offsets,
and the frames. Run on an H100 with `pytest -m gpu`."""
import ctypes as C
import math

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (Color, FILL_EVEN_ODD, FILL_NON_ZERO, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE,
                                 STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Scene, Stroke)
from vello_b200.renderer import Renderer, VelloB200Error
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Arc, Circle, Ellipse, RoundedRect, path_elements

from . import device_curves_ref as ref
from .test_gpu_device_paths import BASE, composed, dev, frame, held, host_fragment

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def r():
    r = Renderer()
    yield r
    r.close()


# ---- the reference: the host Scene loop of the contract -------------------------------------------------------------------
def reference(pts, kinds, roff, poff, cols, style, closed, native=False):
    """(the host Scene, each path's draw object or -1)"""
    s = NativeScene() if native else Scene()
    stroke = isinstance(style, Stroke)
    closes = closed or not stroke
    draw = []
    for i in range(len(poff) - 1):
        els = []
        for k in range(int(poff[i]), int(poff[i + 1])):
            a, b = int(roff[k]), int(roff[k + 1])
            if a < b:
                els += ref.elements(pts, kinds, a, b) + ([("Z",)] if closes else [])
        n0 = s.n_draw_objects
        c = Color(*[float(v) for v in cols[i]])
        if stroke:
            s.stroke(style, Affine.IDENTITY, c, None, els)
        else:
            s.fill(style, Affine.IDENTITY, c, None, els)
        draw.append(n0 if s.n_draw_objects > n0 else -1)
    return s, draw


def build(r, pts, kinds, roff, poff, cols, style=FILL_NON_ZERO, closed=True):
    idx = torch.full((len(poff) - 1,), -7, dtype=torch.int32, device="cuda")
    k = None if kinds is None else dev(kinds, torch.uint8)
    fid, n = r.upload_device_paths(dev(pts, torch.float32), dev(roff, torch.int32), dev(cols, torch.float32),
                                   path_offsets=dev(poff, torch.int32), style=style, closed=closed, draw_index=idx, point_kinds=k)
    return fid, n, idx.cpu().numpy()


def check(r, pts, kinds, roff, poff, cols, style=FILL_NON_ZERO, closed=True, frames=True, native=False,
          aas=(AA_MSAA8, AA_MSAA16, AA_AREA)):
    """Build both fragments, compare the composed scenes word for word and, with `frames`, the frames in the AA modes `aas`."""
    pts = np.asarray(pts, dtype=np.float32).reshape(-1, 2)
    kinds = np.asarray(kinds, np.uint8)
    roff, poff = np.asarray(roff, np.int32), np.asarray(poff, np.int32)
    cols = np.asarray(cols, dtype=np.float32).reshape(-1, 4)
    fid, n, idx = build(r, pts, kinds, roff, poff, cols, style, closed)
    scene, want_idx = reference(pts, kinds, roff, poff, cols, style, closed, native)
    ref_id = r.upload_fragment(scene)
    try:
        assert n == scene.n_draw_objects
        assert list(idx) == want_idx
        lay, offs, words = composed(r, [(fid, None)])
        imgs = [frame(r, aa) for aa in aas] if frames else []
        lay_ref, offs_ref, words_ref = composed(r, [(ref_id, None)])
        assert (lay.as_array() == lay_ref.as_array()).all(), f"layout {lay} != {lay_ref}"
        assert offs == offs_ref
        assert words.size == words_ref.size, f"{words.size} words, want {words_ref.size}"
        diff = np.nonzero(words != words_ref)[0]
        assert diff.size == 0, f"scene words differ at {diff[:8]}: {words[diff[:8]]} != {words_ref[diff[:8]]}"
        for img, aa in zip(imgs, aas):
            assert (img == frame(r, aa)).all(), f"aa {aa}"
    finally:
        r.free_fragment(fid)
        r.free_fragment(ref_id)
    return idx


def join_paths(paths):
    """(points, kinds, ring offsets, path offsets) of a list of paths, each a list of rings (points, kinds)."""
    pts, kinds, roff, poff = [], [], [0], [0]
    for rings in paths:
        for p, k in rings:
            pts += [tuple(map(float, q)) for q in p]
            kinds += list(k)
            roff.append(len(pts))
        poff.append(len(roff) - 1)
    return np.array(pts, np.float32).reshape(-1, 2), np.array(kinds, np.uint8), roff, poff


def shape_rings(shape):
    pts, kinds, roff = ref.points_of(path_elements(shape, 0.1))
    return [(pts[a:b], kinds[a:b]) for a, b in zip(roff[:-1], roff[1:])]


SHAPES = [Circle(70, 70, 40), Circle(128, 128, 520), Ellipse(170, 80, 60, 25, 0.5), RoundedRect(20, 140, 120, 230, 18),
          Arc(180, 180, 50, 35, 0.4, 4.2), Circle(200, 40, 0.5)]


def cols_for(n, seed=1):
    return np.random.default_rng(seed).uniform(0.2, 1, (n, 4)).astype(np.float32)


# ---- fills and strokes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule", [FILL_NON_ZERO, FILL_EVEN_ODD])
def test_kurbo_shapes_filled(r, rule):
    """Circles (also the n > 4 branch of a large radius), ellipses, rounded rectangles and arcs, as shapes.path_elements gives
    them, filled; and all of them as the rings of one path."""
    paths = [shape_rings(s) for s in SHAPES]
    paths.append([ring for p in paths for ring in p])
    pts, kinds, roff, poff = join_paths(paths)
    check(r, pts, kinds, roff, poff, cols_for(len(paths)), rule)


@pytest.mark.parametrize("join", [STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND])
@pytest.mark.parametrize("caps", [(STYLE_CAP_BUTT, STYLE_CAP_SQUARE), (STYLE_CAP_ROUND, STYLE_CAP_BUTT), (STYLE_CAP_SQUARE, STYLE_CAP_ROUND)])
@pytest.mark.parametrize("closed", [False, True])
def test_kurbo_shapes_stroked(r, join, caps, closed):
    paths = [shape_rings(s) for s in SHAPES]
    pts, kinds, roff, poff = join_paths(paths)
    check(r, pts, kinds, roff, poff, cols_for(len(paths), 2), Stroke(5.0, join, 2.5, caps[0], caps[1]), closed)


def glyph(x, y, s):
    """A TrueType-like outline: an outer quadratic contour and a counter (hole) wound the other way, implied on-curve
    midpoints already inserted."""
    outer = [(0, 0), (0.5, -0.2), (1, 0), (1.2, 0.5), (1, 1), (0.5, 1.2), (0, 1), (-0.2, 0.5), (0, 0)]
    hole = [(0.3, 0.3), (0.2, 0.5), (0.3, 0.7), (0.5, 0.8), (0.7, 0.7), (0.8, 0.5), (0.7, 0.3), (0.5, 0.2), (0.3, 0.3)]
    k = [0, 1, 0, 1, 0, 1, 0, 1, 0]
    f = lambda ring: np.array(ring, np.float64) * s + (x, y)  # noqa: E731
    return [(f(outer), k), (f(hole), k)]


MIXED = [  # L, Q and C in one ring, a curved closing segment, and a ring that closes with a line
    ([(20, 20), (80, 20), (110, 5), (120, 40), (140, 60), (150, 100), (110, 120), (60, 110), (30, 130), (20, 20)],
     [0, 0, 1, 0, 1, 1, 0, 0, 1, 0]),
    ([(150, 150), (200, 140), (230, 170), (240, 230), (200, 240), (160, 230)], [0, 1, 0, 1, 1, 0]),
]


@pytest.mark.parametrize("style, closed", [(FILL_NON_ZERO, True), (FILL_EVEN_ODD, True), (Stroke(3.0), False), (Stroke(3.0), True)],
                         ids=["nonzero", "evenodd", "stroke_open", "stroke_closed"])
def test_glyphs_and_mixed_rings(r, style, closed):
    paths = [glyph(10 + 60 * i, 30 + 50 * (i % 3), 40 + 5 * i) for i in range(4)] + [MIXED]
    pts, kinds, roff, poff = join_paths(paths)
    check(r, pts, kinds, roff, poff, cols_for(len(paths), 3), style, closed)


@pytest.mark.parametrize("style", [FILL_NON_ZERO, Stroke(2.0)], ids=["fill", "stroke"])
@pytest.mark.parametrize("closed", [False, True])
def test_degenerate_curves(r, style, closed):
    """First segments collapsing onto p0; collapsed middle segments; the tangent test against the span test; EPS-close control
    points near zero that force the walk; -0 beside +0 at the closing point; an open stroke's cap after a curve; paths whose
    rings all drop."""
    e = 4e-13
    paths = [
        [([(50, 50), (50, 50), (50, 50), (50, 50), (50, 50), (90, 60), (120, 50), (90, 90)], [0, 1, 0, 1, 1, 0, 1, 0])],
        [([(10, 200), (40, 180), (70, 200), (70, 200), (70, 200), (70, 200), (100, 200), (130, 230)], [0, 1, 0, 1, 1, 0, 1, 0])],
        [([(0, 0), (8e-13, 0), (-8e-13, 0), (30, 10), (10, 30)], [0, 1, 0, 0, 0])],  # the quad drops: tangent, not span
        [([(0, 0), (3e-12, 0), (3e-12 + e, e), (3e-12 + 2 * e, 0), (3e-12 + 3 * e, e), (3e-12 + 5 * e, 0), (1e-11, 2e-12)],
          [0, 0, 1, 0, 1, 1, 0])],  # EPS-close after the first kept segment: walked
        [([(-0.0, 20.0), (40, 0), (60, 60), (0.0, 20.0)], [0, 1, 1, 0])],  # closing point value-equal only
        [([(150, 150), (200, 100), (220, 170)], [0, 1, 0])],  # one quad: an open stroke's cap after a curve
        [([(7, 7), (7, 7), (7, 7)], [0, 1, 0]), ([(9, 9)], [0]), ([(3, 3), (3, 3), (3, 3), (3, 3)], [0, 1, 1, 0])],  # drops
        [([(5, 5)], [0])],
    ]
    pts, kinds, roff, poff = join_paths(paths)
    idx = check(r, pts, kinds, roff, poff, cols_for(len(paths), 4), style, closed, frames=False)
    assert idx[6] == -1 and idx[7] == -1


@pytest.mark.parametrize("n", [255, 256, 257, 511])
def test_segments_across_partitions(r, n):
    """Cubic and quadratic segments whose control points and end point fall in different 256-point partitions."""
    pts, kinds = [], []
    for shift in range(3):  # three rings, so that every position of a segment meets a boundary
        m = n + shift
        t = np.linspace(0, 2 * np.pi, m)
        rad = 60 + 40 * shift
        ring = np.stack([128 + rad * np.cos(t), 128 + rad * np.sin(t)], 1)
        k = np.where(np.arange(m) % 3 == 0, 0, 1).astype(np.uint8)
        k[-1] = 0
        if m >= 3 and k[-2] == 1 and k[-3] == 1:
            k[-3] = 0
        ring[-1] = ring[0]
        pts.append(ring)
        kinds.append(k)
    roff = np.cumsum([0] + [len(p) for p in pts]).astype(np.int32)
    pts, kinds = np.concatenate(pts), np.concatenate(kinds)
    check(r, pts, kinds, roff, [0, 1, 3], cols_for(2, n), FILL_EVEN_ODD)
    check(r, pts, kinds, roff, [0, 1, 3], cols_for(2, n), Stroke(1.5), False, frames=False)


def random_circles(rng, n):
    """n random circles, each the four cubics of shapes.path_elements(Circle): 13 points a ring."""
    c = rng.uniform(0, 256, (n, 2))
    rad = rng.uniform(1, 12, n)
    arm = 0.551915024494
    ring = []
    for ix in range(1, 5):
        th0, th1 = (ix - 1) * math.pi / 2, ix * math.pi / 2
        s0, c0 = math.sin(th0), math.cos(th0)
        s1, c1 = (0.0, 1.0) if ix == 4 else (math.sin(th1), math.cos(th1))
        ring += [(c0 - arm * s0, s0 + arm * c0), (c1 + arm * s1, s1 - arm * c1), (c1, s1)]
    unit = np.array([(1.0, 0.0)] + ring)
    pts = (c[:, None, :] + rad[:, None, None] * unit[None]).reshape(-1, 2)
    kinds = np.tile(np.array([0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0], np.uint8), n)
    return pts, kinds, np.arange(0, 13 * n + 1, 13, dtype=np.int32)


def test_random_circles(r):
    rng = np.random.default_rng(5)
    pts, kinds, roff = random_circles(rng, 100_000)
    assert kinds.size == 1_300_000
    check(r, pts, kinds, roff, np.arange(100_001, dtype=np.int32), cols_for(100_000, 5), FILL_NON_ZERO, native=True)


def test_million_point_spline(r):
    """A 1M-point cubic spline, stroked (area sums over this many segments are not bit-stable between renders: MSAA frames)."""
    n = 999_999 + 1
    x = np.linspace(4, 252, n)
    y = 128 + 100 * np.sin(x / 9.0)
    kinds = np.where(np.arange(n) % 3 == 0, 0, 1).astype(np.uint8)
    kinds[-1] = 0
    pts = np.stack([x, y], 1)
    check(r, pts, kinds, [0, n], [0, 1], [[1, 1, 0.2, 1]], Stroke(1.0), False, native=True, aas=(AA_MSAA8, AA_MSAA16))


# ---- equivalences ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("style", [FILL_NON_ZERO, Stroke(2.0)], ids=["fill", "stroke"])
def test_on_curve_kinds_are_the_polyline_call(r, style):
    """Kinds of all zeros, and point_kinds=None, give the fragment upload_device_paths gives without kinds, word for word."""
    from .test_gpu_device_paths import ragged
    pts, roff, poff, cols = ragged(np.random.default_rng(7), 300, 3, 10)
    pts[5:9] = pts[4]
    outs = []
    for kinds in ("absent", None, np.zeros(len(pts), np.uint8)):
        idx = torch.full((len(poff) - 1,), -7, dtype=torch.int32, device="cuda")
        kw = {} if isinstance(kinds, str) else dict(point_kinds=None if kinds is None else dev(kinds, torch.uint8))
        fid, n = r.upload_device_paths(dev(pts, torch.float32), dev(roff, torch.int32), dev(cols, torch.float32),
                                       path_offsets=dev(poff, torch.int32), style=style, closed=False, draw_index=idx, **kw)
        lay, offs, words = composed(r, [(fid, None)])
        outs.append((n, idx.cpu().numpy(), lay.as_array(), offs, words))
        r.free_fragment(fid)
    for o in outs[1:]:
        assert o[0] == outs[0][0] and (o[1] == outs[0][1]).all() and (o[2] == outs[0][2]).all() and o[3] == outs[0][3]
        assert (o[4] == outs[0][4]).all()


# ---- composition -----------------------------------------------------------------------------------------------------------
def overlay(scale=1.0, shift=0.0):
    paths = [shape_rings(Circle(40, 40, 25)), glyph(70, 20, 50), shape_rings(RoundedRect(10, 90, 60, 130, 8))]
    pts, kinds, roff, poff = join_paths(paths)
    return pts * np.float32(scale) + np.float32(shift), kinds, roff, poff, cols_for(3, 8)


def test_beside_host_fragments(r):
    """A curved device fragment among host fragments, under instance transforms and a view; hit tests at an interior point
    of each path; bound colours on its rows; the frames against the same composition of its host twin."""
    pts, kinds, roff, poff, cols = overlay()
    fid, n, idx = build(r, pts, kinds, np.array(roff, np.int32), np.array(poff, np.int32), cols)
    twin = r.upload_fragment(reference(pts, kinds, roff, poff, cols, FILL_NON_ZERO, True)[0])
    base = host_fragment(r)
    xf = [None, Affine.translate(100, 20), Affine.translate(30, 140) * Affine.rotate(0.3)]
    try:
        for view in (None, Affine.scale(1.3)):
            r.set_view(view)
            outs = []
            for f in (fid, twin):
                lay, offs = r.compose([(base, xf[0]), (f, xf[1]), (base, xf[2])])
                outs.append((lay.as_array(), offs, r.download("scene", np.uint32), [frame(r, aa) for aa in (AA_MSAA16, AA_AREA)]))
            assert (outs[0][0] == outs[1][0]).all() and outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()
            for a, b in zip(outs[0][3], outs[1][3]):
                assert (a == b).all()
        r.set_view(None)
        lay, offs = r.compose([(base, None), (fid, Affine.translate(100, 20)), (base, Affine.translate(30, 140))])
        frame(r, AA_MSAA16)
        # interior points, moved by the instance's translation: the circle's centre, the glyph's ring, the rounded rectangle
        got = r.hit_test(np.array([[140, 60], [70 + 50 * 0.1 + 100, 20 + 25 + 20], [135, 130]], np.float32))
        assert list(got) == [offs[1] + int(idx[0]), offs[1] + int(idx[1]), offs[1] + int(idx[2])]
        rows = torch.full((offs[2], 4), float("nan"), device="cuda")
        rows[offs[1] + int(idx[0])] = torch.tensor([0.0, 1.0, 0.0, 1.0])
        r.bind_draw_colors(rows)
        img = frame(r, AA_MSAA16)
        r.bind_draw_colors(None)
        cols2 = cols.copy()
        cols2[0] = [0, 1, 0, 1]
        twin2 = r.upload_fragment(reference(pts, kinds, roff, poff, cols2, FILL_NON_ZERO, True)[0])
        r.compose([(base, None), (twin2, Affine.translate(100, 20)), (base, Affine.translate(30, 140))])
        assert (img == frame(r, AA_MSAA16)).all()
        r.free_fragment(twin2)
    finally:
        r.set_view(None)
        for f in (fid, twin, base):
            r.free_fragment(f)


def test_recompose_rebuilt_curves(r):
    """Curves rebuilt from device arrays and swapped in by recompose damage only their boxes, and the damage-tracked frame
    equals a full frame of the same composition."""
    base = host_fragment(r)
    pts, kinds, roff, poff, cols = overlay(0.4, 160.0)
    roff, poff = np.array(roff, np.int32), np.array(poff, np.int32)
    a, _, _ = build(r, pts, kinds, roff, poff, cols)
    p = RenderParams(BASE, 256, 256, AA_MSAA16)
    r.set_damage_tracking(True)
    b = None
    try:
        r.compose([(base, None), (a, None)])
        r.render_resident(p)
        r.render_resident(p)
        b, _, _ = build(r, pts + np.float32(3.0), kinds, roff, poff, cols)
        r.recompose([(base, None), (b, None)])
        r.render_resident(p)
        got = r.download_target(p)
        mask = r.last_damage()
        assert 0 < mask.sum() < mask.size
        assert not mask[: 130 // 16, : 130 // 16].any(), "the host fragment's tiles stay undamaged"
        r.set_damage_tracking(False)
        r.compose([(base, None), (b, None)])
        assert (got == frame(r, AA_MSAA16)).all()
    finally:
        r.set_damage_tracking(False)
        for f in (base, a, b):
            if f is not None:
                r.free_fragment(f)


# ---- errors ----------------------------------------------------------------------------------------------------------------
def test_kind_errors_leave_no_fragment(r):
    """Every refusal of the kinds, through Python and through the C ABI, names the first offending row, leaves the installed
    scene as it was, makes no fragment (no id is taken and no device memory is kept) and lets the next valid call succeed."""
    from vello_b200.renderer import _DevicePaths
    base = host_fragment(r)
    square = np.array([(40, 40), (120, 20), (200, 40), (200, 200), (40, 200), (40, 40)], np.float32)
    pts = dev(square, torch.float32)
    roff = dev(np.array([0, 3, 6], np.int32), torch.int32)
    cols = dev(np.ones((2, 4), np.float32), torch.float32)
    good = np.array([0, 1, 0, 0, 0, 0], np.uint8)
    f0, _ = r.upload_device_paths(pts, roff, cols, point_kinds=dev(good, torch.uint8))
    r.free_fragment(f0)  # the scratch now holds every case below
    held(r, base)
    a0 = held(r, base)
    before = r.download("scene", np.uint32)
    cases = [
        ([0, 2, 0, 0, 0, 0], "point_kinds[1]"),  # a value other than 0 or 1
        ([0, 1, 0, 0, 7, 0], "point_kinds[4]"),
        ([1, 0, 0, 0, 0, 0], "point_kinds[0]"),  # a ring's first point off-curve
        ([0, 0, 0, 1, 0, 0], "point_kinds[3]"),  # the second ring's first point
        ([0, 1, 1, 0, 0, 0], "point_kinds[2]"),  # a ring's last point off-curve
        ([0, 0, 0, 0, 0, 1], "point_kinds[5]"),
        ([0, 0, 0, 1, 0, 2], "point_kinds[3]"),  # the first offending row of several
    ]
    for k, why in cases:
        with pytest.raises(VelloB200Error, match=r"vb_fragment_from_device_curves") as e:
            r.upload_device_paths(pts, roff, cols, point_kinds=dev(np.array(k, np.uint8), torch.uint8))
        assert why in str(e.value), (k, str(e.value))
        assert (r.download("scene", np.uint32) == before).all(), "the previous scene stays"
    # a third off-curve point in a row
    long_pts = dev(np.array([(0, 0), (10, 0), (20, 5), (30, 0), (40, 0)], np.float32), torch.float32)
    with pytest.raises(VelloB200Error, match=r"point_kinds\[3\]"):
        r.upload_device_paths(long_pts, dev(np.array([0, 5], np.int32), torch.int32), cols[:1],
                              point_kinds=dev(np.array([0, 1, 1, 1, 0], np.uint8), torch.uint8))

    class _Host:  # host memory through a raw pointer: refused by the library, not just the Python checks
        def __init__(self, a):
            self.a = a
            self.__cuda_array_interface__ = dict(shape=a.shape, typestr="|u1", data=(a.ctypes.data, False), version=2, strides=None)
    with pytest.raises(VelloB200Error, match="point_kinds must be device or managed memory"):
        r.upload_device_paths(pts, roff, cols, point_kinds=_Host(good.copy()))

    def raw(kinds_ptr):
        d = _DevicePaths(pts.data_ptr(), 6, 8, roff.data_ptr(), 2, None, 2, cols.data_ptr(), 16)
        fid, n = C.c_uint32(0), C.c_uint32(0)
        rc = r.lib.vb_fragment_from_device_curves(r.handle, C.byref(d), kinds_ptr, C.byref(fid), C.byref(n))
        return rc, fid.value, r.lib.vb_last_error(r.handle).decode()
    host = good.copy()
    rc, _, msg = raw(C.c_void_p(host.ctypes.data))
    assert rc != 0 and "point_kinds must be device" in msg, msg
    bad = dev(np.array([0, 1, 1, 0, 0, 0], np.uint8), torch.uint8)
    rc, _, msg = raw(C.c_void_p(bad.data_ptr()))
    assert rc != 0 and "point_kinds[2]" in msg, msg
    assert (r.download("scene", np.uint32) == before).all()
    assert held(r, base) == a0, "a refused call keeps no device memory"
    odd = dev(np.array([9, 0, 1, 0, 0, 0, 0], np.uint8), torch.uint8)  # kinds at an odd address: any alignment is taken
    rc, fid, msg = raw(C.c_void_p(odd.data_ptr() + 1))
    assert rc == 0 and fid == f0 + 1, (msg, fid, f0)  # the next valid call succeeds, with the next id: no refusal took one
    r.free_fragment(fid)
    r.free_fragment(base)
