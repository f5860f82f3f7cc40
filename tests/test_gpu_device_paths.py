"""Fragments from device arrays (Renderer.upload_device_paths, vb_fragment_from_device_paths): the fragment built on the device
from ragged points / offsets / colours must be word for word the fragment `upload_fragment` makes of the Scene that fills or
strokes each path with its colour, its shape being, per ring, M p_first, L p..., and Z (fills always, strokes when closed).
Every case composes both fragments and compares the composed scene's words, layout and draw offsets, and the frames. Run on an
H100 with `pytest -m gpu`."""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (Color, FILL_EVEN_ODD, FILL_NON_ZERO, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE,
                                 STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Scene, Stroke)
from vello_b200.renderer import Renderer, VelloB200Error
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Circle, Rect

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BASE = Color.from_rgba8(12, 20, 30)
W = H = 256


@pytest.fixture(scope="module")
def r():
    r = Renderer()
    yield r
    r.close()


# ---- the reference: the host Scene loop of the contract -------------------------------------------------------------------
def shapes_of(pts, roff, poff, closes):
    """Per path, the element list of its rings (a ring of no point adds nothing)."""
    out = []
    n_paths = len(poff) - 1 if poff is not None else len(roff) - 1
    for i in range(n_paths):
        r0, r1 = (int(poff[i]), int(poff[i + 1])) if poff is not None else (i, i + 1)
        els = []
        for k in range(r0, r1):
            a, b = int(roff[k]), int(roff[k + 1])
            if a == b:
                continue
            els.append(("M", float(pts[a, 0]), float(pts[a, 1])))
            els += [("L", float(x), float(y)) for x, y in pts[a + 1:b]]
            if closes:
                els.append(("Z",))
        out.append(els)
    return out


def reference(pts, roff, poff, cols, style, closed, native=False):
    """(the host Scene, each path's draw object or -1)"""
    s = NativeScene() if native else Scene()
    draw = []
    stroke = isinstance(style, Stroke)
    for i, els in enumerate(shapes_of(pts, roff, poff, closed or not stroke)):
        n0 = s.n_draw_objects
        c = Color(*[float(v) for v in cols[i]])
        if stroke:
            s.stroke(style, Affine.IDENTITY, c, None, els)
        else:
            s.fill(style, Affine.IDENTITY, c, None, els)
        draw.append(n0 if s.n_draw_objects > n0 else -1)
    return s, draw


def dev(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def build(r, pts, roff, poff, cols, style=FILL_NON_ZERO, closed=True):
    n_paths = len(poff) - 1 if poff is not None else len(roff) - 1
    idx = torch.full((n_paths,), -7, dtype=torch.int32, device="cuda")
    fid, n = r.upload_device_paths(dev(pts.reshape(-1, 2), torch.float32), dev(roff, torch.int32), dev(cols.reshape(-1, 4), torch.float32),
                                   path_offsets=None if poff is None else dev(poff, torch.int32), style=style, closed=closed,
                                   draw_index=idx)
    return fid, n, idx.cpu().numpy()


def composed(r, instances):
    lay, offs = r.compose(instances)
    return lay, offs, r.download("scene", np.uint32)


def frame(r, aa):
    p = RenderParams(BASE, W, H, aa)
    r.render_resident(p)
    return r.download_target(p)


def check(r, pts, roff, poff, cols, style=FILL_NON_ZERO, closed=True, frames=True, native=False, aas=(AA_MSAA8, AA_MSAA16, AA_AREA)):
    """Build both fragments, compare the composed scenes word for word and, with `frames`, the frames in the AA modes `aas`."""
    pts = np.asarray(pts, dtype=np.float32).reshape(-1, 2)
    cols = np.asarray(cols, dtype=np.float32).reshape(-1, 4)
    fid, n, idx = build(r, pts, roff, poff, cols, style, closed)
    scene, want_idx = reference(pts, roff, poff, cols, style, closed, native)
    ref = r.upload_fragment(scene)
    try:
        assert n == scene.n_draw_objects
        assert list(idx) == want_idx
        lay, offs, words = composed(r, [(fid, None)])
        imgs = [frame(r, aa) for aa in aas] if frames else []
        lay_ref, offs_ref, words_ref = composed(r, [(ref, None)])
        assert (lay.as_array() == lay_ref.as_array()).all(), f"layout {lay} != {lay_ref}"
        assert offs == offs_ref
        assert words.size == words_ref.size, f"{words.size} words, want {words_ref.size}"
        diff = np.nonzero(words != words_ref)[0]
        assert diff.size == 0, f"scene words differ at {diff[:8]}: {words[diff[:8]]} != {words_ref[diff[:8]]}"
        for img, aa in zip(imgs, aas):
            assert (img == frame(r, aa)).all(), f"aa {aa}"
    finally:
        r.free_fragment(fid)
        r.free_fragment(ref)
    return idx


def ragged(rng, n_paths, rings_per_path, pts_per_ring, scale=200.0, offset=28.0):
    """Random polygons: per path 0..rings_per_path rings of 0..pts_per_ring points around a centre."""
    roff, poff, pts = [0], [0], []
    for _ in range(n_paths):
        nr = int(rng.integers(0, rings_per_path + 1))
        cx, cy = rng.uniform(offset, offset + scale, 2)
        for _ in range(nr):
            k = int(rng.integers(0, pts_per_ring + 1))
            t = np.sort(rng.uniform(0, 2 * np.pi, k))
            rad = rng.uniform(3, 30, k)
            pts += list(zip(cx + rad * np.cos(t), cy + rad * np.sin(t)))
            roff.append(len(pts))
        poff.append(len(roff) - 1)
    cols = rng.uniform(0, 1, (n_paths, 4))
    return np.array(pts, np.float32).reshape(-1, 2), np.array(roff, np.int32), np.array(poff, np.int32), cols.astype(np.float32)


SQUARE = [(40, 40), (200, 40), (200, 200), (40, 200)]
HOLE = [(80, 80), (80, 160), (160, 160), (160, 80)]


# ---- fills and strokes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule", [FILL_NON_ZERO, FILL_EVEN_ODD])
def test_fills_with_holes(r, rule):
    pts = SQUARE + HOLE + [(10, 10), (60, 20), (30, 70)]
    check(r, pts, [0, 4, 8, 11], [0, 2, 3], [[1, 0.2, 0.1, 1], [0.1, 0.7, 0.9, 0.6]], rule)


@pytest.mark.parametrize("join", [STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND])
@pytest.mark.parametrize("caps", [(STYLE_CAP_BUTT, STYLE_CAP_SQUARE), (STYLE_CAP_ROUND, STYLE_CAP_BUTT), (STYLE_CAP_SQUARE, STYLE_CAP_ROUND)])
@pytest.mark.parametrize("closed", [False, True])
def test_strokes(r, join, caps, closed):
    pts = [(30, 30), (120, 50), (60, 140), (200, 200), (20, 220), (220, 20), (230, 100)]
    check(r, pts, [0, 4, 7], None, [[0.9, 0.3, 0.2, 1.0], [0.2, 0.9, 0.4, 0.7]],
          Stroke(6.0, join, 2.5, caps[0], caps[1]), closed)


@pytest.mark.parametrize("style", [FILL_NON_ZERO, Stroke(3.0)], ids=["fill", "stroke"])
@pytest.mark.parametrize("closed", [False, True])
def test_degenerate_rings_and_paths(r, style, closed):
    """Consecutive duplicates; rings of 0, 1 and 2 points and rings of one point repeated; paths of no ring and paths whose
    rings all encode nothing; the closing point bit-equal, value-equal (-0 against +0) and different."""
    rings = [
        [(50, 50), (50, 50), (90, 50), (90, 50), (90, 50), (90, 90), (90, 90), (50, 50)],  # duplicates, closing point bit-equal
        [], [(10, 10)], [(10, 10), (30, 40)], [(7, 7)] * 5,
        [(0.0, 20.0), (40, 20), (40, 60), (-0.0, 20.0)],  # closing point value-equal only
        [(100, 100), (140, 100), (140, 150), (101, 100)],  # closing point different
        [(60, 60), (60, 60)], [], [(5, 5)],
    ]
    pts, roff = [], [0]
    for ring in rings:
        pts += ring
        roff.append(len(pts))
    poff = [0, 1, 1, 3, 5, 7, 7, 10]  # paths: [0] [] [1 2] [3 4] [5 6] [] [7 8 9]
    cols = np.random.default_rng(1).uniform(0, 1, (7, 4))
    idx = check(r, pts, roff, poff, cols, style, closed)
    assert idx[1] == -1 and idx[5] == -1 and idx[6] == -1


@pytest.mark.parametrize("style", [FILL_NON_ZERO, Stroke(0.5)], ids=["fill", "stroke"])
@pytest.mark.parametrize("closed", [False, True])
def test_eps_close_points_near_zero(r, style, closed):
    """Neighbouring points EPS-close but unequal (below 1.7e-5 in magnitude): the keep rule is the encoders' walk, not the
    neighbour test. Also caps whose markers fall within EPS of the ring's end."""
    e = np.float32(4e-13)
    rings = [
        [(0, 0), (e, 0), (2 * e, 0), (3 * e, 0), (4 * e, 0), (5 * e, e)],  # each step below EPS, the walk keeps some
        [(1e-6, 1e-6), (1e-6 + 1e-13, 1e-6), (3e-12, 0), (1e-12, 0)],
        [(0, 0), (3e-12, 0), (1e-12, 0)],  # the open cap marker within EPS of the ring's end
        [(-0.0, 0.0), (0.0, -0.0), (0.0, 0.0), (2e-12, 0)],
        [(10, 10), (60, 10), (60, 60)],
    ]
    pts, roff = [], [0]
    for ring in rings:
        pts += ring
        roff.append(len(pts))
    check(r, pts, roff, None, np.full((len(rings), 4), 0.5), style, closed, frames=False)


def test_no_paths(r):
    fid, n, idx = build(r, np.zeros((0, 2), np.float32), np.array([0], np.int32), None, np.zeros((0, 4), np.float32))
    assert n == 0 and idx.size == 0
    lay, _, words = composed(r, [(fid, None)])
    lay_ref, _, words_ref = composed(r, [])
    r.free_fragment(fid)
    assert (lay.as_array() == lay_ref.as_array()).all() and (words == words_ref).all()


@pytest.mark.parametrize("n", [31, 32, 33, 255, 256, 257, 511, 512, 513, 256 * 33 + 7])
def test_partition_boundaries(r, n):
    """Rings and paths ending on and beside warp, CTA and look-back partition boundaries (256 points a partition)."""
    rng = np.random.default_rng(n)
    t = np.linspace(0, 2 * np.pi, n, endpoint=False)
    ring = np.stack([128 + 100 * np.cos(t), 128 + 100 * np.sin(t)], 1)
    ring[rng.integers(0, n, n // 5)] = ring[0]  # some duplicates
    small = rng.uniform(20, 230, (n, 2))
    pts = np.concatenate([ring, small])
    roff = np.array([0, n] + list(range(n + 3, 2 * n, 3)) + [2 * n], np.int32)
    poff = np.array([0, 1] + list(range(2, len(roff) - 1, 4)) + [len(roff) - 1], np.int32)
    cols = rng.uniform(0, 1, (len(poff) - 1, 4))
    check(r, pts, roff, poff, cols, FILL_EVEN_ODD)
    check(r, pts, roff, poff, cols, Stroke(1.5), False, frames=False)


def test_million_point_polyline(r):
    rng = np.random.default_rng(3)
    n = 1_000_000
    x = np.linspace(4, 252, n)
    y = 128 + 100 * np.sin(x / 9.0) + rng.normal(0, 2, n)
    pts = np.stack([x, y], 1)
    pts[1000:1010] = pts[999]  # a run of duplicates
    # area coverage sums a tile's segments in an order the pipeline does not fix: with a million segments in 256 x 256 pixels
    # two frames of the same words may differ in the last bit there, so the frames are compared in the MSAA modes
    check(r, pts, np.array([0, n], np.int32), None, [[1, 1, 0.2, 1]], Stroke(1.0), False, native=True, aas=(AA_MSAA8, AA_MSAA16))


def test_random_polygons(r):
    pts, roff, poff, cols = ragged(np.random.default_rng(5), 30_000, 3, 12)
    check(r, pts, roff, poff, cols, FILL_NON_ZERO, native=True)


# ---- composition -----------------------------------------------------------------------------------------------------------
def host_fragment(r):
    s = NativeScene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.3, 0.8, 1.0), None, Rect(10, 10, 120, 90))
    s.stroke(Stroke(4.0), Affine.translate(30, 40), Color(0.9, 0.5, 0.1, 1.0), None, Circle(60, 60, 30))
    return r.upload_fragment(s)


def test_beside_host_fragments(r):
    """A device fragment among host fragments, with instance transforms, bound instance transforms and a view, hit tests at an
    interior point of each path, bound colours on its rows, and the frames against the same composition of its host twin."""
    pts = np.array(SQUARE + HOLE + [(10, 10), (60, 20), (30, 70)], np.float32) * 0.5
    roff, poff = np.array([0, 4, 8, 11], np.int32), np.array([0, 2, 3], np.int32)
    cols = np.array([[1, 0.2, 0.1, 1], [0.1, 0.7, 0.9, 0.6]], np.float32)
    fid, n, idx = build(r, pts, roff, poff, cols, FILL_NON_ZERO)
    ref = r.upload_fragment(reference(pts, roff, poff, cols, FILL_NON_ZERO, True)[0])
    base = host_fragment(r)
    xf = [None, Affine.translate(100, 20), Affine.translate(30, 140) * Affine.rotate(0.3)]
    try:
        for view in (None, Affine.scale(1.3)):
            r.set_view(view)
            outs = []
            for f in (fid, ref):
                lay, offs = r.compose([(base, xf[0]), (f, xf[1]), (base, xf[2])])
                outs.append((lay.as_array(), offs, r.download("scene", np.uint32), [frame(r, aa) for aa in (AA_MSAA16, AA_AREA)]))
            assert (outs[0][0] == outs[1][0]).all() and outs[0][1] == outs[1][1] and (outs[0][2] == outs[1][2]).all()
            for a, b in zip(outs[0][3], outs[1][3]):
                assert (a == b).all()
        r.set_view(None)
        lay, offs = r.compose([(base, xf[0]), (fid, xf[1]), (base, xf[2])])
        frame(r, AA_MSAA16)
        # interior points: path 0 between the square and the hole, path 1 inside its triangle (both moved by xf[1])
        pts_in = np.array([[25 + 100, 30 + 20], [16 + 100, 16 + 20]], np.float32)
        got = r.hit_test(pts_in)
        assert list(got) == [offs[1] + idx[0], offs[1] + idx[1]]
        # bound instance transforms and bound colours on the device fragment's rows
        t = torch.tensor([[1, 0, 0, 1, 0, 0], [1, 0, 0, 1, 100, 20], [1, 0, 0, 1, 30, 140]], dtype=torch.float32, device="cuda")
        r.bind_instance_transforms(t)
        rows = torch.full((offs[2], 4), float("nan"), device="cuda")
        rows[offs[1] + int(idx[1])] = torch.tensor([0.0, 1.0, 0.0, 1.0])
        r.bind_draw_colors(rows)
        img = frame(r, AA_MSAA16)
        r.bind_draw_colors(None)
        r.bind_instance_transforms(None)
        cols2 = cols.copy()
        cols2[1] = [0, 1, 0, 1]
        ref2 = r.upload_fragment(reference(pts, roff, poff, cols2, FILL_NON_ZERO, True)[0])
        r.compose([(base, None), (ref2, Affine.translate(100, 20)), (base, Affine.translate(30, 140))])
        assert (img == frame(r, AA_MSAA16)).all()
        r.free_fragment(ref2)
    finally:
        r.set_view(None)
        for f in (fid, ref, base):
            r.free_fragment(f)


def test_recompose_rebuilt_overlay(r):
    """An overlay rebuilt from device arrays and swapped in by recompose damages only its boxes, and the damage-tracked frame
    equals a full frame of the same composition."""
    rng = np.random.default_rng(9)
    base = host_fragment(r)
    pts, roff, poff, cols = ragged(rng, 6, 2, 8, scale=40, offset=170)
    a, _, _ = build(r, pts, roff, poff, cols)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.set_damage_tracking(True)
    try:
        r.compose([(base, None), (a, None)])
        r.render_resident(p)
        r.render_resident(p)
        pts2 = pts + np.float32(3.0)
        b, _, _ = build(r, pts2, roff, poff, cols)
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
            r.free_fragment(f)


# ---- the allocation ---------------------------------------------------------------------------------------------------------
def held(r, base):
    """The device memory the renderer holds (frame stats' arena_bytes, which count every fragment's allocation), once the
    fragments freed so far are released: a compose after the device is idle reaps them."""
    torch.cuda.synchronize()
    r.compose([(base, None)])
    return int(r.render_resident(RenderParams(BASE, W, H, AA_MSAA16)).arena_bytes)


def fragment_bytes(units):
    """A fragment's allocation for streams of `units` (tag bytes, words, draw tags, words, transforms, style words): the
    header, the streams with the tags padded to words, 4 words of slack, rounded up to 16 bytes (vb_fragment_upload's)."""
    words = 8 + (units[0] + 3) // 4 + units[1] + units[2] + units[3] + 6 * units[4] + units[5]
    return ((words + 4) * 4 + 15) // 16 * 16


@pytest.mark.parametrize("style", [FILL_NON_ZERO, Stroke(2.0)], ids=["fill", "stroke"])
def test_allocation_is_the_worst_case(r, style):
    """The fragment holds exactly the allocation the worst case of its counts asks for (the formula tests/test_device_paths.py
    checks against the host encoder), and its streams lie inside it."""
    from .test_device_paths import worst_case
    pts, roff, poff, cols = ragged(np.random.default_rng(11), 40, 3, 9)
    pts[5:9] = pts[4]  # duplicates
    base = host_fragment(r)
    try:
        f, _, _ = build(r, pts, roff, poff, cols, style, False)  # sizes the scratch, which must not grow below
        r.free_fragment(f)
        held(r, base)
        a0 = held(r, base)
        f, n, _ = build(r, pts, roff, poff, cols, style, False)
        a1 = held(r, base)
        bound = worst_case(len(pts), len(roff) - 1, len(poff) - 1)
        assert a1 - a0 == fragment_bytes(bound)
        lay, _ = r.compose([(f, None)])
        assert lay.draw_tag_base - lay.path_data_base <= bound[1] and n <= bound[2]
        r.free_fragment(f)
    finally:
        r.free_fragment(base)


# ---- errors ----------------------------------------------------------------------------------------------------------------
def test_errors_leave_no_fragment(r):
    """Every refusal, from the Python checks, the library's host checks and its device checks, leaves the installed scene as
    it was, makes no fragment (no id is taken and no device memory is kept) and lets the next valid call succeed."""
    from vello_b200.renderer import _DevicePaths
    import ctypes as C
    base = host_fragment(r)
    pts = dev(np.array(SQUARE, np.float32), torch.float32)
    cols = dev(np.ones((1, 4), np.float32), torch.float32)
    no_cols = dev(np.ones((0, 4), np.float32), torch.float32)
    good = dev(np.array([0, 4], np.int32), torch.int32)
    f0, _ = r.upload_device_paths(pts, dev(np.array([0, 1, 2, 4], np.int32), torch.int32), dev(np.ones((3, 4), np.float32), torch.float32))
    r.free_fragment(f0)  # the scratch now holds every case below
    held(r, base)
    a0 = held(r, base)
    before = r.download("scene", np.uint32)
    nan_pts = pts.clone()
    nan_pts[2, 1] = float("inf")
    nan_cols = cols.clone()
    nan_cols[0, 3] = float("nan")
    i32 = lambda *v: dev(np.array(v, np.int32), torch.int32)  # noqa: E731
    cases = [
        (dict(points=pts, ring_offsets=i32(1, 4), colors=cols), "ring_offsets[0]"),
        (dict(points=pts, ring_offsets=i32(0, 3, 2, 4), colors=dev(np.ones((3, 4), np.float32), torch.float32)), "ring_offsets[2]"),
        (dict(points=pts, ring_offsets=i32(0, 3), colors=cols), "ring_offsets[1]"),
        (dict(points=pts, ring_offsets=i32(0), colors=no_cols), "ring_offsets[0]"),  # points but no ring
        (dict(points=pts, ring_offsets=good, colors=cols, path_offsets=i32(0, 2)), "path_offsets[1]"),
        (dict(points=pts, ring_offsets=good, colors=cols, path_offsets=i32(1, 1)), "path_offsets[0]"),
        (dict(points=pts, ring_offsets=good, colors=no_cols, path_offsets=i32(0)), "path_offsets[0]"),  # rings but no path
        (dict(points=nan_pts, ring_offsets=good, colors=cols), "point 2"),
        (dict(points=pts, ring_offsets=good, colors=nan_cols), "colour of path 0"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=7), "fill_rule"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=Stroke(float("inf"))), "width"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=Stroke(0.0)), "width"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=Stroke(1.0, join=3)), "join"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=Stroke(1.0, start_cap=5)), "caps"),
        (dict(points=pts, ring_offsets=good, colors=cols, style=Stroke(1.0, miter_limit=float("nan"))), "miter"),
        (dict(points=pts.cpu(), ring_offsets=good, colors=cols), None),
    ]
    for kw, why in cases:
        with pytest.raises((VelloB200Error, TypeError)) as e:
            r.upload_device_paths(kw.pop("points"), kw.pop("ring_offsets"), kw.pop("colors"), **kw)
        if why is not None:
            assert why in str(e.value), str(e.value)
        assert (r.download("scene", np.uint32) == before).all(), "the previous scene stays"

    # host memory through a raw pointer: refused by the library, not just the Python checks
    class _Host:
        def __init__(self, a):
            self.a = a
            self.__cuda_array_interface__ = dict(shape=a.shape, typestr="<f4", data=(a.ctypes.data, False), version=2, strides=None)
    with pytest.raises(VelloB200Error, match="device or managed memory"):
        r.upload_device_paths(_Host(np.array(SQUARE, np.float32)), good, cols)

    # the library's own host checks, reached through the C ABI with what the Python checks would refuse
    def raw(**fields):
        d = _DevicePaths(pts.data_ptr(), 4, 8, good.data_ptr(), 1, None, 1, cols.data_ptr(), 16)
        for k, v in fields.items():
            setattr(d, k, v)
        fid, n = C.c_uint32(0), C.c_uint32(0)
        rc = r.lib.vb_fragment_from_device_paths(r.handle, C.byref(d), C.byref(fid), C.byref(n))
        return rc, fid.value, r.lib.vb_last_error(r.handle).decode()
    for fields, why in [
        (dict(point_pitch_bytes=6), "point pitch"), (dict(point_pitch_bytes=10), "point pitch"),
        (dict(point_pitch_bytes=1 << 32), "point pitch"), (dict(color_pitch_bytes=12), "colour pitch"),
        (dict(color_pitch_bytes=18), "colour pitch"), (dict(points=pts.data_ptr() + 2), "4-byte aligned"),
        (dict(points=None), "NULL"), (dict(ring_offsets=None), "NULL"), (dict(colors=None), "NULL"),
        (dict(n_paths=2), "n_paths must equal n_rings"), (dict(n_points=1 << 31), "int32"), (dict(kind=2), "kind"),
    ]:
        rc, fid, msg = raw(**fields)
        assert rc != 0 and why in msg, (fields, msg)
    assert (r.download("scene", np.uint32) == before).all()
    assert held(r, base) == a0, "a refused call keeps no device memory"
    fid, n = r.upload_device_paths(pts, good, cols)  # the next valid call succeeds, with the next id: no refusal took one
    assert n == 1 and fid == f0 + 1
    r.free_fragment(fid)
    r.free_fragment(base)
