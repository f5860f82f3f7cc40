"""Dashed fragments from device arrays (Renderer.upload_device_dashes, vb_fragment_from_device_dashes): the fragment built on
the device must be word for word the fragment `upload_fragment` makes of the Scene that strokes each path with its colour and
the dashed Stroke, its shape being, per ring of two or more points, M, the segments, and Z when closed. Every case composes
both fragments and compares the composed scene's words, layout and draw offsets, and the frames. Run on an H100 with
`pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16
from vello_b200.encoding import (Color, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER,
                                 STYLE_JOIN_ROUND, Scene, Stroke)
from vello_b200.renderer import Renderer
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Arc, Circle, Ellipse, RoundedRect
from vello_b200.renderer import _DevicePaths, _Dash

from . import device_dashes_ref as ref
from .test_gpu_device_curves import cols_for, join_paths, shape_rings
from .test_gpu_device_paths import BASE, composed, dev, frame, held, host_fragment

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def r():
    r = Renderer()
    yield r
    r.close()


def with_offset(stroke, off):
    return Stroke(stroke.width, stroke.join, stroke.miter_limit, stroke.start_cap, stroke.end_cap, stroke.dash_pattern, off)


def reference(pts, kinds, roff, poff, cols, stroke, closed, offsets, native=False):
    """(the host Scene, each path's draw object or -1)"""
    s = NativeScene() if native else Scene()
    draw = []
    for i in range(len(poff) - 1):
        n0 = s.n_draw_objects
        off = stroke.dash_offset if offsets is None else float(offsets[i])
        s.stroke(with_offset(stroke, off), Affine.IDENTITY, Color(*[float(v) for v in cols[i]]), None,
                 ref.shape(pts, kinds, roff, poff, i, closed))
        draw.append(n0 if s.n_draw_objects > n0 else -1)
    return s, draw


def check(r, pts, kinds, roff, poff, cols, stroke, closed=True, offsets=None, frames=True, native=False,
          aas=(AA_MSAA8, AA_MSAA16, AA_AREA)):
    pts = np.asarray(pts, dtype=np.float32).reshape(-1, 2)
    kinds = np.asarray(kinds, np.uint8)
    roff, poff = np.asarray(roff, np.int32), np.asarray(poff, np.int32)
    cols = np.asarray(cols, dtype=np.float32).reshape(-1, 4)
    offsets = None if offsets is None else np.asarray(offsets, np.float32)
    idx = torch.full((len(poff) - 1,), -7, dtype=torch.int32, device="cuda")
    fid, n = r.upload_device_dashes(dev(pts, torch.float32), dev(roff, torch.int32), dev(cols, torch.float32), stroke,
                                    path_offsets=dev(poff, torch.int32), closed=closed, draw_index=idx,
                                    point_kinds=dev(kinds, torch.uint8),
                                    dash_offsets=None if offsets is None else dev(offsets, torch.float32))
    idx = idx.cpu().numpy()
    scene, want_idx = reference(pts, kinds, roff, poff, cols, stroke, closed, offsets, native)
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


def polylines(seed, n_paths, n_pts=12, spread=200.0):
    rng = np.random.default_rng(seed)
    paths = []
    for _ in range(n_paths):
        rings = []
        for _ in range(int(rng.integers(1, 3))):
            p = rng.uniform(20, 20 + spread, (int(rng.integers(2, n_pts)), 2)).astype(np.float32)
            rings.append((p, [0] * len(p)))
        paths.append(rings)
    return join_paths(paths)


# ---- polylines: joins, caps, patterns, open and closed ------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", [(10.0, 5.0), (0.0, 8.0), (6.0, 3.0, 2.0), (1000.0, 1.0)], ids=["10_5", "dots", "odd", "long"])
@pytest.mark.parametrize("closed", [False, True], ids=["open", "closed"])
@pytest.mark.parametrize("join, cap", [(STYLE_JOIN_BEVEL, STYLE_CAP_BUTT), (STYLE_JOIN_MITER, STYLE_CAP_SQUARE),
                                       (STYLE_JOIN_ROUND, STYLE_CAP_ROUND)], ids=["bevel_butt", "miter_square", "round_round"])
def test_polylines(r, pattern, closed, join, cap):
    pts, kinds, roff, poff = polylines(3, 6)
    stroke = Stroke(3.0, join, 4.0, cap, cap, pattern, 2.5)
    check(r, pts, kinds, roff, poff, cols_for(len(poff) - 1), stroke, closed, native=pattern == (10.0, 5.0))


@pytest.mark.parametrize("pattern", [(10.0, 5.0), (0.0, 8.0), (6.0, 3.0, 2.0), (1000.0, 1.0)], ids=["10_5", "dots", "odd", "long"])
def test_kurbo_shapes(r, pattern):
    """Circles, ellipses, rounded rectangles and arcs: curved pieces, and the curved segment after Z of a ring in one dash."""
    shapes = [Circle(70, 70, 40), Ellipse(170, 80, 60, 25, 0.5), RoundedRect(20, 140, 120, 230, 18), Arc(180, 180, 50, 35, 0.4, 4.2)]
    pts, kinds, roff, poff = join_paths([shape_rings(s) for s in shapes])
    stroke = Stroke(2.5, STYLE_JOIN_ROUND, 4.0, STYLE_CAP_ROUND, STYLE_CAP_BUTT, pattern, -1.5)
    for closed in (False, True):
        check(r, pts, kinds, roff, poff, cols_for(len(poff) - 1, 2), stroke, closed, native=closed)


def test_curved_tail_after_the_close(r):
    pts = np.array([(7.5, 9.5), (40, 30), (5, 3), (5, 3), (7.5, 9.5), (100, 100), (180, 120), (140, 200), (100, 100)], np.float32)
    kinds = [0, 1, 0, 1, 0, 0, 1, 1, 0]
    stroke = Stroke(2.0, dash_pattern=(100.0, 1.0))
    check(r, pts, kinds, [0, 5, 9], [0, 1, 2], cols_for(2), stroke, True)
    check(r, pts, kinds, [0, 5, 9], [0, 2], cols_for(1), stroke, True)


def test_multi_ring_paths_with_short_and_empty_rings(r):
    P = [(10, 10), (90, 10), (90, 90), (50, 50), (50, 50), (120, 30), (200, 40), (210, 120), (30, 200), (60, 230)]
    roff = [0, 3, 4, 4, 5, 8, 8, 10]
    for closed in (False, True):
        check(r, P, [0] * len(P), roff, [0, 2, 4, 7], cols_for(3), Stroke(2.0, dash_pattern=(7.0, 4.0), dash_offset=3.0), closed)


def test_per_path_offsets_and_dropped_paths(r):
    pts, kinds, roff, poff = polylines(9, 40)
    offs = np.random.default_rng(4).uniform(-50, 50, len(poff) - 1).astype(np.float32)
    offs[:4] = [0.0, 15.0, -15.0, 1e4]
    check(r, pts, kinds, roff, poff, cols_for(len(poff) - 1), Stroke(2.0, dash_pattern=(10.0, 5.0)), True, offsets=offs)
    # zero-length dashes with butt caps: every piece is dropped, so those paths draw nothing (-1)
    idx = check(r, pts, kinds, roff, poff, cols_for(len(poff) - 1),
                Stroke(2.0, STYLE_JOIN_BEVEL, 4.0, STYLE_CAP_BUTT, STYLE_CAP_BUTT, (0.0, 8.0)), False)
    assert (idx == -1).all()


def test_long_ring(r):
    """A 100k-point ring, walked by one warp."""
    t = np.linspace(0, 40 * np.pi, 100_000)
    p = np.stack([128 + 100 * np.cos(t) * (0.3 + t / 200), 128 + 100 * np.sin(t) * (0.3 + t / 200)], 1).astype(np.float32)
    check(r, p, [0] * len(p), [0, len(p)], [0, 1], cols_for(1), Stroke(1.0, dash_pattern=(4.0, 4.0)), False,
          aas=(AA_MSAA8, AA_MSAA16))


def test_random_polygons(r):
    pts, kinds, roff, poff = polylines(21, 2000, n_pts=8, spread=230.0)
    check(r, pts, kinds, roff, poff, cols_for(len(poff) - 1), Stroke(1.0, dash_pattern=(6.0, 3.0)), True, frames=False)


def test_allocation_is_the_worst_case_of_the_intermediate(r):
    pts, kinds, roff, poff = polylines(5, 8)
    pattern, off = (5.0, 2.0), 1.0
    mid = ref.intermediate(pts, kinds, roff, poff, True, pattern, [off] * (len(poff) - 1))
    base = host_fragment(r)
    before = held(r, base)
    fid, _ = r.upload_device_dashes(dev(pts, torch.float32), dev(roff, torch.int32), dev(cols_for(len(poff) - 1), torch.float32),
                                    Stroke(2.0, dash_pattern=pattern, dash_offset=off), path_offsets=dev(poff, torch.int32))
    from .test_device_paths import worst_case
    P, R, N = len(mid[0]), len(mid[2]) - 1, len(poff) - 1
    units = worst_case(P, R, N)
    words = 8 + (units[0] + 3) // 4 + units[1] + units[2] + units[3] + 6 * units[4] + units[5]
    want = ((words + 4) * 4 + 15) & ~15
    try:
        assert held(r, base) - before == want
    finally:
        r.free_fragment(fid)
        r.free_fragment(base)


def test_recompose_beside_a_host_fragment(r):
    base = host_fragment(r)
    pts, kinds, roff, poff = polylines(11, 10)
    cols = dev(cols_for(len(poff) - 1), torch.float32)
    ids = []
    try:
        for off in (0.0, 1.5, 3.0):
            fid, _ = r.upload_device_dashes(dev(pts, torch.float32), dev(roff, torch.int32), cols,
                                            Stroke(2.0, dash_pattern=(6.0, 3.0), dash_offset=off), path_offsets=dev(poff, torch.int32))
            ids.append(fid)
            r.recompose([(base, None), (fid, None)])
            img = frame(r, AA_MSAA16)
            s, _ = reference(pts, kinds, roff, poff, cols.cpu().numpy(), Stroke(2.0, dash_pattern=(6.0, 3.0)), True, [off] * (len(poff) - 1))
            hid = r.upload_fragment(s)
            r.compose([(base, None), (hid, None)])
            assert (img == frame(r, AA_MSAA16)).all()
            r.free_fragment(hid)
    finally:
        for f in ids + [base]:
            r.free_fragment(f)


# ---- refusals: each leaves no fragment and the renderer as it was ---------------------------------------------------------------
def call(r, d, dash, kinds=None):
    fid, n = C.c_uint32(0), C.c_uint32(0)
    rc = r.lib.vb_fragment_from_device_dashes(r.handle, C.byref(d), kinds, C.byref(dash) if dash is not None else None,
                                              C.byref(fid), C.byref(n))
    return rc, r.lib.vb_last_error(r.handle).decode()


def test_refusals_leave_no_fragment(r):
    base = host_fragment(r)
    P = dev(np.array([(10, 10), (50, 10), (50, 50)], np.float32), torch.float32)
    R = dev(np.array([0, 3], np.int32), torch.int32)
    Cl = dev(cols_for(1), torch.float32)
    fid, _ = r.upload_device_dashes(P, R, Cl, Stroke(2.0, dash_pattern=(4.0, 2.0)))  # sizes the renderer's scratch buffers
    r.free_fragment(fid)
    before = held(r, base)

    def paths(kind=1):
        d = _DevicePaths(C.c_void_p(P.data_ptr()), 3, 8, C.c_void_p(R.data_ptr()), 1, None, 1, C.c_void_p(Cl.data_ptr()), 16)
        d.kind, d.width, d.miter_limit, d.join, d.start_cap, d.end_cap, d.closed = kind, 2.0, 4.0, 0, 0, 0, 1
        return d

    def dash(pattern=(4.0, 2.0), offset=0.0, offsets=None, pitch=4):
        arr = (C.c_double * max(len(pattern), 1))(*pattern)
        dash._keep = arr
        return _Dash(C.cast(arr, C.c_void_p) if pattern else None, len(pattern), offset, offsets, pitch)

    bad_off = dev(np.array([np.inf], np.float32), torch.float32)
    far_off = dev(np.array([1e30], np.float32), torch.float32)
    cases = [
        (paths(), None, "NULL dash"),
        (paths(0), dash(), "kind must be 1"),
        (paths(), dash(()), "empty"),
        (paths(), dash((1.0, -1.0)), ">= 0"),
        (paths(), dash((1.0, float("nan"))), ">= 0"),
        (paths(), dash((0.0, 0.0)), "sum to 0"),
        (paths(), dash(offset=float("inf")), "dash offset"),
        (paths(), dash(pattern=(1e-30, 1e-30), offset=1.0), "dash offset"),
        (paths(), dash((1e-9, 1e-9)), "2^31 dash breaks"),  # refused by the bound, before any walk
        (paths(), dash(offsets=C.c_void_p(bad_off.data_ptr() + 2)), "aligned"),
        (paths(), dash(offsets=C.c_void_p(bad_off.data_ptr()), pitch=2), "pitch"),
        (paths(), dash(offsets=C.c_void_p(bad_off.data_ptr())), "path 0 is not finite"),
        (paths(), dash(offsets=C.c_void_p(far_off.data_ptr())), "path 0 is not finite"),
    ]
    for d, ds, match in cases:
        rc, msg = call(r, d, ds)
        assert rc != 0 and match in msg, (match, msg)
    bad_roff = dev(np.array([0, 2], np.int32), torch.int32)
    d = paths()
    d.ring_offsets = C.c_void_p(bad_roff.data_ptr())
    rc, msg = call(r, d, dash())
    assert rc != 0 and "ring_offsets[1]" in msg
    with pytest.raises(ValueError, match="dashed"):
        r.upload_device_paths(P, R, Cl, style=Stroke(2.0, dash_pattern=(1.0, 1.0)))
    assert held(r, base) == before
    r.free_fragment(base)
