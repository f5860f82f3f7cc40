"""Bound stroke widths (Renderer.bind_stroke_widths, vb_bind_stroke_widths): every frame strokes draw object k with the width in
row k of a device array, read when the frame runs. `r` binds; `ref` renders the host route on the same GPU: the packed scene
with the bound strokes' width words patched in (every stroke with a style entry of its own), or the scene re-encoded with those
widths. Run on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, DRAWTAG_BEGIN_CLIP, DRAWTAG_END_CLIP, FILL_NON_ZERO, MIX_MULTIPLY, STYLE_CAP_BUTT,
                                 STYLE_CAP_ROUND, STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Color, Gradient,
                                 Image, Packed, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Arc, BezPath, Circle, Line, Rect, RoundedRect

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_draw_colors import box_tiles
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels
from .test_gpu_path_points import points
from .test_gpu_transforms import transforms
from .test_gpu_visibility import build, flags_of, frame, on_device, same, sorted_lines
from .test_stroke_widths import draw_styles

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
IMG = np.random.default_rng(41).integers(0, 256, (16, 20, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (0.6, Color(0.2, 0.9, 0.3, 0.8)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]
JOINS = [STYLE_JOIN_ROUND, STYLE_JOIN_MITER, STYLE_JOIN_BEVEL]
CAPS = [STYLE_CAP_BUTT, STYLE_CAP_SQUARE, STYLE_CAP_ROUND]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


@pytest.fixture
def fresh():
    """Two new renderers: the ptcl holds offsets that follow a renderer's arena history."""
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


# ---- scenes as lists of calls, each of which encodes exactly one draw object -----------------------------------------------
def _shape(i, x, y):
    k = i % 6
    if k == 0:
        return Circle(x + 20, y + 20, 18)  # closed, cubics
    if k == 1:
        p = BezPath()
        p.move_to(x, y + 30), p.quad_to(x + 20, y - 10, x + 40, y + 30), p.quad_to(x + 50, y + 45, x + 30, y + 44)
        return p  # open quads
    if k == 2:
        p = BezPath()
        p.move_to(x, y), p.curve_to(x + 50, y, x - 10, y + 40, x + 40, y + 40), p.line_to(x + 5, y + 20), p.close_path()
        p.move_to(x + 45, y), p.line_to(x + 60, y + 10)
        return p  # a closed cubic subpath and an open line subpath
    if k == 3:
        return Arc(x + 20, y + 20, 22, 14, 0.3, 4.0)  # an open arc
    if k == 4:
        return RoundedRect(x, y, x + 45, y + 35, 7)
    return Line(x, y, x + 45, y + 30)


def stroke_of(i, w, dashed=None):
    dash = (7.0, 4.0) if (i % 4 == 3 if dashed is None else dashed) else ()
    return Stroke(float(w), join=JOINS[i % 3], miter_limit=[4.0, 10.0, 1.5][(i // 3) % 3], start_cap=CAPS[i % 3], end_cap=CAPS[(i + 1) % 3],
                  dash_pattern=dash)


def width_ops(seed=0, widths=None, dx=0.0, n=14, styles=None):
    """Strokes of every join, cap, miter limit, dashes, open and closed subpaths, quads, cubics and arcs, between fills, an
    image, a blurred rectangle, a gradient and a layer holding a stroke (whose END_CLIP's path takes the stroke's style). With `widths`
    None every stroke's width differs, so every stroke has a style entry of its own. Stroke i's join, caps, miter limit and
    dashes follow styles[i] (default i): strokes of equal width and equal `styles` share a style entry when consecutive."""
    g = np.random.default_rng(seed)
    widths = [1.0 + 0.73 * i for i in range(n)] if widths is None else widths
    styles = list(range(len(widths))) if styles is None else styles
    ops = []
    for i, w in enumerate(widths):
        x, y = dx + 15 + 62 * (i % 6), 15 + 70 * (i // 6)
        c = Color(*map(float, g.uniform(0.1, 1.0, 3)), 1.0)
        ops.append(("draw", lambda s, i=i, w=w, x=x, y=y, c=c, si=styles[i]: s.stroke(stroke_of(si, w), Affine.rotate(0.02 * i), c, None,
                                                                                      _shape(i, x, y))))
        if i % 5 == 1:
            ops.append(("draw", lambda s, x=x, y=y: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.2, 0.2, 0.7), None, Rect(x + 8, y + 8, x + 30, y + 25))))
        if i == 3:
            ops.append(("draw", lambda s: s.draw_image(Image(IMG), Affine.translate(dx + 300, 250) * Affine.scale(2.0))))
            ops.append(("draw", lambda s: s.draw_blurred_rounded_rect(Affine.translate(dx + 220, 240), Rect(0, 0, 60, 40), Color(0.2, 0.7, 0.4, 1.0), 8.0, 5.0)))
            ops.append(("draw", lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((dx, 0), (dx + 100, 0), STOPS), None, Rect(dx + 10, 290, 110, 315))))
        if i == 6:
            ops.append(("push", lambda s: s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.9, Affine.IDENTITY, Circle(dx + 120, 260, 55))))
            ops.append(("draw", lambda s: s.stroke(stroke_of(1, 4.321), Affine.IDENTITY, Color(0.1, 0.2, 0.9, 1.0), None, Circle(dx + 120, 260, 35))))
            ops.append(("pop", lambda s: s.pop_layer()))
    return ops


def strokes(packed):
    """Per draw object: whether its row applies (a stroke, not a layer's draw object), and its style entry."""
    L = packed.layout
    entry, stroke = draw_styles(packed)
    tags = np.asarray(packed.scene, dtype=np.uint32)[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects]
    return stroke & ~np.isin(tags, [DRAWTAG_BEGIN_CLIP, DRAWTAG_END_CLIP]), entry


def applies(packed, rows):
    is_stroke, _ = strokes(packed)
    rows = np.asarray(rows, dtype=np.float32)
    k = np.zeros(packed.layout.n_draw_objects, dtype=bool)
    k[:len(rows)] = is_stroke[:len(rows)] & np.isfinite(rows) & (rows > 0)
    return k


def patched(packed, rows):
    """The host route: the packed scene with the width word of each bound stroke's style entry replaced by its row's bits."""
    L = packed.layout
    _, entry = strokes(packed)
    scene = np.array(packed.scene, dtype=np.uint32)
    on = np.nonzero(applies(packed, rows))[0]
    assert len(set(entry[on].tolist())) == len(on), "bound strokes share a style entry"
    for k in on:
        scene[L.style_base + 2 * entry[k] + 1] = np.float32(rows[k]).view(np.uint32)
    return Packed(scene, L, packed.ramps, packed.atlas)


def snapshot_want(packed, rows):
    n = packed.layout.n_draw_objects
    want = np.zeros(max(n, packed.layout.n_paths), dtype=np.float32)
    a = applies(packed, rows)
    want[:n][a] = np.asarray(rows, dtype=np.float32)[:n][a[:len(rows)]] if a.any() else 0
    return want


def rand_widths(n, seed, lo=0.5, hi=9.0):
    return np.random.default_rng(seed).uniform(lo, hi, n).astype(np.float32)


def raw(r, name):
    return r.download(name, np.uint32)


# ---- 1. equality with the patched scene --------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_equals_the_patched_scene(fresh, aa):
    r, ref = fresh
    s, _ = build(width_ops(seed=1))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    pts = np.random.default_rng(3).uniform(0, [W, H], (4000, 2)).astype(np.float32)
    for seed, (lo, hi) in enumerate([(0.3, 2.0), (2.0, 12.0), (0.05, 30.0)]):
        rows = rand_widths(n, seed, lo, hi)
        r.bind_stroke_widths(on_device(rows))
        ref.upload(patched(packed, rows))
        img, st = frame(r, aa)
        want, ref_st = frame(ref, aa)
        assert (img == want).all(), seed
        assert st.lines == ref_st.lines
        for name in ("lines", "ptcl", "draw_bboxes"):
            assert np.array_equal(raw(r, name), raw(ref, name)), (name, seed)
        assert np.array_equal(r.download("stroke_widths", np.float32), snapshot_want(packed, rows))
        assert (r.hit_test(pts) == ref.hit_test(pts)).all()
        assert (r.hit_map() == ref.hit_map()).all()


def test_streams_and_native_installations(rr):
    """Scenes installed from their streams, by either front end, bind as packed ones do."""
    from vello_b200.scene_native import NativeScene
    r, ref = rr
    ops = width_ops(seed=2)
    s, _ = build(ops)
    ns, _ = build(ops, s=NativeScene())
    rows = rand_widths(s.n_draw_objects, 4)
    ref.upload(patched(resolve(s.encoding), rows))
    r.upload_scene(s)
    r.bind_stroke_widths(on_device(rows))
    assert (frame(r)[0] == frame(ref)[0]).all()
    ref.upload(patched(ns.resolve(), rows))
    ns.upload_device(r)
    r.bind_stroke_widths(on_device(rows))
    assert (frame(r)[0] == frame(ref)[0]).all()


def test_shared_entries_equal_the_reencoded_scene(rr):
    """Consecutive strokes of equal width share a style entry; rows still widen each one alone."""
    r, ref = rr
    enc = [3.0] * 4 + [5.0] * 3 + [2.0] * 5
    styles = [int(w) for w in enc]
    ops = width_ops(seed=5, widths=enc, styles=styles)
    s, _ = build(ops)
    n = s.n_draw_objects
    is_stroke, entry = strokes(resolve(s.encoding))
    assert len(set(entry[is_stroke].tolist())) < is_stroke.sum()
    # the strokes of the width list, in order (not the layer's own stroke, the draw after its push)
    ks = [k for k in np.nonzero(is_stroke)[0] if ops[k - 1][0] != "push"]
    assert len(ks) == len(enc)
    r.upload(resolve(s.encoding))
    for seed in range(3):
        g = np.random.default_rng(seed)
        new = [float(np.float32(w * g.uniform(0.3, 3.0))) for w in enc]
        ref.upload(resolve(build(width_ops(seed=5, widths=new, styles=styles))[0].encoding))
        rows = np.full(n, np.nan, dtype=np.float32)
        rows[ks] = new
        r.bind_stroke_widths(on_device(rows))
        for aa in (AA_MSAA8, AA_MSAA16, AA_AREA):
            img, st = frame(r, aa)
            want, ref_st = frame(ref, aa)
            same(img, want, aa)
            assert st.lines == ref_st.lines
            assert np.array_equal(sorted_lines(r), sorted_lines(ref)), (seed, aa)


# ---- 2. rows -----------------------------------------------------------------------------------------------------------------
def test_row_rules(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=6))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    ref.upload(packed)
    encoded, _ = frame(ref)
    is_stroke, _ = strokes(packed)
    rows = rand_widths(n, 7)
    # NaN, +-inf, 0 and negative rows fall back to the encoded width
    bad = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -3.0], dtype=np.float32)
    ks = np.nonzero(is_stroke)[0]
    rows[ks[:len(bad)]] = bad
    r.bind_stroke_widths(on_device(rows))
    ref.upload(patched(packed, rows))
    assert (frame(r)[0] == frame(ref)[0]).all()
    snap = r.download("stroke_widths", np.float32)
    assert (snap[ks[:len(bad)]] == 0).all() and np.array_equal(snap, snapshot_want(packed, rows))
    # rows of fills, images, blurred rectangles and layers change nothing
    other = np.where(is_stroke, np.nan, 25.0).astype(np.float32)
    r.bind_stroke_widths(on_device(other))
    assert (frame(r)[0] == encoded).all()
    assert not r.download("stroke_widths", np.float32).any()
    # a partial n: strokes from n on keep their encoded width
    m = n // 2
    r.bind_stroke_widths(on_device(rows[:m]))
    ref.upload(patched(packed, rows[:m]))
    assert (frame(r)[0] == frame(ref)[0]).all()
    assert not r.download("stroke_widths", np.float32)[m:].any()
    # strided columns, (n, 1) and 1-D tensors
    ref.upload(patched(packed, rows))
    want, _ = frame(ref)
    state = torch.zeros((n, 7), dtype=torch.float32, device="cuda")
    state[:, 5] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    for t in (state[:, 5], state[:, 5:6], on_device(rows[:, None]), on_device(rows)):
        r.bind_stroke_widths(t)
        assert (frame(r)[0] == want).all()


def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=8))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [rand_widths(n, 100 + j, 0.2, 10.0) for j in range(20)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(n, dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_stroke_widths(t)
    caps = None
    for j, rows in enumerate(seq):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        assert st.kernel_launches <= unbound + 1
        if j % 5 == 0:
            ref.upload(patched(packed, rows))
            assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    t2 = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    t2[:, 1] = t
    torch.cuda.synchronize()
    r.bind_stroke_widths(t2[:, 1])  # another pointer and pitch is another key
    r.render_resident(p)
    assert r.debug_graph_captures() == caps + 1
    r.bind_stroke_widths(None)  # unbound again: what a renderer that never bound launches and configures
    st = r.render_resident(p)
    assert st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)
    assert r.download("stroke_widths", np.float32).size == 0


def test_reruns_split_ranges_and_enqueued_frames(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=9))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.render_resident(p)
    rows = rand_widths(n, 10, 4.0, 14.0)  # wider: more join and cap lines
    ref.upload(patched(packed, rows))
    want, ref_st = frame(ref)
    t = on_device(rows)
    r.bind_stroke_widths(t)
    st = r.render_resident(p)
    assert st.lines == ref_st.lines and (r.download_target(p) == want).all()
    # a blocking frame re-run after an arena overflow reads the rows again
    r.limit_arena("lines", int(st.lines) - 1)
    try:
        st = r.render_resident(p)
        assert st.retries >= 1
        assert (r.download_target(p) == want).all()
    finally:
        r.limit_arena("lines", 0xFFFFFFFF)
    # ranges that contain flatten read them again
    for a, b in [("pathtag", "flatten"), ("flatten", "flatten")]:
        if a == "flatten":
            r.run_stages(p, "pathtag", "pathtag")
        r.run_stages(p, a, b)
        out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        r.run_stages(p, "draw", "fine", out.data_ptr())
        assert (out.cpu().numpy() == want).all(), (a, b)
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.enqueue(p, out.data_ptr())
    r.finish()
    assert (out.cpu().numpy() == want).all()


# ---- 3. with other features ------------------------------------------------------------------------------------------------
def test_view_culling_and_constant_screen_width(rr):
    r, ref = rr
    # a thin stroke just above the frame: only its bound width reaches into it
    s = Scene()
    s.stroke(Stroke(0.5), Affine.IDENTITY, Color(0.9, 0.1, 0.1, 1.0), None, Line(40, -12, 300, -12))
    s.stroke(Stroke(1.0), Affine.IDENTITY, Color(0.1, 0.1, 0.9, 1.0), None, Circle(150, 120, 60))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.8, 0.2, 1.0), None, Rect(250, 40, 330, 90))
    packed = resolve(s.encoding)
    r.upload(packed)
    view = Affine.translate(0, 0) * Affine.scale(1.0)
    r.set_view(view)
    try:
        rows = np.array([30.0, 2.0, 9.0], dtype=np.float32)
        r.bind_stroke_widths(on_device(rows))
        img, _ = frame(r)
        ref.upload(patched(packed, rows))
        ref.set_view(view)
        want, _ = frame(ref)
        ref.set_view(None)
        assert (img == want).all()
        assert (img[:4, 60:280] != img[300:304, 60:280]).any(), "the widened stroke above the frame is missing"
        # constant on-screen width across zooms: rows w / z under a uniform zoom z equal the re-encoded scene under the view
        for z in (0.5, 2.0, 3.7):
            v = Affine.translate(-20 * z, -10 * z) * Affine.scale(z)
            r.set_view(v)
            rows = np.array([3.0 / z, 4.0 / z, 1.0], dtype=np.float32)
            r.bind_stroke_widths(on_device(rows))
            img, _ = frame(r)
            ref.upload(patched(packed, rows))
            ref.set_view(v)
            assert (img == frame(ref)[0]).all(), z
            ref.set_view(None)
    finally:
        r.set_view(None)
        ref.set_view(None)
    # the general view case on the mixed scene
    s, _ = build(width_ops(seed=11))
    packed = resolve(s.encoding)
    rows = rand_widths(s.n_draw_objects, 12)
    v = Affine.translate(-60, -30) * Affine.scale(1.8)
    r.upload(packed)
    r.set_view(v)
    ref.upload(patched(packed, rows))
    ref.set_view(v)
    try:
        r.bind_stroke_widths(on_device(rows))
        assert (frame(r)[0] == frame(ref)[0]).all()
    finally:
        r.set_view(None)
        ref.set_view(None)


def test_with_transforms_points_visibility_and_all_bindings(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=13))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    rows = rand_widths(n, 14)
    # bound transforms and points moved, with widths: the host route patches all three
    tr = transforms(packed)
    tr[:, 4:] += np.float32(7.0)
    pts = points(packed) + np.float32(1.5)
    r.bind_transforms(on_device(tr))
    r.bind_path_points(on_device(pts))
    r.bind_stroke_widths(on_device(rows))
    host = patched(packed, rows)
    L = packed.layout
    sc = np.array(host.scene, dtype=np.uint32)
    sc[L.transform_base:L.style_base] = tr.reshape(-1).view(np.uint32)
    sc[L.path_data_base:L.path_data_base + pts.size] = pts.reshape(-1).view(np.uint32)
    ref.upload(Packed(sc, L, host.ramps, host.atlas))
    want, _ = frame(ref)
    assert (frame(r)[0] == want).all()
    # a hidden stroke stays hidden, and all seven bindings at once (colours NaN: encoded; stops and instances: see compose)
    is_stroke, _ = strokes(packed)
    hidden = set(np.nonzero(is_stroke)[0][::3].tolist())
    r.bind_draw_visibility(on_device(flags_of(n, hidden)))
    r.bind_draw_colors(on_device(np.full((n, 4), np.nan, dtype=np.float32)))
    img, _ = frame(r)
    sub = patched(packed, rows)
    sc = np.array(sub.scene, dtype=np.uint32)
    sc[L.transform_base:L.style_base] = tr.reshape(-1).view(np.uint32)
    sc[L.path_data_base:L.path_data_base + pts.size] = pts.reshape(-1).view(np.uint32)
    ref.upload(Packed(sc, L, sub.ramps, sub.atlas))
    vis = np.ones(n, dtype=np.uint8)
    vis[list(hidden)] = 0
    ref.bind_draw_visibility(on_device(vis))
    assert (img == frame(ref)[0]).all()
    ref.bind_draw_visibility(None)
    for b in ("bind_draw_visibility", "bind_draw_colors", "bind_path_points", "bind_transforms", "bind_stroke_widths"):
        getattr(r, b)(None)


def test_composed_instances_batches_and_seven_bindings(rr):
    r, ref = rr
    frag_ops = [width_ops(seed=20 + k, dx=0.0, n=8) for k in range(2)]
    frags = [build(o)[0] for o in frag_ops]
    inst = [0, 1, 0]
    ids = [r.upload_fragment(f) for f in frags]
    _, offs = r.compose([(ids[i], None) for i in inst])
    n = int(offs[-1])
    xf = rand_rows(len(inst), 21, 40, 30) * np.float32([0.6, 0.6, 0.6, 0.6, 1, 1])
    rows = rand_widths(n, 22)
    r.bind_instance_transforms(on_device(xf.astype(np.float32)))
    r.bind_stroke_widths(on_device(rows))
    # the host route: each instance re-encoded with its global rows as its strokes' widths (every stroke has its own entry)
    host = Scene()
    for k, i in enumerate(inst):
        base = int(offs[k])
        sc = build(frag_ops[i])[0]
        is_stroke, entry = strokes(resolve(sc.encoding))
        for j in np.nonzero(is_stroke)[0]:
            fl, _ = sc.encoding.styles[entry[j]]
            sc.encoding.styles[entry[j]] = (fl, float(rows[base + j]))
        host.append(sc, aff(xf[k]))
    ref.upload(resolve(host.encoding))
    img, _ = frame(r)
    same(img, frame(ref)[0], AA_MSAA16)
    # all seven bindings at once: colours, points, stops, transforms and visibility at their encoded values
    r.bind_gradient_stops(on_device(np.full((1, 5), np.nan, dtype=np.float32)))
    r.bind_draw_colors(on_device(np.full((n, 4), np.nan, dtype=np.float32)))
    r.bind_draw_visibility(on_device(np.ones(n, dtype=np.uint8)))
    r.bind_transforms(on_device(np.full((1, 6), np.nan, dtype=np.float32)))
    r.bind_path_points(on_device(np.full((1, 2), np.nan, dtype=np.float32)))
    assert (frame(r)[0] == img).all()
    for b in ("bind_gradient_stops", "bind_draw_visibility", "bind_draw_colors", "bind_path_points", "bind_transforms", "bind_stroke_widths", "bind_instance_transforms"):
        getattr(r, b)(None)
    for f in ids:
        r.free_fragment(f)
    # a batch: rows are global, in cell order
    cells = [width_ops(seed=30 + k, n=8) for k in range(3)]
    whole, cell_offs = Scene(), [0]
    for c in cells:
        build(c, s=whole)
        cell_offs.append(whole.n_draw_objects)
    packed = resolve(whole.encoding)
    rows = rand_widths(whole.n_draw_objects, 31)
    r.upload(packed)
    r.bind_stroke_widths(on_device(rows))
    r.set_cells(cell_offs)
    ref.upload(patched(packed, rows))
    ref.set_cells(cell_offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


def test_hit_tests_follow_the_widened_outline(rr):
    r, _ = rr
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.2, 0.2, 1.0), None, Rect(0, 0, 200, 200))
    s.stroke(Stroke(2.0), Affine.IDENTITY, Color(0.9, 0.1, 0.1, 1.0), None, Line(20, 100, 180, 100))
    r.upload(resolve(s.encoding))
    probe = np.array([[100, 100], [100, 106], [100, 113]], dtype=np.float32)
    frame(r, AA_AREA, 200, 200)
    assert r.hit_test(probe).tolist() == [1, 0, 0]
    r.bind_stroke_widths(on_device(np.array([np.nan, 20.0], dtype=np.float32)))
    frame(r, AA_AREA, 200, 200)
    assert r.hit_test(probe).tolist() == [1, 1, 0]
    m = r.hit_map()
    assert (m[91:109, 30:170] == 1).all() and (m[115:, :] == 0).all()
    r.bind_stroke_widths(None)


# ---- 4. damage tracking ----------------------------------------------------------------------------------------------------
def test_damage_is_the_boxes_of_changed_widths(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=50))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    is_stroke, _ = strokes(packed)
    rows = np.full(n, np.nan, dtype=np.float32)
    t = on_device(rows)
    r.bind_stroke_widths(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)

    def step(new):
        t.copy_(torch.from_numpy(new))
        torch.cuda.synchronize()
        before = r.download("draw_bboxes", np.float32).reshape(-1, 4)
        r.render_resident(p, dst.data_ptr())
        ref.upload(patched(packed, new))
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        return r.last_damage(), before, r.download("draw_bboxes", np.float32).reshape(-1, 4)

    try:
        assert step(rows)[0].sum() == n_tiles
        assert step(rows)[0].sum() == 0
        ks = np.nonzero(is_stroke)[0]
        cur = rows.copy()
        for ch in ([ks[0]], [ks[3], ks[7]], [ks[5]]):
            new = cur.copy()
            new[ch] = np.float32(11.0)
            got, before, after = step(new)
            want = box_tiles(before[ch], W, H) | box_tiles(after[ch], W, H)
            assert want.any() and (got == want).all(), ch
            cur = new
        # back to the encoded width: a change; a fill's row, or a fallback to an unchanged encoded width: none
        new = cur.copy()
        new[ks[5]] = np.nan
        got, before, after = step(new)
        assert (got == box_tiles(before[[ks[5]]], W, H) | box_tiles(after[[ks[5]]], W, H)).all()
        cur = new
        fills = np.nonzero(~is_stroke)[0]
        new = cur.copy()
        new[fills] = np.float32(40.0)
        assert step(new)[0].sum() == 0
        cur = new
        _, entry = strokes(packed)
        enc_w = np.asarray(packed.scene, dtype=np.uint32)[packed.layout.style_base + 2 * entry[ks[1]] + 1].view(np.float32)
        new = cur.copy()
        new[ks[1]] = enc_w  # the encoded width itself
        assert step(new)[0].sum() == 0
        new[ks[1]] = -1.0  # falls back to the same encoded width
        assert step(new)[0].sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_stroke_widths(None)


def test_upload_diff_and_recompose_after_a_bound_base_are_full(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=51))
    packed = resolve(s.encoding)
    n = s.n_draw_objects
    r.upload(packed)
    r.bind_stroke_widths(on_device(rand_widths(n, 52)))
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        r.render_resident(p, dst.data_ptr())
        r.set_upload_diff(True)
        r.upload(packed)  # diffed against a base with bound widths: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        ref.upload(packed)
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload(packed)  # an unbound base: nothing
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == 0
        r.set_upload_diff(False)
        fid = r.upload_fragment(s)
        r.compose([(fid, None)])
        r.render_resident(p, dst.data_ptr())
        r.bind_stroke_widths(on_device(rand_widths(n, 53)))
        r.render_resident(p, dst.data_ptr())
        r.recompose([(fid, None)])  # a bound base: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        r.free_fragment(fid)
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 5. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_stroke_widths(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding_and_installations_unbind(rr):
    r, ref = rr
    s, _ = build(width_ops(seed=60))
    n = s.n_draw_objects
    packed = resolve(s.encoding)
    r.upload(packed)
    rows = rand_widths(n, 61)
    t = on_device(rows)
    r.bind_stroke_widths(t)
    before, _ = frame(r)
    ref.upload(patched(packed, rows))
    assert (before == frame(ref)[0]).all()

    def refused(x, args, word):
        assert _bind_raw(x, *args) == VB_E_INVALID, args
        msg = x.lib.vb_last_error(x.handle)
        assert msg.startswith(b"vb_bind_stroke_widths: ") and word in msg, (args, msg)

    ptr = t.data_ptr()
    host = np.zeros(n, dtype=np.float32)
    for args, word in (((ptr, 0, 4), b"rows"), ((ptr, n + 1, 4), b"rows"), ((host.ctypes.data, n, 4), b"device"), ((ptr + 2, n - 1, 4), b"aligned"),
                       ((ptr, n, 0), b"pitch"), ((ptr, n, 2), b"pitch"), ((ptr, n, 6), b"pitch"), ((ptr, n, 1 << 32), b"pitch")):
        refused(r, args, word)
        assert (frame(r)[0] == before).all(), args
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    refused(r, (ptr, n, 4), b"enqueued")
    r.finish()
    assert (r.download_target(p) == before).all()
    x = Renderer()
    try:
        refused(x, (ptr, 1, 4), b"scene")
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        refused(x, (ptr, n, 4), b"exchange")
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        refused(g.renderer(0), (ptr, 1, 4), b"vb_group")
    finally:
        g.close()
    assert (frame(r)[0] == before).all()
    # every installation unbinds; None unbinds
    ref.upload(packed)
    encoded, _ = frame(ref)
    fid = r.upload_fragment(s)
    installs = [lambda: r.upload(packed), lambda: r.upload_scene(s), lambda: r.render_to_texture(packed, p),
                lambda: list(r.render_stream([packed], p)), lambda: r.recompose([(fid, None)]), lambda: r.compose([(fid, None)])]
    for install in installs:
        r.compose([(fid, None)])
        r.bind_stroke_widths(t)
        assert (frame(r)[0] == before).all()
        install()
        assert (frame(r)[0] == encoded).all()
    r.free_fragment(fid)
    r.upload(packed)
    r.bind_stroke_widths(t)
    r.bind_stroke_widths(None)
    assert (frame(r)[0] == encoded).all()
