"""Bound gradient stops (Renderer.bind_gradient_stops, vb_bind_gradient_stops): every frame renders the installed scene with
stop k of its ramp patches replaced by row k of a device array, read when the frame runs. `r` binds; `ref` takes the host
route, the same streams with the rows' stops substituted, installed with vb_scene_upload_streams, and every frame of `r` must
equal it. Run on an H100 with `pytest -m gpu`."""
import copy
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT, FILL_NON_ZERO, MIX_MULTIPLY, Color,
                                 Gradient, Image, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Circle, Rect

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels
from .test_gradient_stops import ramp_np

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
IMG = np.random.default_rng(21).integers(0, 256, (18, 22, 4), dtype=np.uint8)
SHARED = [(0.0, Color(0.9, 0.2, 0.1, 1.0)), (0.5, Color(0.2, 0.8, 0.3, 0.6)), (1.0, Color(0.1, 0.2, 0.9, 1.0))]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def stops_of(g, n):
    """n seeded stops, exactly representable in float32, in order."""
    o = np.sort(g.uniform(0, 1, n)).astype(np.float32)
    c = g.uniform(0, 1, (n, 4)).astype(np.float32)
    c[:, 3] = g.choice(np.float32([1.0, 0.7, 0.25, 0.0]), n)
    return [(float(o[i]), Color(*map(float, c[i]))) for i in range(n)]


def grads(seed=0, dx=0.0):
    """Linear, radial and sweep gradients in both alpha spaces and every extend mode; two gradients with equal stops (one
    de-duplicated ramp); gradients inside a clip and a blend layer; and a solid fill, an image and a blurred rectangle."""
    g = np.random.default_rng(seed)
    s = Scene()
    k = 0
    for kind in ("linear", "radial", "sweep"):
        for ext in (EXTEND_PAD, EXTEND_REPEAT, EXTEND_REFLECT):
            premul = bool(k % 2)
            x, y = dx + 10 + 62 * (k % 6), 10 + 60 * (k // 6)
            st = stops_of(g, 2 + k % 3)
            if kind == "linear":
                br = Gradient.linear((x + 10, y), (x + 40, y + 20), st, ext, premul)
            elif kind == "radial":
                br = Gradient.radial((x + 20, y + 20), 3.0, (x + 28, y + 25), 22.0, st, ext, premul)
            else:
                br = Gradient.sweep((x + 28, y + 25), 0.3, 4.0, st, ext, premul)
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, br, None, Rect(x, y, x + 56, y + 52))
            k += 1
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (60, 0), SHARED), None, Rect(dx + 10, 130, dx + 90, 170))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.3, 0.6, 0.2, 0.8), None, Circle(dx + 150, 150, 25))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (60, 0), SHARED), None, Rect(dx + 200, 130, dx + 280, 170))
    s.draw_image(Image(IMG), Affine.translate(dx + 300, 130) * Affine.scale(2.0))
    s.draw_blurred_rounded_rect(Affine.translate(dx + 20, 190), Rect(0, 0, 60, 30), Color(0.8, 0.5, 0.1, 1.0), 6.0, 4.0)
    s.push_clip_layer(FILL_NON_ZERO, Affine.rotate(0.1), Circle(dx + 180, 240, 60))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.radial((dx + 180, 240), 5.0, (dx + 180, 240), 70.0, stops_of(g, 3)), None,
           Rect(dx + 110, 180, dx + 250, 300))
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Rect(dx + 150, 200, dx + 300, 310))
    s.stroke(Stroke(6.0), Affine.IDENTITY, Gradient.linear((dx + 150, 0), (dx + 300, 0), stops_of(g, 4), premul_interp=False), None,
             Circle(dx + 220, 255, 40))
    s.pop_layer()
    s.pop_layer()
    return s


def rows_of(scene):
    """The scene's stops as float32 (n, 5) rows."""
    return np.array([(o, c.r, c.g, c.b, c.a) for p in scene.encoding.ramp_patches for o, c in p["stops"]], dtype=np.float32)


def rand_stops(scene, seed):
    """The scene's rows with colours and offsets moved: offsets out of order and outside [0, 1] included."""
    rows = rows_of(scene)
    g = np.random.default_rng(seed)
    rows[:, 1:] = g.uniform(0, 1, (len(rows), 4)).astype(np.float32)
    rows[:, 4] = g.choice(np.float32([1.0, 0.6, 0.1, 0.0]), len(rows))
    rows[:, 0] = np.float32(g.uniform(-0.2, 1.2, len(rows)))
    return rows


def substituted(scene, rows, n=None):
    """The host route's scene: stop k of the patches replaced by row k, for k < n whose row is finite."""
    n = len(rows) if n is None else n
    s = copy.deepcopy(scene)
    k = 0
    for p in s.encoding.ramp_patches:
        st = []
        for o, c in p["stops"]:
            if k < n and np.isfinite(rows[k]).all():
                o, c = float(rows[k, 0]), Color(*map(float, rows[k, 1:]))
            st.append((o, c))
            k += 1
        p["stops"] = st
    return s


def on_device(rows):
    t = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).cuda()
    torch.cuda.synchronize()
    return t


def frame(r, aa=AA_MSAA16, w=W, h=H):
    p = RenderParams(BASE, w, h, aa)
    st = r.render_resident(p)
    return r.download_target(p), st


def same(img, want, aa):
    if aa == AA_AREA:
        assert_pixels(img, want, aa)
    else:
        assert (img == want).all()


def check_rows(r, ref, scene, host_scene):
    """Each gradient's ramp row of r's last frame equals the host route's for that gradient and make_ramp of its stops; the
    draw data differs only in ramp ids, and the draw boxes are equal."""
    rd, fd = r.download("draw_data", np.uint32), ref.download("draw_data", np.uint32)
    rr_, fr = r.download("ramps", np.uint32).reshape(-1, 512), ref.download("ramps", np.uint32).reshape(-1, 512)
    ramp_words = [p["draw_data_offset"] for p in scene.encoding.ramp_patches]
    keep = np.ones(len(rd), dtype=bool)
    keep[ramp_words] = False
    assert np.array_equal(rd[keep], fd[keep])
    for p, w in zip(host_scene.encoding.ramp_patches, ramp_words):
        assert rd[w] & 3 == fd[w] & 3
        row = rr_[rd[w] >> 2]
        assert np.array_equal(row, fr[fd[w] >> 2])
        st = np.array([(o, c.r, c.g, c.b, c.a) for o, c in p["stops"]], dtype=np.float32)
        assert np.array_equal(row, ramp_np(st, p["premul"]))
    assert np.array_equal(r.download("draw_bboxes", np.float32), ref.download("draw_bboxes", np.float32))


# ---- 1. equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_bound_equals_the_host_route(rr, aa):
    r, ref = rr
    s = grads()
    r.upload_scene(s)
    n0 = resolve(s.encoding).ramps.shape[0]
    rows = rand_stops(s, 1)
    r.bind_gradient_stops(on_device(rows))
    host = substituted(s, rows)
    ref.upload_scene(host)
    img, _ = frame(r, aa)
    want, _ = frame(ref, aa)
    same(img, want, aa)
    check_rows(r, ref, s, host)
    # the scene's ramps, then one row per gradient: the two gradients that shared a ramp have rows of their own
    n_patches = len(s.encoding.ramp_patches)
    assert r.download("ramps", np.uint32).size // 512 == n0 + n_patches


def test_partial_strided_and_non_finite_rows(rr):
    r, ref = rr
    s = grads(3)
    base = rows_of(s)
    n_all = len(base)
    state = torch.zeros((n_all, 9), dtype=torch.float32, device="cuda")
    r.upload_scene(s)
    rows = rand_stops(s, 4)
    # a stop of each column non-finite
    for col, v in zip(range(5), (np.nan, np.inf, -np.inf, np.nan, np.inf)):
        rows[2 + 3 * col, col] = v
    state[:, 2:7] = torch.from_numpy(rows)
    torch.cuda.synchronize()
    first = [0]
    for p in s.encoding.ramp_patches:
        first.append(first[-1] + len(p["stops"]))
    straddle = next(f + 1 for f, e in zip(first, first[1:]) if e - f >= 3)  # n inside a gradient's stops
    for n in (n_all, straddle, 1, n_all - 1):
        r.bind_gradient_stops(state[:n, 2:7])
        host = substituted(s, rows, n)
        ref.upload_scene(host)
        img, _ = frame(r)
        want, _ = frame(ref)
        assert (img == want).all(), n
        check_rows(r, ref, s, host)


# ---- 2. updates without calls ----------------------------------------------------------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    s = grads(5)
    r.upload_scene(s)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [rand_stops(s, 200 + j) for j in range(8)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(seq[0].shape, dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_gradient_stops(t)
    caps = None
    for j in range(8):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        # the draw-data region (k_draw_data) and the rows (k_bound_ramps)
        assert st.kernel_launches == unbound + 2
        ref.upload_scene(substituted(s, seq[j]))
        assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    # with colours bound as well, the stops add k_bound_ramps alone
    cols = on_device(np.tile(np.float32([0.2, 0.4, 0.6, 1.0]), (s.n_draw_objects, 1)))
    r.bind_draw_colors(cols)
    both = r.render_resident(p).kernel_launches
    r.bind_gradient_stops(None)
    assert r.render_resident(p).kernel_launches == both - 1 == unbound + 1
    r.bind_draw_colors(None)
    # unbound again: the launches, config and graph of a renderer that never bound
    ref.upload_scene(s)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)
    caps = r.debug_graph_captures()
    r.render_resident(p)
    assert r.debug_graph_captures() == caps


# ---- 3. with other features ------------------------------------------------------------------------------------------------
def test_view_run_stages_and_rerun(rr):
    r, ref = rr
    s = grads(6)
    rows = rand_stops(s, 7)
    r.upload_scene(s)
    r.bind_gradient_stops(on_device(rows))
    ref.upload_scene(substituted(s, rows))
    view = Affine.translate(-30, 20) * Affine.scale(1.3) * Affine.rotate(0.08)
    r.set_view(view)
    ref.set_view(view)
    try:
        assert (frame(r)[0] == frame(ref)[0]).all()
    finally:
        r.set_view(None)
        ref.set_view(None)
    want, _ = frame(ref)
    assert (frame(r)[0] == want).all(), "the binding survives the view"
    # split vb_run_stages ranges: a range from DRAW writes the rows again, from the rows as they are then
    p = RenderParams(BASE, W, H, AA_MSAA16)
    t = on_device(rand_stops(s, 77))
    r.bind_gradient_stops(t)
    r.run_stages(p, "pathtag", "flatten")
    t.copy_(torch.from_numpy(rows))
    torch.cuda.synchronize()
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    out.zero_()
    r.run_stages(p, "pathtag", "binning")
    r.run_stages(p, "tile_alloc", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    # a blocking frame re-run after an arena overflow reads the same rows
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    st = r.render_resident(p)
    assert st.retries == 1
    assert (r.download_target(p) == want).all()


def test_with_colours_and_points(rr):
    r, ref = rr
    s = grads(8)
    r.upload_scene(s)
    stops = rand_stops(s, 9)
    cols = np.random.default_rng(10).uniform(0, 1, (s.n_draw_objects, 4)).astype(np.float32)
    xy = np.array(s.encoding.path_data, dtype=np.float32).reshape(-1, 2)
    xy += np.random.default_rng(11).uniform(-3, 3, xy.shape).astype(np.float32)
    r.bind_draw_colors(on_device(cols))
    r.bind_gradient_stops(on_device(stops))
    r.bind_path_points(on_device(xy))
    host = substituted(s, stops)
    e = host.encoding
    for k, tag in enumerate(e.draw_tags):  # the colours, as re-encoding them would write
        if tag in (0x44, 0x2D4):
            off = sum((t >> 2) & 7 for t in e.draw_tags[:k])
            e.draw_data[off] = Color(*map(float, cols[k])).premul_rgba8_u32()
    e.path_data[:] = [float(v) for v in xy.reshape(-1)]
    ref.upload_scene(host)
    assert (frame(r)[0] == frame(ref)[0]).all()
    check_rows(r, ref, s, host)
    r.bind_draw_colors(None)  # stops and points stay bound
    e.draw_data[:] = list(substituted(s, stops).encoding.draw_data)
    ref.upload_scene(host)
    assert (frame(r)[0] == frame(ref)[0]).all()
    r.bind_path_points(None)
    r.bind_gradient_stops(None)


def test_composed_with_transforms_and_recompose(rr):
    r, ref = rr
    frags = [grads(k) for k in range(2)]
    inst = [0, 1, 0]
    ids = [r.upload_fragment(f) for f in frags]
    lay, offs = r.compose([(ids[i], None) for i in inst])
    whole = Scene()
    for i in inst:
        whole.append(frags[i])
    stops = rand_stops(whole, 12)
    xf = rand_rows(len(inst), 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    r.bind_instance_transforms(on_device(xf))
    r.bind_gradient_stops(on_device(stops))
    host, k0 = Scene(), 0
    for k, i in enumerate(inst):
        m = len(rows_of(frags[i]))
        host.append(substituted(frags[i], stops[k0:k0 + m]), aff(xf[k]))
        k0 += m
    ref.upload_scene(host)
    assert (frame(r)[0] == frame(ref)[0]).all()
    r.recompose([(ids[i], None) for i in inst])  # unbinds
    ref.upload_scene(whole)
    assert (frame(r)[0] == frame(ref)[0]).all()
    r.bind_gradient_stops(on_device(stops))  # a recomposed scene binds as well
    ref.upload_scene(substituted(whole, stops))
    assert (frame(r)[0] == frame(ref)[0]).all()
    for f in ids:
        r.free_fragment(f)


def test_batch_global_indices(rr):
    r, ref = rr
    cells = [grads(k) for k in range(3)]
    whole, offs = Scene(), [0]
    for c in cells:
        whole.append(c)
        offs.append(whole.n_draw_objects)
    stops = rand_stops(whole, 13)
    r.upload_scene(whole)
    r.bind_gradient_stops(on_device(stops))
    r.set_cells(offs)  # the binding survives it
    ref.upload_scene(substituted(whole, stops))
    ref.set_cells(offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


def test_hit_tests_and_maps_do_not_change(rr):
    r, ref = rr
    s = grads(14)
    r.upload_scene(s)
    ref.upload_scene(s)
    rows = rand_stops(s, 15)
    rows[:, 4] = 0.0  # even fully transparent
    r.bind_gradient_stops(on_device(rows))
    frame(r, AA_AREA)
    frame(ref, AA_AREA)
    pts = np.random.default_rng(16).uniform(0, [W, H], (5000, 2)).astype(np.float32)
    got = r.hit_test(pts)
    assert (got >= 0).sum() > 500 and (got == ref.hit_test(pts)).all()
    assert (r.hit_map() == ref.hit_map()).all()


# ---- 4. damage tracking ----------------------------------------------------------------------------------------------------
def box_tiles(boxes, w=W, h=H):
    wt, ht = (w + 15) // 16, (h + 15) // 16
    m = np.zeros((ht, wt), dtype=bool)
    s = np.float32(1 / 16)
    for x0, y0, x1, y1 in boxes:
        if not (x0 < x1 and y0 < y1):
            continue
        tx0, tx1 = int(np.clip(np.floor(np.float32(x0) * s), 0, wt)), int(np.clip(np.ceil(np.float32(x1) * s), 0, wt))
        ty0, ty1 = int(np.clip(np.floor(np.float32(y0) * s), 0, ht)), int(np.clip(np.ceil(np.float32(y1) * s), 0, ht))
        m[ty0:ty1, tx0:tx1] = True
    return m


def test_damage_follows_changed_ramps(rr):
    r, ref = rr
    s = grads(17)
    r.upload_scene(s)
    rows = rand_stops(s, 18)
    t = on_device(rows)
    r.bind_gradient_stops(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    # the draw object of each patch, and each patch's first stop
    tags = s.encoding.draw_tags
    offs, o = [], 0
    for tag in tags:
        offs.append(o)
        o += (tag >> 2) & 7
    patch_draw = [offs.index(pt["draw_data_offset"]) for pt in s.encoding.ramp_patches]
    first = np.cumsum([0] + [len(pt["stops"]) for pt in s.encoding.ramp_patches])
    r.set_damage_tracking(True)

    def step(new=None):
        nonlocal rows
        if new is not None:
            rows = new.astype(np.float32)
            t.copy_(torch.from_numpy(rows))
            torch.cuda.synchronize()
        r.render_resident(p, dst.data_ptr())
        ref.upload_scene(substituted(s, rows))
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        return r.last_damage()

    try:
        assert step().sum() == n_tiles
        boxes = r.download("draw_bboxes", np.float32).reshape(-1, 4)
        for changed in ([0], [3, 7], [len(patch_draw) - 1, len(patch_draw) - 3]):
            new = rows.copy()
            for g in changed:
                new[first[g], 1:4] = 1.0 - new[first[g], 1:4]
                new[first[g], 4] = 1.0
            got = step(new)
            assert got.any() and (got == box_tiles(boxes[[patch_draw[g] for g in changed]])).all(), changed
        assert step().sum() == 0
        # rows rewritten to values that make the same texels: no damage (an opaque stop's colour one ulp up, which both
        # ramps confirm convert alike; and a non-finite value, which falls back to an unchanged encoded stop)
        g = 0
        opaque = rows.copy()
        opaque[first[g]:first[g + 1], 4] = 1.0
        step(opaque)
        same_rows = opaque.copy()
        same_rows[first[g]:first[g + 1], 1:4] = np.nextafter(rows[first[g]:first[g + 1], 1:4], np.float32(2))
        pt = s.encoding.ramp_patches[g]
        assert np.array_equal(ramp_np(rows[first[g]:first[g + 1]], pt["premul"]), ramp_np(same_rows[first[g]:first[g + 1]], pt["premul"]))
        assert step(same_rows).sum() == 0
        nf = same_rows.copy()
        nf[first[1], 2] = np.nan
        step(nf)
        nf2 = nf.copy()
        nf2[first[1], 3] = np.inf
        assert step(nf2).sum() == 0
        # bind, unbind and rebind each make the next frame full
        for bind in (on_device(rows), None, t):
            r.bind_gradient_stops(bind)
            if bind is None:
                rows = np.full_like(rows, np.nan)  # the host route of an unbound frame: every stop as encoded
            r.render_resident(p, dst.data_ptr())
            assert r.last_damage().sum() == n_tiles
            r.render_resident(p, dst.data_ptr())
            assert r.last_damage().sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_gradient_stops(None)


def test_diffs_after_a_bound_base_are_full(rr):
    r, ref = rr
    s = grads(19)
    r.upload_scene(s)
    t = on_device(rand_stops(s, 20))
    r.bind_gradient_stops(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        r.set_upload_diff(True)
        r.upload_scene(s)  # diffed against a bound base: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        ref.upload_scene(s)
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload_scene(s)  # unbound base: the same upload damages nothing
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == 0
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 5. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_gradient_stops(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding(rr):
    r, ref = rr
    s = grads(22)
    r.upload_scene(s)
    rows = rand_stops(s, 23)
    n = len(rows)
    t = on_device(rows)
    r.bind_gradient_stops(t)
    before, _ = frame(r)

    def unchanged(what):
        assert r.lib.vb_last_error(r.handle), what
        assert (frame(r)[0] == before).all(), what

    ptr = t.data_ptr()
    host = np.zeros((n, 5), dtype=np.float32)
    for args in ((ptr, 0, 20), (ptr, n + 1, 20), (host.ctypes.data, n, 20), (ptr + 2, n, 20), (ptr, n, 16), (ptr, n, 22),
                 (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        unchanged(args)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    assert _bind_raw(r, ptr, n, 20) == VB_E_INVALID  # between enqueue and finish
    r.finish()
    assert (r.download_target(p) == before).all()
    # no scene, a packed scene, a renderer of a vb_group, one with the exchange configured
    packed = resolve(s.encoding)
    x = Renderer()
    try:
        assert _bind_raw(x, ptr, 1, 20) == VB_E_INVALID and b"scene" in x.lib.vb_last_error(x.handle)
        x.upload(packed)
        assert _bind_raw(x, ptr, 1, 20) == VB_E_INVALID and b"packed" in x.lib.vb_last_error(x.handle)
        x.render_to_texture(packed, p)
        assert _bind_raw(x, ptr, 1, 20) == VB_E_INVALID
        x.upload_scene(s)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        assert _bind_raw(x, ptr, n, 20) == VB_E_INVALID and b"exchange" in x.lib.vb_last_error(x.handle)
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        assert _bind_raw(g.renderer(0), ptr, 1, 20) == VB_E_INVALID
    finally:
        g.close()
    # every installation unbinds; None unbinds
    ref.upload_scene(s)
    encoded, _ = frame(ref)
    fid = r.upload_fragment(s)
    for install in (lambda: r.upload(packed), lambda: r.upload_scene(s), lambda: r.render_to_texture(packed, p),
                    lambda: r.compose([(fid, None)]), lambda: r.recompose([(fid, None)])):
        r.compose([(fid, None)])
        r.bind_gradient_stops(t)
        assert not (frame(r)[0] == encoded).all()
        install()
        assert (frame(r)[0] == encoded).all()
    r.free_fragment(fid)
    r.upload_scene(s)
    r.bind_gradient_stops(t)
    r.bind_gradient_stops(None)
    assert (frame(r)[0] == encoded).all()
