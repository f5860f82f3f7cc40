"""Views of a resident scene (Renderer.set_view, vb_set_view): the scene is uploaded once and rendered under a view as
`Scene().append(scene, view)` renders. The reference of every case is that appended scene resolved and uploaded from the
host (`encoding.viewed` is the same bytes, tests/test_view.py); against the oracle where the frame fits it, and against the
host-mapped render where flatten culls to the frame. Run on an H100 with `pytest -m gpu`."""
import math

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, Color, FILL_EVEN_ODD, FILL_NON_ZERO, Image, MIX_CLIP, STYLE_CAP_ROUND, STYLE_JOIN_MITER,
                                 Scene, Stroke, resolve, viewed)
from vello_b200.shapes import Affine, BezPath, Rect

from . import parity
from .test_gpu_parity import assert_pixels

pytestmark = pytest.mark.gpu

BASE = Color.from_rgba8(12, 20, 30)


@pytest.fixture(scope="module")
def renderers():
    """`r` renders under views; `ref` renders the host-mapped references and never has a view."""
    from vello_b200.renderer import Renderer
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def appended(scene, view):
    out = Scene()
    out.append(scene, view)
    return out


def render(r, p, bin_rows=(0, 0), tile_rows=(0, 0)):
    st = r.render_resident(p, 0, bin_rows, tile_rows)
    return r.download_target(p, bin_rows, 0, tile_rows), st


def view_frame(r, packed, view, p):
    """`packed` uploaded once, rendered under `view`."""
    r.set_view(view)
    r.upload(packed)
    return render(r, p)


def host_frame(ref, packed, view, p):
    """The reference: the appended scene, resolved and uploaded from the host, no view."""
    ref.set_view(None)
    ref.upload(viewed(packed, view))
    return render(ref, p)


# ---- bit-exact transforms: scenes that stay inside the frame, so nothing is culled -------------------------------------
EXACT_SCENES = {
    "tiger": lambda: (scenes.tiger(256, 256), 256, 256),
    "stroke_styles": scenes.stroke_styles,
    "brushes": scenes.brushes,
    "many_clips": scenes.many_clips,
    "deep_blend": scenes.deep_blend,
    "gradient_extend": scenes.gradient_extend,
    "two_point_radial": scenes.two_point_radial,
}
EXACT_VIEWS = {  # about the centre of the scene's lines, in a square frame that holds them under every one of these views
    "identity": Affine(),
    "integer_pan": Affine.translate(9.0, -14.0),
    "fractional_pan": Affine.translate(3.375, -7.8125),
    "rotation": Affine.rotate(0.6),
    "mirror": Affine.scale(-1.0, 1.0),
    "skew": Affine((1.0, 0.0, 0.35, 1.0, 0.0, 0.0)),
    "nonuniform_scale": Affine.scale(1.3, 0.7),
}


def centred(oracle, packed, view):
    """(frame size, `view` about the centre of the scene's lines, placed in the middle of the frame). The lines' extents are
    the oracle's path boxes (strokes included), whatever the scene's nominal size."""
    oracle.render(packed, 16, 16, 0, AA_MSAA16)
    b = oracle.buffer("path_bboxes")
    b = b[(b["x1"] > b["x0"]) | (b["y1"] > b["y0"])]
    x0, y0, x1, y1 = int(b["x0"].min()), int(b["y0"].min()), int(b["x1"].max()), int(b["y1"].max())
    f = (int(1.6 * max(x1 - x0, y1 - y0)) + 64 + 15) // 16 * 16  # a rotation, skew or 1.3x scale stays inside
    return f, Affine.translate(f / 2, f / 2) * view * Affine.translate(-(x0 + x1) / 2, -(y0 + y1) / 2)


@pytest.mark.parametrize("vname", sorted(EXACT_VIEWS))
@pytest.mark.parametrize("sname", sorted(EXACT_SCENES))
def test_view_transforms_bit_exact(renderers, oracle, sname, vname):
    r, _ = renderers
    scene = EXACT_SCENES[sname]()[0]
    packed = resolve(scene.encoding)
    fw, view = centred(oracle, packed, EXACT_VIEWS[vname])
    fh = fw
    want = resolve(appended(scene, view).encoding)
    for aa in (AA_MSAA16, AA_MSAA8, AA_AREA):
        p = RenderParams(BASE, fw, fh, aa)
        img, st = view_frame(r, packed, view, p)
        ref = oracle.render(want, fw, fh, BASE.premul_rgba8_u32(), aa)
        if aa == AA_MSAA16:
            parity.compare_all(r, oracle, want.layout, fw, fh)  # every buffer, bump.lines included: nothing was culled
        if aa == AA_AREA:
            parity.assert_replay(r, oracle, want, img, fw, fh, aa, BASE)
        assert_pixels(img, ref, aa)


# ---- culling keeps pixels ----------------------------------------------------------------------------------------------
def zoom(k, cx, cy, size, rot=0.0):
    """Zoom by k into scene point (cx, cy), which lands in the frame's centre."""
    return Affine.translate(size / 2, size / 2) * Affine.rotate(rot) * Affine.scale(k) * Affine.translate(-cx, -cy)


def cull_views(size):
    s = size
    return {
        "zoom2_centre": zoom(2, s / 2, s / 2, s),
        "zoom4_topleft": zoom(4, s / 8, s / 8, s),
        "zoom16_bottomright": zoom(16, 7 * s / 8, 7 * s / 8, s),
        "zoom64_topright_rot": zoom(64, 7 * s / 8, s / 8, s, 0.4),
        "zoom8_bottomleft": zoom(8, s / 8, 7 * s / 8, s),
        "pan_half_right": Affine.translate(s / 2 + 0.5, 0.0),
        "pan_half_up": Affine.translate(0.25, -s / 2),
        "pan_off_below": Affine.translate(0.0, s + 40.0),
        "pan_off_right": Affine.translate(s + 40.0, 3.0),
    }


CULL_SCENES = {
    "paris_like": lambda: (scenes.paris_like(2500, 1024, seed=41), 1024),
    "tiger": lambda: (scenes.tiger(512, 512), 512),
}


@pytest.mark.parametrize("sname", sorted(CULL_SCENES))
def test_culling_keeps_pixels(renderers, oracle, sname):
    r, ref = renderers
    scene, size = CULL_SCENES[sname]()
    packed = resolve(scene.encoding)
    for vname, view in cull_views(size).items():
        for aa in (AA_MSAA16, AA_MSAA8, AA_AREA):
            p = RenderParams(BASE, size, size, aa)
            img, st = view_frame(r, packed, view, p)
            want, wst = host_frame(ref, packed, view, p)
            assert st.lines < wst.lines, (vname, st.lines, wst.lines)
            if aa == AA_AREA:
                parity.assert_replay(r, oracle, viewed(packed, view), img, size, size, aa, BASE)
                assert_pixels(img, want, aa)
            else:
                assert np.array_equal(img, want), (vname, aa, int((img != want).any(axis=2).sum()))


def crafted(kind, W, H):
    s = Scene()
    red, green, blue = Color.from_rgba8(220, 40, 40), Color.from_rgba8(40, 200, 60, 200), Color.from_rgba8(40, 60, 230, 180)
    if kind == "cover_rect":  # covers the frame, right edge (and top / bottom edges) off-frame
        s.fill(FILL_NON_ZERO, Affine(), red, None, Rect(-20.0, -30.0, W + 500.0, H + 700.0))
        s.fill(FILL_EVEN_ODD, Affine(), green, None, Rect(W / 3, -5.0, W + 9000.0, H / 2))
    elif kind == "clip_outside":  # clip paths entirely right of and below the frame, with draws inside and after them
        for clip in (Rect(W + 30.0, 10.0, W + 300.0, H - 10.0), Rect(10.0, H + 30.0, W - 10.0, H + 400.0)):
            s.push_layer(FILL_NON_ZERO, MIX_CLIP, COMPOSE_SRC_OVER, 1.0, Affine(), clip)
            s.fill(FILL_NON_ZERO, Affine(), red, None, Rect(-50.0, -50.0, W + 500.0, H + 500.0))
            s.pop_layer()
        s.fill(FILL_NON_ZERO, Affine(), blue, None, Rect(20.0, 20.0, W - 20.0, H - 20.0))
    elif kind == "joins_caps":  # miter joins and round caps whose reach just crosses each edge from outside
        lw = 24.0
        miter = Stroke(width=lw, join=STYLE_JOIN_MITER, miter_limit=10.0)
        round_cap = Stroke(width=lw, start_cap=STYLE_CAP_ROUND, end_cap=STYLE_CAP_ROUND)
        d = 6.0  # centre line this far outside the edge: only the join tip / the cap reaches in
        far = [Affine(), Affine.translate(W + 900.0, 0.0), Affine.translate(0.0, H + 900.0), Affine.translate(0.0, -H - 900.0)]
        for path in (BezPath([("M", W + d + 40, 40.0), ("L", W + d, H / 2), ("L", W + d + 40, H - 40.0)]),
                     BezPath([("M", -d - 40, 40.0), ("L", -d, H / 2), ("L", -d - 40, H - 40.0)]),
                     BezPath([("M", 40.0, -d - 40), ("L", W / 2, -d), ("L", W - 40.0, -d - 40)]),
                     BezPath([("M", 40.0, H + d + 40), ("L", W / 2, H + d), ("L", W - 40.0, H + d + 40)])):
            for t in far:  # the copies far outside are culled, the ones whose reach crosses an edge are not
                s.stroke(miter, t, green, None, path)
        for path in (BezPath([("M", W + d, 20.0), ("L", W + d + 300, 20.0)]), BezPath([("M", 30.0, H + d), ("L", 30.0, H + d + 300)]),
                     BezPath([("M", 60.0, -d), ("L", 60.0, -d - 300)]), BezPath([("M", -d, 90.0), ("L", -d - 300, 90.0)])):
            for t in far:
                s.stroke(round_cap, t, blue, None, path)
    return s


@pytest.mark.parametrize("kind", ["cover_rect", "clip_outside", "joins_caps"])
def test_culling_crafted_edges(renderers, oracle, kind):
    r, ref = renderers
    W, H = 320, 240
    packed = resolve(crafted(kind, W, H).encoding)
    for view in (Affine(), Affine.translate(0.5, -0.25), Affine.translate(16.0, 16.0)):
        for aa in (AA_MSAA16, AA_MSAA8, AA_AREA):
            p = RenderParams(BASE, W, H, aa)
            img, st = view_frame(r, packed, view, p)
            want, wst = host_frame(ref, packed, view, p)
            assert st.lines < wst.lines
            if aa == AA_AREA:
                parity.assert_replay(r, oracle, viewed(packed, view), img, W, H, aa, BASE)
                assert_pixels(img, want, aa)
            else:
                assert np.array_equal(img, want), (kind, view.coeffs, aa)


def test_nan_view_product(renderers):
    """A view whose product with a draw's transform overflows to inf - inf: a NaN hull is kept, and the frame is the host's."""
    r, ref = renderers
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.translate(2e38, -2e38), Color.from_rgba8(200, 30, 30), None, Rect(0.0, 0.0, 50.0, 40.0))
    s.fill(FILL_NON_ZERO, Affine.scale(0.25, 0.5), Color.from_rgba8(30, 200, 30), None, Rect(20.0, 20.0, 220.0, 190.0))
    packed = resolve(s.encoding)
    view = Affine((2.0, 2.0, 2.0, 2.0 + 2.0 ** -20, 0.0, 0.0))
    assert np.isnan(viewed(packed, view).scene[packed.layout.transform_base:packed.layout.style_base].view(np.float32)).any()
    for aa in (AA_MSAA16, AA_MSAA8):
        p = RenderParams(BASE, 160, 120, aa)
        img, _ = view_frame(r, packed, view, p)
        want, _ = host_frame(ref, packed, view, p)
        assert np.array_equal(img, want)


def test_non_finite_view_is_rejected(renderers):
    from vello_b200.renderer import VelloB200Error
    r, _ = renderers
    for bad in ((math.nan, 0, 0, 1, 0, 0), (1, 0, 0, 1, math.inf, 0), (1e39, 0, 0, 1, 0, 0)):
        with pytest.raises(VelloB200Error):
            r.set_view(Affine(tuple(float(v) for v in bad)))
    r.set_view(None)


# ---- composition with the other features -------------------------------------------------------------------------------
def test_view_with_tile_row_stripes(renderers):
    r, _ = renderers
    size = 1024
    packed = resolve(scenes.paris_like(1500, size, seed=7).encoding)
    view = zoom(3, 300.0, 700.0, size, 0.2)
    p = RenderParams(BASE, size, size, AA_MSAA16)
    full, _ = view_frame(r, packed, view, p)
    rows = [0, 5, 17, 40, 64]
    parts = [render(r, p, tile_rows=(a, b))[0] for a, b in zip(rows, rows[1:])]
    assert np.array_equal(np.concatenate(parts), full)


def test_view_with_batch(renderers):
    from vello_b200.renderer import Renderer
    r, _ = renderers
    ss = [scenes.random_small(k)[0] for k in range(5)]
    view = Affine.translate(40.5, -12.25) * Affine.rotate(0.3) * Affine.scale(1.6, 1.1)  # culls in every cell
    p = RenderParams(BASE, 200, 150, AA_MSAA16)
    r.set_view(view)
    cells = r.render_batch(ss, p)
    one = Renderer()
    one.set_view(view)
    for k, s in enumerate(ss):
        alone = Scene()  # with its open layers popped: a batch closes them behind each scene, as pop_layer does
        alone.append(s)
        for _ in range(s.encoding.n_open_clips):
            alone.pop_layer()
        one.upload(resolve(alone.encoding))
        assert np.array_equal(cells[k], render(one, p)[0]), k
    one.close()


def test_view_with_group_device_zero_twice(renderers):
    from vello_b200.renderer import RendererGroup
    r, _ = renderers
    size = 1024
    packed = resolve(scenes.paris_like(2000, size, seed=4).encoding)
    view = zoom(4, 600.0, 420.0, size)
    p = RenderParams(BASE, size, size, AA_MSAA16)
    want, _ = view_frame(r, packed, view, p)
    g = RendererGroup([0, 0])
    g.upload(packed)
    g.set_view(view)
    for _ in range(2):
        g.render_resident(p)
        assert np.array_equal(g.frame_to_host(p), want)
    g.close()


def test_view_with_device_resolve_and_override(renderers):
    torch = pytest.importorskip("torch")
    from vello_b200.scene_native import NativeScene
    r, ref = renderers
    rng = np.random.default_rng(5)
    data = rng.integers(0, 256, (21, 26, 4), dtype=np.uint8)
    im = Image(data)

    def draw(s, image):
        s.fill(FILL_NON_ZERO, Affine.translate(20, 30), image, Affine.rotate(0.3) * Affine.scale(2.1), Rect(0, 0, 150, 120))
        s.draw_image(image, Affine.translate(180, 60) * Affine.scale(3.0))

    host = NativeScene()
    draw(host, im)
    view = Affine.translate(-60.0, 25.5) * Affine.scale(1.5)
    p = RenderParams(BASE, 256, 256, AA_MSAA16)
    want, _ = host_frame(ref, host.resolve(), view, p)
    tex = r.register_texture(torch.from_numpy(data).cuda())
    dev = NativeScene()
    draw(dev, tex)
    r.set_view(view)
    dev.upload_device(r)
    assert np.array_equal(render(r, p)[0], want)
    r.unregister_texture(tex)
    r.set_view(None)


# ---- graphs and stream order --------------------------------------------------------------------------------------------
def test_view_change_replays_the_graph(renderers):
    from vello_b200.renderer import Renderer
    r, _ = renderers
    size = 512
    packed = resolve(scenes.paris_like(1200, size, seed=12).encoding)
    views = [zoom(k, 100.0 + 30 * k, 300.0 - 20 * k, size, 0.1 * k) for k in (1, 2, 3, 5)]
    p = RenderParams(BASE, size, size, AA_MSAA16)
    r.set_cuda_graph(True)
    r.upload(packed)
    for v in views:  # arenas grown for every view (growing one captures again), graph captured
        r.set_view(v)
        render(r, p)
    caps = r.debug_graph_captures()
    off = Renderer()
    off.set_cuda_graph(False)
    off.upload(packed)
    for v in views:
        r.set_view(v)
        img, _ = render(r, p)
        off.set_view(v)
        assert np.array_equal(img, render(off, p)[0])
    assert r.debug_graph_captures() == caps
    off.close()


def test_enqueued_frames_keep_their_views(renderers):
    torch = pytest.importorskip("torch")
    r, ref = renderers
    size = 512
    packed = resolve(scenes.paris_like(1200, size, seed=13).encoding)
    views = [Affine(), zoom(2, 200.0, 200.0, size), zoom(6, 400.0, 90.0, size, -0.7)]
    p = RenderParams(BASE, size, size, AA_MSAA16)
    r.upload(packed)
    for v in views:  # arenas large enough for each view: an enqueued frame is not re-run
        r.set_view(v)
        render(r, p)
    outs = [torch.empty((size, size, 4), dtype=torch.uint8, device="cuda") for _ in views]
    for v, o in zip(views, outs):
        r.set_view(v)
        r.enqueue(p, o.data_ptr())
    assert r.finish().failed == 0
    for v, o in zip(views, outs):
        assert np.array_equal(o.cpu().numpy(), host_frame(ref, packed, v, p)[0])


def test_cleared_view_is_the_unviewed_pipeline(renderers):
    from vello_b200.renderer import Renderer
    r, _ = renderers
    size = 512
    packed = resolve(scenes.paris_like(1200, size, seed=14).encoding)
    p = RenderParams(BASE, size, size, AA_MSAA16)
    view_frame(r, packed, zoom(4, 100.0, 100.0, size), p)
    r.set_view(None)
    img, st = render(r, p)
    fresh = Renderer()
    fresh.upload(packed)
    want, wst = render(fresh, p)
    assert np.array_equal(img, want)
    assert st.kernel_launches == wst.kernel_launches and st.lines == wst.lines
    for name in ("lines", "path_bboxes", "draw_bboxes", "paths", "tiles", "draw_monoids"):
        assert r.download(name, np.uint8).tobytes() == fresh.download(name, np.uint8).tobytes(), name
    cfg = r.download("config", np.uint32)
    assert cfg[CFG_TRANSFORM_BASE] == packed.layout.transform_base and cfg[CFG_SCENE_WORDS] == packed.scene.size
    assert cfg[CFG_VIEW_SRC] == 0 and cfg[CFG_FRAME_CULL] == 0
    fresh.close()


# word offsets in VbConfig (vb_types.h)
CFG_TRANSFORM_BASE, CFG_SCENE_WORDS, CFG_VIEW_SRC, CFG_FRAME_CULL = 13, 27, 34, 35


def test_view_of_a_layout_outside_the_scene_writes_nothing():
    """A layout whose style stream ends past the uploaded words: the view region is empty, the frame launches no view kernel
    and reads its transforms as zeros (vb_scene's bound), exactly like the unviewed frame of that layout reads past the scene."""
    import dataclasses
    from vello_b200.encoding import Packed
    from vello_b200.renderer import Renderer
    good = resolve(scenes.stroke_styles()[0].encoding)
    lay = dataclasses.replace(good.layout, style_base=int(good.scene.size) + 600)
    bad = Packed(good.scene, lay, good.ramps, good.atlas)
    p = RenderParams(BASE, 256, 256, AA_MSAA16)
    r = Renderer()
    r.upload(good)
    _, plain = render(r, p)
    r.set_view(Affine.translate(3.0, 4.0))
    _, viewed_st = render(r, p)
    assert viewed_st.kernel_launches == plain.kernel_launches + 1  # the view kernel of a scene that holds its transforms
    cfg = r.download("config", np.uint32)
    n_t = (good.layout.style_base - good.layout.transform_base) // 6
    assert cfg[CFG_TRANSFORM_BASE] == good.scene.size and cfg[CFG_SCENE_WORDS] == good.scene.size + 6 * n_t
    r.set_view(None)
    r.upload(bad)
    _, bad_plain = render(r, p)
    r.set_view(Affine.translate(3.0, 4.0))
    _, bad_viewed = render(r, p)
    assert bad_viewed.failed == 0 and bad_viewed.kernel_launches == bad_plain.kernel_launches
    cfg = r.download("config", np.uint32)
    assert cfg[CFG_TRANSFORM_BASE] == cfg[CFG_SCENE_WORDS] == good.scene.size  # an empty region
    assert r.download("scene", np.uint32).tobytes() == good.scene.astype(np.uint32).tobytes()
    r.close()


def test_streamed_frame_rerun_keeps_its_view(renderers):
    """vb_render_begin with the view changed between frames while a frame in flight overflows the lines arena: the frame is
    re-run under the view it was enqueued with, and every frame equals the host-mapped render of its own view."""
    import ctypes as C
    from vello_b200.renderer import FrameStats, Renderer, _Layout, _params_struct
    _, ref = renderers
    size = 512
    packed = resolve(scenes.paris_like(1200, size, seed=15).encoding)
    views = [zoom(2, 200.0, 260.0, size), zoom(5, 300.0, 100.0, size, 0.5), Affine(), zoom(3, 150.0, 380.0, size, -0.3)]
    p = RenderParams(BASE, size, size, AA_MSAA16)
    r = Renderer()
    r.set_view(views[0])
    r.upload(packed)
    _, st = render(r, p)
    r.limit_arena("lines", st.lines - 1)  # frame 0 of the stream overflows while the view has already moved on
    scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    ps = _params_struct(p)
    outs = [np.zeros((size, size, 4), dtype=np.uint8) for _ in views]
    stats = []
    for v, out in zip(views, outs):
        r.set_view(v)
        fs = FrameStats()
        rc = r.lib.vb_render_begin(r.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None,
                                   512, ramps.shape[0], atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), out.ctypes.data,
                                   C.byref(fs))
        r._check(rc, "vb_render_begin")
        stats.append(fs)
    r._check(r.lib.vb_readback_wait(r.handle), "vb_readback_wait")
    # frame 0 needs exactly st.lines under views[0], so it overflowed and was re-run after views[1] was set; a frame left
    # unwritten or re-run under a later view would differ from its reference below
    assert all(fs.failed == 0 for fs in stats[2:])
    for k, (v, out) in enumerate(zip(views, outs)):
        assert np.array_equal(out, host_frame(ref, packed, v, p)[0]), k
    r.close()


def test_retry_under_a_view_composes_once(renderers, oracle):
    from vello_b200.renderer import Renderer
    size = 1024
    scene = scenes.paris_like(2500, size, seed=21)
    packed = resolve(scene.encoding)
    view = zoom(4, 300.0, 500.0, size, 0.3)
    p = RenderParams(BASE, size, size, AA_MSAA16)
    r = Renderer()
    img0, st0 = view_frame(r, packed, view, p)
    need = st0.lines
    r.limit_arena("lines", need - 1)
    img, st = render(r, p)
    assert st.retries == 1 and st.lines == need
    assert np.array_equal(img, img0)
    assert r.download("scene", np.uint32).tobytes() == packed.scene.astype(np.uint32).tobytes()  # the upload is untouched
    want = viewed(packed, view)
    ref = oracle.render(want, size, size, BASE.premul_rgba8_u32(), AA_MSAA16)
    assert np.array_equal(img, ref)
    r.close()
