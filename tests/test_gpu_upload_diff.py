"""Upload diff (Renderer.set_upload_diff, vb_set_upload_diff): with damage tracking on, the frame after a re-uploaded scene repaints
only the tiles of the draw objects that were added, removed or changed, found on the device. `r` tracks and diffs, rendering
into one device array; `ref` renders the same scenes with tracking off, always in full. Every frame of `r` must equal `ref`'s
byte for byte, and its damage must equal the serial reference's (tests/upload_diff_ref.py) exactly. Run on an H100 with
`pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, DRAWTAG_COLOR, FILL_EVEN_ODD, FILL_NON_ZERO, Color, Gradient, Image, Packed, Scene,
                                 Stroke, resolve)
from vello_b200.renderer import FrameStats, Renderer, RendererGroup, VelloB200Error, _Layout, _params_struct
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Rect

from . import upload_diff_ref as udr
from .test_gpu_damage import SENTINEL, changed_tiles, pixel_mask
from .test_i16_path import integral_scene, to_i16

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 512, 384
BASE = Color.from_rgba8(12, 20, 30)
MIX_MULTIPLY = 1


@pytest.fixture()
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


# ---- scenes: a list of items, so that edits are list edits ---------------------------------------------------------------------
def rand_items(g, n, images):
    items = []
    for k in range(n):
        x, y = (float(v) for v in g.uniform([-10, -10], [W - 20, H - 20]))
        w, h = (float(v) for v in g.uniform(8, 90, 2))
        c = tuple(int(v) for v in g.integers(0, 256, 3)) + (int(g.choice([255, 160])),)
        kind = k % 7
        if kind == 3:
            items.append(("stroke", x, y, w, h, c, float(g.uniform(1, 6))))
        elif kind == 5:
            items.append(("grad", x, y, w, h, ((0.0, c), (1.0, (c[2], c[0], c[1], 255))), None))
        elif kind == 6 and images:
            items.append(("image", x, y, images[k % len(images)]))
        else:
            items.append(("fill", x, y, w, h, c, FILL_NON_ZERO))
    return items


def build(items, cls=Scene, prefix=None):
    s = cls()
    if prefix is not None:
        s.append(prefix)
    for it in items:
        k = it[0]
        if k == "fill":
            _, x, y, w, h, c, style = it
            s.fill(style, Affine.translate(x, y), Color.from_rgba8(*c), None, Rect(0, 0, w, h))
        elif k == "stroke":
            _, x, y, w, h, c, width = it
            s.stroke(Stroke(width), Affine.translate(x, y), Color.from_rgba8(*c), None, Rect(0, 0, w, h))
        elif k == "grad":
            _, x, y, w, h, stops, bt = it
            grad = Gradient.linear((0, 0), (w, h), [(o, Color.from_rgba8(*c)) for o, c in stops])
            s.fill(FILL_NON_ZERO, Affine.translate(x, y), grad, Affine.translate(*bt) if bt else None, Rect(0, 0, w, h))
        elif k == "image":
            _, x, y, im = it
            s.draw_image(im, Affine.translate(x, y))
        elif k == "clip":
            _, x, y, w, h = it
            s.push_clip_layer(FILL_NON_ZERO, Affine.translate(x, y), Rect(0, 0, w, h))
        elif k == "layer":
            _, x, y, w, h, alpha = it
            s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, alpha, Affine.translate(x, y), Rect(0, 0, w, h))
        elif k == "pop":
            s.pop_layer()
    return s


def colour_draws(packed):
    return [i for i, rec in enumerate(udr.records(packed.scene, packed.layout)) if rec[8] == DRAWTAG_COLOR]


def recoloured(packed, draws, g):
    scene = np.array(packed.scene, dtype=np.uint32)
    rec = udr.records(scene, packed.layout)
    for i in draws:
        scene[packed.layout.draw_data_base + rec[i][9]] = np.uint32(g.integers(0, 2**32)) | np.uint32(0xFF)
    return Packed(scene, packed.layout, packed.ramps, packed.atlas)


def moved(packed, draws, d, i16=False):
    """The path data of `draws` shifted by d pixels (whole pixels for i16 points)."""
    scene = np.array(packed.scene, dtype=np.uint32)
    L = packed.layout
    rec = udr.records(scene, L)
    for i in draws:
        words = scene[L.path_data_base + rec[i][2]:L.path_data_base + rec[i][3]]
        if i16:
            words += np.uint32(d) | (np.uint32(d) << 16)
        else:
            words[:] = (words.view(np.float32) + np.float32(d)).view(np.uint32)
    return Packed(scene, L, packed.ramps, packed.atlas)


def ramps_swapped(packed):
    """Rows 0 and 1 of the ramps exchanged, and every gradient's ramp word with them: the same pixels."""
    scene = np.array(packed.scene, dtype=np.uint32)
    L = packed.layout
    for rec in udr.records(scene, L):
        if rec[8] in udr.GRADIENTS:
            w = L.draw_data_base + rec[9]
            row = int(scene[w]) >> 2
            if row in (0, 1):
                scene[w] = ((1 - row) << 2) | (int(scene[w]) & 3)
    ramps = np.array(packed.ramps)
    ramps[[0, 1]] = ramps[[1, 0]]
    return Packed(scene, L, ramps, packed.atlas)


def render_device(r, packed, p, dst):
    """vb_render with a device destination (out_is_device = 1)."""
    scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    st = FrameStats()
    rc = r.lib.vb_render(r.handle, scene.ctypes.data, scene.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None, 512,
                         ramps.shape[0], atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(_params_struct(p, (0, 0), (0, 0))),
                         C.c_void_p(dst.data_ptr()), 1, C.byref(st))
    r.last_stats = st
    r._check(rc, "vb_render")
    r._frame_size = (p.width, p.height)


class Diffed:
    """`r` (tracking and the diff on, into `dst`) and `ref` (tracking off), and what the reference needs of r's last frame."""

    def __init__(self, r, ref, aa=AA_MSAA16, w=W, h=H):
        self.r, self.ref, self.w, self.h = r, ref, w, h
        self.p = RenderParams(BASE, w, h, aa)
        self.dst = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        r.set_damage_tracking(True)
        r.set_upload_diff(True)
        self.last = None  # (keys, boxes, pixels) of r's last frame
        self.pending_atlas = None

    def upload(self, scene, route="host"):
        """Install `scene` on both renderers; route "render" installs on ref only (r's vb_render uploads in step)."""
        r, ref = self.r, self.ref
        if route == "device":
            self.layout = scene.upload_device(r)
            scene.upload_device(ref)
            self.atlas = None
            return
        packed = scene if isinstance(scene, Packed) else resolve(scene.encoding)
        self.layout, self.atlas, self.packed = packed.layout, packed.atlas, packed
        if route == "host":
            r.upload(packed)
        ref.upload(packed)

    def frame(self, route="host", p=None, dst=None):
        p = p or self.p
        dst = self.dst if dst is None else dst
        if route == "render":
            render_device(self.r, self.packed, p, dst)
        else:
            self.r.render_resident(p, dst.data_ptr())
        self.ref.render_resident(p)
        n = p.width * p.height * 4
        return dst.view(-1)[:n].view(p.height, p.width, 4).cpu().numpy(), self.ref.download_target(p)

    def state(self):
        r, L = self.r, self.layout
        scene = r.download("scene", np.uint32)
        ramps = r.download("ramps", np.uint32).reshape(-1, 512)
        keys = udr.keys(scene, L, ramps, self.atlas)
        boxes = r.download("draw_bboxes", np.float32).reshape(-1, 4)[:L.n_draw_objects]
        return keys, boxes

    def step(self, scene, route="host", diffed=True, what=""):
        """Upload `scene` (None: it already is), render a frame of each; check the pixels and the damage. Returns the damage."""
        before = self.last
        if scene is not None:
            self.upload(scene, route)
        img, want = self.frame(route)
        assert (img == want).all(), f"{what}: {int((img != want).any(axis=2).sum())} pixels differ from the full frame"
        dmg = self.r.last_damage()
        keys, boxes = self.state()
        if diffed:
            assert before is not None
            exp = udr.damage(before[0], keys, before[1], boxes, self.w, self.h)
            assert (dmg == exp).all(), f"{what}: {int((dmg != exp).sum())} tiles differ from the reference's damage " \
                                       f"({int(dmg.sum())} vs {int(exp.sum())})"
            missing = changed_tiles(before[2], want) & ~dmg
            assert not missing.any(), f"{what}: tiles {np.argwhere(missing)[:4].tolist()} changed but are not damaged"
        else:
            assert dmg.all(), f"{what}: expected a full frame"
        self.last = (keys, boxes, want)
        return dmg


def images(g, n=2, size=24):
    return [Image(g.integers(0, 256, (size, size, 4), dtype=np.uint8)) for _ in range(n)]


# ---- exactness and the damage over many re-uploads, in every AA mode ----------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_diffed_frames_equal_full_frames(rr, aa):
    r, ref = rr
    s = Diffed(r, ref, aa)
    g = np.random.default_rng(7)
    ims = images(g)
    tiger = scenes.tiger(W, H)
    pre = rand_items(g, 6, ims)
    items = rand_items(g, 40, ims)
    items[20:20] = [("clip", 100, 80, 200, 150)] + rand_items(g, 5, []) + [("pop",)]
    grad_ix = [k for k, it in enumerate(items) if it[0] == "grad"]

    def packed_of(pre_items, its):
        sc = build(pre_items)
        sc.append(tiger)
        return resolve(build(its, prefix=sc).encoding)

    p0 = packed_of(pre, items)
    s.step(p0, diffed=False, what="first")
    assert not s.step(p0, what="identical").any()
    cols = colour_draws(p0)
    s.step(recoloured(p0, [cols[40]], g), what="recolour 1")
    s.step(recoloured(p0, list(g.choice(cols, 5, replace=False)), g), what="recolour 5")
    s.step(moved(p0, [cols[60]], 7.5), what="move 1")
    s.step(moved(p0, list(g.choice(cols, 3, replace=False)), -4.25), what="move 3")
    extra = rand_items(g, 3, [])
    s.step(packed_of(extra[:1] + pre, items), what="insert at the start")
    s.step(packed_of(pre[1:], items), what="delete at the start")
    s.step(packed_of(pre, items[:10] + extra + items[10:]), what="insert in the middle")
    s.step(packed_of(pre, items[:10] + items[12:]), what="delete in the middle")
    s.step(packed_of(pre, items + extra[:2]), what="insert at the end")
    s.step(packed_of(pre, items[:-2]), what="delete at the end")
    s.step(p0, what="back")
    it = list(items)
    _, x, y, w, h, stops, bt = it[grad_ix[0]]
    it[grad_ix[0]] = ("grad", x, y, w, h, ((0.0, (255, 0, 0, 255)), (1.0, (0, 0, 255, 255))), bt)
    s.step(packed_of(pre, it), what="gradient stops")
    s.step(p0, what="back")
    assert p0.ramps.shape[0] >= 2
    assert not s.step(ramps_swapped(p0), what="ramps reordered").any()
    s.step(p0, what="back")
    new0 = Image(g.integers(0, 256, (24, 24, 4), dtype=np.uint8))  # other pixels, placed where ims[0] was
    it = [(k[0], k[1], k[2], new0) if k[0] == "image" and k[3] is ims[0] else k for k in items]
    assert any(k[0] == "image" and k[3] is ims[0] for k in items)
    s.step(packed_of(pre, it), what="image pixels")
    it = [("clip", 100, 80, 120, 150) if k[0] == "clip" else k for k in items]
    s.step(packed_of(pre, it), what="clip path")
    s.step(packed_of(pre, items[:30] + [("layer", 40, 40, 300, 200, 0.6)] + items[30:33] + [("pop",)] + items[33:]), what="layer added")
    s.step(p0, what="layer removed")
    it = list(items)
    k = next(k for k, v in enumerate(it) if v[0] == "fill")
    it[k] = it[k][:6] + (FILL_EVEN_ODD,)
    s.step(packed_of(pre, it), what="fill rule")
    it = list(items)
    k = next(k for k, v in enumerate(it) if v[0] == "stroke")
    it[k] = it[k][:6] + (it[k][6] + 2.0,)
    s.step(packed_of(pre, it), what="stroke width")
    it = list(items)
    _, x, y, w, h, stops, bt = it[grad_ix[1]]
    it[grad_ix[1]] = ("grad", x, y, w, h, stops, (5.0, 3.0))  # a brush transform: a transform tag inside the path's tag range
    s.step(packed_of(pre, it), what="brush transform")
    it[grad_ix[1]] = ("grad", x, y, w, h, stops, (9.0, -2.0))
    s.step(packed_of(pre, it), what="brush transform changed")
    f32 = resolve(integral_scene(seed=5).encoding)
    p16 = to_i16(f32)
    s.step(p16, what="i16 scene")
    d16 = udr.records(f32.scene, f32.layout)
    s.step(to_i16(moved(f32, [3, 17], 2.0)), what="i16 paths moved")
    assert d16
    s.step(p16, what="i16 back")
    paris = resolve(scenes.paris_like(3000, 512, seed=4).encoding)
    s.step(paris, what="paris-like")
    pc = colour_draws(paris)
    s.step(recoloured(paris, [pc[100]], g), what="paris recolour 1")
    s.step(moved(paris, list(g.choice(pc, 10, replace=False)), 3.0), what="paris move 10")
    s.step(paris, what="paris back")
    assert not s.step(paris, what="paris identical").any()
    s.step(recoloured(paris, pc, g), what="paris every path")
    s.step(p0, what="tiger again")


# ---- the three upload routes ----------------------------------------------------------------------------------------------------
def test_device_resolve_route(rr):
    r, ref = rr
    s = Diffed(r, ref, AA_MSAA8)
    g = np.random.default_rng(21)
    items = rand_items(g, 60, [])
    s.step(build(items, NativeScene), "device", diffed=False, what="first")
    assert not s.step(build(items, NativeScene), "device", what="identical").any()
    it = list(items)
    it[11] = ("fill",) + it[11][1:5] + ((1, 2, 3, 255), FILL_NON_ZERO)
    s.step(build(it, NativeScene), "device", what="recolour")
    s.step(build(items[:30] + rand_items(g, 2, []) + items[30:], NativeScene), "device", what="insert")
    s.step(build(items[1:], NativeScene), "device", what="delete at the start")
    grads = [k for k, v in enumerate(items) if v[0] == "grad"]
    it = [v for k, v in enumerate(items) if k != grads[0]]  # every later ramp moves up a row
    s.step(build(it, NativeScene), "device", what="ramps moved")
    s.step(build(items, NativeScene), "device", what="back")


def test_render_route(rr):
    r, ref = rr
    s = Diffed(r, ref, AA_AREA)
    g = np.random.default_rng(23)
    ims = images(g)
    items = rand_items(g, 50, ims)
    p0 = resolve(build(items).encoding)
    s.step(p0, "render", diffed=False, what="first")
    assert not s.step(p0, "render", what="identical").any()
    s.step(recoloured(p0, colour_draws(p0)[:2], g), "render", what="recolour 2")
    s.step(resolve(build(items[:-3]).encoding), "render", what="delete at the end")
    s.step(p0, "render", what="back")
    # a host destination stays full
    r.render_to_texture(p0, s.p)
    assert r.last_damage().all()


# ---- clean tiles are not written ---------------------------------------------------------------------------------------------------
def test_clean_tiles_are_not_written(rr):
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(29)
    items = rand_items(g, 80, images(g))
    p0 = resolve(build(items).encoding)
    s.step(p0, diffed=False)
    full = s.last[2]
    s.dst.fill_(SENTINEL)  # poison every pixel; a frame without damage must leave all of them
    torch.cuda.synchronize()
    s.upload(p0)
    img, _ = s.frame()
    assert not r.last_damage().any() and (img == SENTINEL).all()
    s.dst.fill_(SENTINEL)
    torch.cuda.synchronize()
    s.upload(recoloured(p0, colour_draws(p0)[5:7], g))
    img, want = s.frame()
    m = pixel_mask(r.last_damage(), W, H)
    assert m.any() and not m.all()
    assert (img[m] == want[m]).all() and (img[~m] == SENTINEL).all()
    assert (full[~m] == want[~m]).all()


# ---- each fallback to a full frame ----------------------------------------------------------------------------------------------
def test_full_frame_fallbacks(rr):
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(31)
    items = rand_items(g, 60, [])
    pa = resolve(build(items).encoding)
    pb = recoloured(pa, colour_draws(pa)[3:4], g)
    s.step(pa, diffed=False, what="first")
    s.step(pb, what="diffed")

    r.set_upload_diff(False)
    s.step(pa, diffed=False, what="switch off")
    r.set_upload_diff(True)
    s.step(pb, what="switched on again")

    s.upload(pa)  # two uploads without a frame between them
    s.step(pb, diffed=False, what="two uploads")
    s.step(pa, what="after two uploads")

    view = Affine.translate(-6, 4)
    r.set_view(view)
    ref.set_view(view)
    s.step(pb, diffed=False, what="view set")
    r.set_view(None)
    ref.set_view(None)
    s.step(pa, diffed=False, what="view cleared")
    s.step(pb, what="after the view")

    small = RenderParams(BASE, W - 32, H - 16, AA_MSAA16)
    s.upload(pa)
    s.frame(p=small)
    assert r.last_damage().all()
    s.step(pb, diffed=False, what="size back")
    s.step(pa, what="after the size")

    r.limit_arena("segments", 1)  # an enqueued frame is never re-run: it fails
    r.enqueue(s.p, s.dst.data_ptr())
    with pytest.raises(VelloB200Error):
        r.finish()
    s.step(pb, diffed=False, what="failed frame")
    s.step(pa, what="after the failure")

    frag = r.upload_fragment(build(items[:5]))
    rfrag = ref.upload_fragment(build(items[:5]))
    r.compose([(frag, None)])
    ref.compose([(rfrag, None)])
    img, want = s.frame()
    assert r.last_damage().all() and (img == want).all()
    t = torch.tensor([[1, 0, 0, 1, 3, 2]], dtype=torch.float32, device="cuda")
    t_ref = t.clone()
    r.bind_instance_transforms(t)
    ref.bind_instance_transforms(t_ref)
    img, want = s.frame()
    assert (img == want).all()
    s.last = None
    s.step(pa, diffed=False, what="bound base")
    s.step(pb, what="after the bound base")
    assert r.last_stats.arena_bytes > 0


def test_recompose_and_diffed_upload_without_a_frame_between(rr):
    """A recompose and a diffed upload without a frame between them, in either order: the frame is full, and still exact."""
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(47)
    items = rand_items(g, 60, [])
    pa = resolve(build(items).encoding)
    pb = recoloured(pa, colour_draws(pa)[3:4], g)
    frags = [build(items[k:k + 10]) for k in range(0, 60, 10)]
    ids, rids = [r.upload_fragment(f) for f in frags], [ref.upload_fragment(f) for f in frags]
    moved_last = [(k, Affine.translate(6, 3) if k == 5 else None) for k in range(6)]

    def compose(how, inst):
        getattr(r, how)([(ids[k], t) for k, t in inst])
        ref.compose([(rids[k], t) for k, t in inst])

    def frame(what, full):
        img, want = s.frame()
        dmg = r.last_damage()
        assert (img == want).all(), f"{what}: {int((img != want).any(axis=2).sum())} pixels differ from the full frame"
        assert dmg.all() if full else not dmg.all(), f"{what}: expected {'a full' if full else 'an incremental'} frame"

    compose("compose", [(k, None) for k in range(6)])
    frame("composed", True)
    compose("recompose", moved_last)
    frame("a recompose alone", False)
    compose("recompose", [(k, None) for k in range(6)])
    s.step(pa, diffed=False, what="a recompose, then a diffed upload")
    s.step(pb, what="a diffed upload alone")
    s.upload(pa)
    compose("recompose", moved_last)
    frame("a diffed upload, then a recompose", True)


# ---- overflow re-runs, hit tests, graphs ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arena", ["ptcl", "segments"])
def test_overflow_rerun_keeps_the_damage(rr, arena):
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(37)
    items = rand_items(g, 120, images(g))
    tiger = Scene()
    tiger.append(scenes.tiger(W, H))  # many commands per tile: ptcl's dynamic chunks are needed
    p0 = resolve(build(items, prefix=tiger).encoding)
    s.step(p0, diffed=False)
    s.upload(recoloured(p0, colour_draws(p0)[::3], g))
    r.limit_arena(arena, 1 if arena == "segments" else (W // 16) * (H // 16) * 64)  # after the upload: it keeps the diff
    dmg = s.step(None, what=f"{arena} overflow")
    assert r.last_stats.retries >= 1 and dmg.any() and not dmg.all()


def test_hit_tests_on_diffed_frames(rr):
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(41)
    items = rand_items(g, 100, images(g))
    p0 = resolve(build(items).encoding)
    s.step(p0, diffed=False)
    dmg = s.step(resolve(build(items[:40] + items[45:]).encoding))
    assert not dmg.all()
    pts = np.random.default_rng(2).uniform([0, 0], [W, H], (4000, 2)).astype(np.float32)
    assert (r.hit_test(pts) == ref.hit_test(pts)).all()


def test_alternating_uploads_replay_graphs(rr):
    r, ref = rr
    s = Diffed(r, ref)
    g = np.random.default_rng(43)
    items = rand_items(g, 80, [])
    pa = resolve(build(items).encoding)
    pb = recoloured(pa, colour_draws(pa)[7:9], g)
    s.step(pa, diffed=False)
    s.step(pb)
    s.step(pa)
    caps = r.debug_graph_captures()
    for k in range(8):
        s.step(pb if k % 2 == 0 else pa)
    assert r.debug_graph_captures() == caps


# ---- errors --------------------------------------------------------------------------------------------------------------------
def test_errors():
    r = Renderer()
    try:
        r.set_upload_diff(True)
        r.set_upload_diff(False)
        r.upload(resolve(scenes.tiger(64, 64).encoding))
        arena, nbytes = C.c_void_p(), C.c_size_t()
        r._check(r.lib.vb_exchange_configure(r.handle, 0, 1, C.byref(arena), C.byref(nbytes)), "vb_exchange_configure")
        with pytest.raises(VelloB200Error):
            r.set_upload_diff(True)
        r.set_upload_diff(False)
    finally:
        r.close()
    assert r.lib.vb_set_upload_diff(None, 1) != 0
    g = RendererGroup([0])
    try:
        with pytest.raises(VelloB200Error):
            g.renderer(0).set_upload_diff(True)
    finally:
        g.close()
