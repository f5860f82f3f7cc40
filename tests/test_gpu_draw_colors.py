"""Bound draw colours (Renderer.bind_draw_colors, vb_bind_draw_colors): every frame renders draw object k as if it had been
encoded with Color(row k) of a device array, read when the frame runs. `r` binds; `ref` takes the host route, the scene
re-encoded with those colours and uploaded, and every frame of `r` must equal it. Run on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, DRAWTAG_COLOR, Color, FILL_EVEN_ODD, FILL_NON_ZERO, Gradient, Image, MIX_MULTIPLY,
                                 MIX_SCREEN, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Circle, Rect, RoundedRect

from .test_draw_colors import premul_np, tie_rows
from .test_gpu_compose import BASE, _render_cells
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
BLUR_TAG = 0x2D4
IMG = np.random.default_rng(11).integers(0, 256, (18, 22, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def mixed(colors=None, seed=0, base=0, dx=0.0):
    """Fills, strokes, blurred rectangles, a gradient, an image, nested clips and blend layers. A draw object k whose paint is
    one colour takes colors[base + k] when that key is present, else its seeded colour."""
    g = np.random.default_rng(seed)
    s = Scene()
    colors = colors or {}

    def col():
        c = g.uniform(0, 1, 4)
        c[3] = g.choice([1.0, 0.75, 0.3])
        return colors.get(base + s.n_draw_objects, Color(*map(float, c)))

    for i in range(6):
        s.fill(FILL_NON_ZERO, Affine.translate(dx + 20 + 45 * i, 15 + 9 * i), col(), None, Rect(0, 0, 40, 30))
    s.stroke(Stroke(5.0), Affine.IDENTITY, col(), None, Circle(dx + 120, 120, 50))
    s.draw_blurred_rounded_rect(Affine.translate(dx + 200, 60), Rect(0, 0, 70, 40), col(), 8.0, 5.0)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (100, 0), STOPS), None, Rect(dx + 10, 180, 130, 240))
    s.draw_image(Image(IMG), Affine.translate(dx + 150, 180) * Affine.scale(2.0))
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Circle(dx + 190, 160, 90))
    s.fill(FILL_EVEN_ODD, Affine.IDENTITY, col(), None, RoundedRect(dx + 110, 90, 290, 250, 14))
    s.push_clip_layer(FILL_NON_ZERO, Affine.rotate(0.1), Rect(dx + 130, 100, 260, 220))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, col(), None, Circle(dx + 200, 170, 60))
    s.draw_blurred_rounded_rect_in(Circle(dx + 210, 150, 40), Affine.IDENTITY, Rect(dx + 180, 120, 240, 180), col(), 6.0, 4.0)
    s.pop_layer()
    s.pop_layer()
    s.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, Rect(dx + 260, 200, 370, 300))
    s.stroke(Stroke(3.0), Affine.IDENTITY, col(), None, Rect(dx + 270, 210, 350, 290))
    s.pop_layer()
    for i in range(8):
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, col(), None, Circle(dx + 30 + 40 * i, 280, 14))
    return s


def solid_draws(scene):
    """The draw objects whose paint is one colour (FILL_COLOR, BLURRED_ROUNDED_RECT)."""
    tags = scene.encoding.draw_tags
    return [k for k, t in enumerate(tags) if t in (DRAWTAG_COLOR, BLUR_TAG)]


def recolor(rows, draws):
    """The colours a frame bound to `rows` renders: Color(row k) for every listed draw object k below len(rows) whose row is
    finite."""
    return {k: Color(*map(float, rows[k])) for k in draws if k < len(rows) and np.isfinite(rows[k]).all()}


def rand_colors(n, seed):
    g = np.random.default_rng(seed)
    rows = g.uniform(0, 1, (n, 4)).astype(np.float32)
    rows[:, 3] = g.choice(np.float32([1.0, 0.5, 0.2, 0.0]), n)
    return rows


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


def draw_data(packed):
    L = packed.layout
    return packed.scene[L.draw_data_base:L.transform_base]


# ---- 1. equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_bound_equals_the_host_route(rr, aa):
    r, ref = rr
    s = mixed()
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    rows = rand_colors(n, 1)
    r.bind_draw_colors(on_device(rows))
    img, _ = frame(r, aa)
    packed = resolve(mixed(recolor(rows, solid_draws(s))).encoding)
    ref.upload(packed)
    want, _ = frame(ref, aa)
    got = r.download("draw_data", np.uint32)
    assert np.array_equal(got, draw_data(packed)) and np.array_equal(got, ref.download("draw_data", np.uint32))
    for name in ("ptcl", "draw_bboxes"):
        assert np.array_equal(r.download(name, np.uint32), ref.download(name, np.uint32)), name
    same(img, want, aa)


# ---- 2. conversion at the ties ---------------------------------------------------------------------------------------------
def test_conversion_at_the_ties(rr):
    r, _ = rr
    rows = tie_rows()
    s = Scene()
    for k in range(len(rows)):
        x, y = k % 64 * 4, k // 64 * 4
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.5, 0.5, 0.5, 1.0), None, Rect(x, y, x + 2, y + 2))
    r.upload(resolve(s.encoding))
    r.bind_draw_colors(on_device(rows))
    frame(r, AA_MSAA16, 256, 256)
    got = r.download("draw_data", np.uint32)
    want = premul_np(rows)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(rows[i].tolist(), hex(got[i]), hex(want[i])) for i in bad[:5]]


# ---- 3. non-finite rows, ignored rows, a short array -----------------------------------------------------------------------
def test_non_finite_ignored_and_tail_rows(rr):
    r, ref = rr
    s = mixed()
    n = s.n_draw_objects
    solid = solid_draws(s)
    others = [k for k in range(n) if k not in solid]
    assert len(others) >= 6  # gradient, image, BEGIN_CLIP x3, END_CLIP x3
    rows = rand_colors(n, 3)
    for j, (c, v) in enumerate([(0, np.nan), (1, np.inf), (2, -np.inf), (3, np.nan), (3, np.inf)]):
        rows[solid[j], c] = v
    packed0 = resolve(s.encoding)
    r.upload(packed0)
    for m in (n, n - 5, 3):
        r.bind_draw_colors(on_device(rows[:m]))
        img, _ = frame(r)
        packed = resolve(mixed(recolor(rows[:m], solid)).encoding)
        ref.upload(packed)
        assert np.array_equal(r.download("draw_data", np.uint32), draw_data(packed)), m
        assert (img == frame(ref)[0]).all(), m
    # rows of gradients, images and clips change nothing
    only_others = rand_colors(n, 4)
    only_others[solid] = np.nan
    r.bind_draw_colors(on_device(only_others))
    img, _ = frame(r)
    assert np.array_equal(r.download("draw_data", np.uint32), draw_data(packed0))
    ref.upload(packed0)
    assert (img == frame(ref)[0]).all()


# ---- 4. updates without calls ----------------------------------------------------------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    s = mixed()
    n = s.n_draw_objects
    packed0 = resolve(s.encoding)
    r.upload(packed0)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [rand_colors(n, 100 + j) for j in range(12)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_draw_colors(t)
    caps = None
    for j in range(12):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        assert st.kernel_launches == unbound + 1
        ref.upload(resolve(mixed(recolor(seq[j], solid_draws(s))).encoding))
        assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    # unbound again: the launches, config and graph of a renderer that never bound
    r.bind_draw_colors(None)
    ref.upload(packed0)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches == unbound
    # the config of the unbound frame before the binding, but for the arena capacities (VbConfig's lines_size .. ptcl_size),
    # which only grow: a recoloured frame may need more command-list space
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)
    caps = r.debug_graph_captures()
    r.render_resident(p)
    assert r.debug_graph_captures() == caps


# ---- 5. with other features ------------------------------------------------------------------------------------------------
def test_view_run_stages_and_rerun(rr):
    r, ref = rr
    s = mixed()
    rows = rand_colors(s.n_draw_objects, 5)
    r.upload(resolve(s.encoding))
    r.bind_draw_colors(on_device(rows))
    ref.upload(resolve(mixed(recolor(rows, solid_draws(s))).encoding))
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
    # a frame split into vb_run_stages ranges: the range from DRAW writes the region again, from the rows as they are then
    p = RenderParams(BASE, W, H, AA_MSAA16)
    t = on_device(rand_colors(s.n_draw_objects, 55))
    r.bind_draw_colors(t)
    r.run_stages(p, "pathtag", "flatten")
    t.copy_(torch.from_numpy(rows))
    torch.cuda.synchronize()
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    # a blocking frame re-run after an arena overflow reads the same rows
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    st = r.render_resident(p)
    assert st.retries == 1
    assert (r.download_target(p) == want).all()


def test_with_bound_instance_transforms(rr):
    r, ref = rr
    frags = [mixed(seed=k) for k in range(3)]
    inst = [0, 1, 2, 1, 0]
    ids = [r.upload_fragment(f) for f in frags]
    lay, offs = r.compose([(ids[i], None) for i in inst])
    n = lay.n_draw_objects
    xf = rand_rows(len(inst), 6, 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    rows = rand_colors(n, 7)
    rows[offs[1] + 2] = np.nan
    r.bind_instance_transforms(on_device(xf))
    r.bind_draw_colors(on_device(rows))
    host = Scene()
    for k, i in enumerate(inst):
        local = mixed(seed=i)
        solid = [offs[k] + d for d in solid_draws(local)]
        host.append(mixed(recolor(rows, solid), seed=i, base=offs[k]), aff(xf[k]))
    packed = resolve(host.encoding)
    ref.upload(packed)
    img, _ = frame(r)
    want, _ = frame(ref)
    assert np.array_equal(r.download("draw_data", np.uint32), draw_data(packed))
    assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
    assert (img == want).all()
    r.bind_instance_transforms(None)  # colours stay bound
    host = Scene()
    for k, i in enumerate(inst):
        solid = [offs[k] + d for d in solid_draws(mixed(seed=i))]
        host.append(mixed(recolor(rows, solid), seed=i, base=offs[k]))
    ref.upload(resolve(host.encoding))
    assert (frame(r)[0] == frame(ref)[0]).all()
    for f in ids:
        r.free_fragment(f)


def test_batch_global_indices(rr):
    r, ref = rr
    cells = [mixed(seed=k) for k in range(3)]
    whole, offs = Scene(), [0]
    for c in cells:
        whole.append(c)
        offs.append(whole.n_draw_objects)
    rows = rand_colors(offs[-1], 8)
    r.upload(resolve(whole.encoding))
    r.bind_draw_colors(on_device(rows))
    r.set_cells(offs)  # the binding survives it
    host = Scene()
    for k, c in enumerate(cells):
        solid = [offs[k] + d for d in solid_draws(c)]
        host.append(mixed(recolor(rows, solid), seed=k, base=offs[k]))
    ref.upload(resolve(host.encoding))
    ref.set_cells(offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


# ---- 6. hit tests and hit maps ---------------------------------------------------------------------------------------------
def test_hit_tests_and_maps_do_not_change(rr):
    r, ref = rr
    s = mixed()
    packed = resolve(s.encoding)
    r.upload(packed)
    ref.upload(packed)
    rows = rand_colors(s.n_draw_objects, 9)
    rows[:, 3] = 0.0  # even fully transparent
    r.bind_draw_colors(on_device(rows))
    frame(r, AA_AREA)
    frame(ref, AA_AREA)
    pts = np.random.default_rng(10).uniform(0, [W, H], (5000, 2)).astype(np.float32)
    got = r.hit_test(pts)
    assert (got >= 0).sum() > 500 and (got == ref.hit_test(pts)).all()
    assert (r.hit_map() == ref.hit_map()).all()


# ---- 7. damage tracking ----------------------------------------------------------------------------------------------------
def box_tiles(boxes, w=W, h=H):
    """The tiles of draw boxes, rounded out as tile_alloc (and k_damage) round them."""
    wt, ht = (w + 15) // 16, (h + 15) // 16
    m = np.zeros((ht, wt), dtype=bool)
    for x0, y0, x1, y1 in boxes:
        if not (x0 < x1 and y0 < y1):
            continue
        s = np.float32(1 / 16)
        tx0, tx1 = int(np.clip(np.floor(np.float32(x0) * s), 0, wt)), int(np.clip(np.ceil(np.float32(x1) * s), 0, wt))
        ty0, ty1 = int(np.clip(np.floor(np.float32(y0) * s), 0, ht)), int(np.clip(np.ceil(np.float32(y1) * s), 0, ht))
        m[ty0:ty1, tx0:tx1] = True
    return m


class Tracked:
    """`r` tracks damage into the device array `dst` with `rows` bound; `ref` renders the re-encoded scene in full."""

    def __init__(self, r, ref, seed):
        self.r, self.ref = r, ref
        self.s = mixed()
        self.solid = solid_draws(self.s)
        self.packed = resolve(self.s.encoding)
        r.upload(self.packed)
        self.rows = rand_colors(self.s.n_draw_objects, seed)
        self.t = on_device(self.rows)
        r.bind_draw_colors(self.t)
        self.bound = True
        self.dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        self.p = RenderParams(BASE, W, H, AA_MSAA16)
        self.n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
        r.set_damage_tracking(True)

    def step(self, rows=None):
        """One frame with `rows` written into the bound array; its damaged tiles. The destination must equal a full frame."""
        if rows is not None:
            self.rows = rows.astype(np.float32)
            self.t.copy_(torch.from_numpy(self.rows))
            torch.cuda.synchronize()
        self.r.render_resident(self.p, self.dst.data_ptr())
        self.ref.upload(resolve(mixed(recolor(self.rows, self.solid) if self.bound else None).encoding))
        assert (self.dst.cpu().numpy() == frame(self.ref)[0]).all()
        return self.r.last_damage()


def test_damage_follows_changed_colours(rr):
    r, ref = rr
    d = Tracked(r, ref, 11)
    try:
        assert d.step().sum() == d.n_tiles  # the first tracked frame is full
        boxes = r.download("draw_bboxes", np.float32).reshape(-1, 4)
        solid = d.solid
        for changed in ([solid[2]], [solid[0], solid[7], solid[-1]], [solid[9], solid[10]]):
            new = d.rows.copy()
            for k in changed:
                new[k] = (0.9, 0.1, 0.5, 0.6) if d.rows[k, 0] < 0.5 else (0.1, 0.8, 0.3, 1.0)
            got = d.step(new)
            assert got.any() and (got == box_tiles(boxes[changed])).all(), changed
        assert d.step().sum() == 0  # nothing changed
        new = d.rows.copy()
        new[solid[1]] = (0.5, 0.5, 0.5, 1.0)
        new[solid[4], 1] = np.nan
        d.step(new)
        same = new.copy()
        same[solid[1], 0] = np.float32(0.5000001)  # converts to the same word
        same[solid[4], 2] = np.inf  # still falls back to the encoded word
        assert d.step(same).sum() == 0
        # bind, unbind and rebind each make the next frame full
        t2 = on_device(same)
        for bind in (t2, None, d.t):
            r.bind_draw_colors(bind)
            d.bound = bind is not None
            assert d.step().sum() == d.n_tiles
            assert d.step().sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_draw_colors(None)


def test_diffs_after_a_bound_base_are_full(rr):
    r, ref = rr
    d = Tracked(r, ref, 12)
    try:
        d.step()
        # an upload diffed against a bound base: full, and without colours bound afterwards the scene as encoded
        r.set_upload_diff(True)
        r.upload(d.packed)
        r.render_resident(d.p, d.dst.data_ptr())
        assert r.last_damage().sum() == d.n_tiles
        ref.upload(d.packed)
        assert (d.dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload(d.packed)  # unbound base: the same upload damages nothing
        r.render_resident(d.p, d.dst.data_ptr())
        assert r.last_damage().sum() == 0
        r.set_upload_diff(False)
        # a recompose after a bound base: full
        fid = r.upload_fragment(d.s)
        r.compose([(fid, None)])
        r.bind_draw_colors(d.t)
        r.render_resident(d.p, d.dst.data_ptr())
        r.render_resident(d.p, d.dst.data_ptr())
        r.recompose([(fid, None)])
        r.render_resident(d.p, d.dst.data_ptr())
        assert r.last_damage().sum() == d.n_tiles
        assert (d.dst.cpu().numpy() == frame(ref)[0]).all()
        r.free_fragment(fid)
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 8. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_draw_colors(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding(rr):
    r, ref = rr
    s = mixed()
    n = s.n_draw_objects
    packed = resolve(s.encoding)
    r.upload(packed)
    rows = rand_colors(n, 13)
    t = on_device(rows)
    r.bind_draw_colors(t)
    before, _ = frame(r)

    def unchanged(what):
        assert r.lib.vb_last_error(r.handle), what
        assert (frame(r)[0] == before).all(), what

    ptr = t.data_ptr()
    host = np.zeros((n, 4), dtype=np.float32)
    for args in ((ptr, 0, 16), (ptr, n + 1, 16), (host.ctypes.data, n, 16), (ptr + 2, n, 16), (ptr, n, 12), (ptr, n, 18),
                 (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        unchanged(args)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    assert _bind_raw(r, ptr, n, 16) == VB_E_INVALID  # between enqueue and finish
    r.finish()
    assert (r.download_target(p) == before).all()
    with pytest.raises(ValueError):  # not (n, 4) float32 with 4-byte columns
        r.bind_draw_colors(torch.zeros((n, 4), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        r.bind_draw_colors(torch.zeros((4, n), dtype=torch.float32, device="cuda").t())
    unchanged("python checks")
    # no scene installed, a renderer of a vb_group, and one with the exchange configured
    x = Renderer()
    try:
        assert _bind_raw(x, ptr, 1, 16) == VB_E_INVALID and b"scene" in x.lib.vb_last_error(x.handle)
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        assert _bind_raw(x, ptr, n, 16) == VB_E_INVALID and b"exchange" in x.lib.vb_last_error(x.handle)
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        assert _bind_raw(g.renderer(0), ptr, 1, 16) == VB_E_INVALID
    finally:
        g.close()
    # every installation unbinds; None unbinds
    ref.upload(packed)
    encoded, _ = frame(ref)
    for install in (lambda: r.upload(packed), lambda: r.render_to_texture(packed, p), lambda: r.recompose([(fid, None)]),
                    lambda: r.compose([(fid, None)])):
        fid = r.upload_fragment(s)
        r.compose([(fid, None)])
        r.bind_draw_colors(t)
        assert not (frame(r)[0] == encoded).all()
        install()
        assert (frame(r)[0] == encoded).all()
        r.free_fragment(fid)
    r.bind_draw_colors(t)
    r.bind_draw_colors(None)
    assert (frame(r)[0] == encoded).all()
