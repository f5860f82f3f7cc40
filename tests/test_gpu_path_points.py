"""Bound path points (Renderer.bind_path_points, vb_bind_path_points): every frame reads point k of the scene's path data from
row k of a device array, read when the frame runs. `r` binds; `ref` takes the host route, the packed scene with path-data
words 2k and 2k + 1 overwritten by the f32 bits of every finite row k and uploaded, and every frame of `r` must equal it. Run
on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, DRAWTAG_BEGIN_CLIP, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL,
                                 STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Color, FILL_EVEN_ODD, FILL_NON_ZERO, Gradient, Image, MIX_MULTIPLY,
                                 MIX_SCREEN, Packed, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Arc, BezPath, Circle, Ellipse, Rect, RoundedRect

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_draw_colors import box_tiles, mixed as colour_mixed, rand_colors, recolor, solid_draws
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels
from .test_i16_path import integral_scene, to_i16

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
IMG = np.random.default_rng(21).integers(0, 256, (18, 22, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]
JOINS_CAPS = [(STYLE_JOIN_BEVEL, STYLE_CAP_BUTT), (STYLE_JOIN_MITER, STYLE_CAP_SQUARE), (STYLE_JOIN_ROUND, STYLE_CAP_ROUND)]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def bez(*els):
    p = BezPath()
    p.els = list(els)
    return p


def star(cx, cy, r0, r1, n=7):
    a = np.arange(2 * n) * np.pi / n
    rad = np.where(np.arange(2 * n) % 2 == 0, r1, r0)
    pts = [(float(cx + q * np.cos(t)), float(cy + q * np.sin(t))) for q, t in zip(rad, a)]
    return bez(("M", *pts[0]), *[("L", *p) for p in pts[1:]], ("Z",))


class Recording:
    """A Scene that notes, for every draw object a call adds, the point rows the call produced (`n_points` before and after
    it): the encoder's own account of which rows belong to which path, independent of the tag arithmetic."""

    def __init__(self):
        self.scene = Scene()
        self.spans = {}

    def __getattr__(self, name):
        f = getattr(self.scene, name)
        if not callable(f):
            return f

        def call(*a, **k):
            d, p = self.scene.n_draw_objects, self.scene.n_points
            f(*a, **k)
            if self.scene.n_draw_objects > d:
                assert self.scene.n_draw_objects == d + 1
                self.spans[d] = (p, self.scene.n_points)
        return call


def mixed(seed=0, dx=0.0, s=None):
    """Non-zero and even-odd fills, open and closed strokes of every join and cap, a dash, quads, cubics and arcs, gradient
    and image fills, nested clips and blend layers (into `s`, a new Scene by default)."""
    g = np.random.default_rng(seed)

    def col():
        c = g.uniform(0, 1, 4)
        c[3] = g.choice([1.0, 0.8, 0.5])
        return Color(*map(float, c))

    s = Scene() if s is None else s
    s.fill(FILL_NON_ZERO, Affine.translate(dx, 0), col(), None, star(60, 60, 20, 50))
    s.fill(FILL_EVEN_ODD, Affine.IDENTITY, col(), None, bez(("M", dx + 120, 20), ("L", dx + 200, 90), ("L", dx + 110, 90), ("L", dx + 190, 20),
                                                         ("L", dx + 155, 110), ("Z",)))
    for j, (join, cap) in enumerate(JOINS_CAPS):
        zig = bez(("M", dx + 220, 20 + 30 * j), ("L", dx + 250, 45 + 30 * j), ("L", dx + 280, 20 + 30 * j), ("L", dx + 320, 40 + 30 * j))
        s.stroke(Stroke(7.0, join=join, start_cap=cap, end_cap=cap), Affine.IDENTITY, col(), None, zig)
    s.stroke(Stroke(5.0, join=STYLE_JOIN_MITER), Affine.rotate(0.05), col(), None, star(dx + 340, 60, 12, 28, 5))
    s.stroke(Stroke(2.5, dash_pattern=(9.0, 4.0), dash_offset=2.0), Affine.IDENTITY, col(), None, Circle(dx + 60, 170, 40))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, col(), None, bez(("M", dx + 120, 130), ("Q", dx + 200, 100, dx + 210, 170),
                                                         ("C", dx + 220, 230, dx + 150, 250, dx + 130, 200), ("Z",)))
    s.stroke(Stroke(4.0), Affine.IDENTITY, col(), None, Arc(dx + 290, 170, 50, 35, 0.3, 3.5, 0.2))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((dx + 20, 230), (dx + 140, 300), STOPS), None, Ellipse(dx + 80, 265, 60, 30, 0.4))
    s.fill(FILL_NON_ZERO, Affine.translate(dx + 160, 250) * Affine.scale(2.0), Image(IMG), None, star(11, 9, 5, 12, 6))
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Circle(dx + 250, 250, 70))
    s.push_clip_layer(FILL_EVEN_ODD, Affine.rotate(0.1), star(dx + 250, 220, 30, 60, 6))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, col(), None, RoundedRect(dx + 190, 190, 320, 300, 16))
    s.pop_layer()
    s.pop_layer()
    s.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, Rect(dx + 300, 230, 380, 310))
    s.stroke(Stroke(3.0), Affine.IDENTITY, col(), None, Rect(dx + 310, 240, 370, 300))
    s.pop_layer()
    return s


def path_data(packed):
    L = packed.layout
    return packed.scene[L.path_data_base:L.draw_tag_base]


def points(packed):
    """The encoded points of a packed f32 scene, (n_points, 2) float32."""
    return path_data(packed).view(np.float32).reshape(-1, 2).copy()


def patched(packed, rows):
    """The host route: the packed scene with path-data words 2k, 2k + 1 replaced by the bits of every finite row k."""
    L = packed.layout
    scene = np.array(packed.scene, dtype=np.uint32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    ok = np.isfinite(rows).all(1)
    pd = scene[L.path_data_base:L.path_data_base + 2 * len(rows)].reshape(-1, 2)
    pd[ok] = rows[ok].view(np.uint32)
    return Packed(scene, L, packed.ramps, packed.atlas)


def path_first(packed):
    """The first point of every path (n_paths + 1 entries), from the tag bytes: a byte of segment type t reads t new points,
    one more when it ends a subpath, and a TAG_PATH byte ends a path."""
    L = packed.layout
    tags = packed.scene[L.path_tag_base:L.path_data_base].view(np.uint8)
    first, n = [0], 0
    for t in tags.tolist():
        n += (t & 3) + ((t >> 2) & 1)
        if t & 0x10:
            first.append(n)
    return first[:L.n_paths + 1]


def moved(packed, seed, amp=4.0):
    g = np.random.default_rng(seed)
    p = points(packed)
    return (p + g.uniform(-amp, amp, p.shape)).astype(np.float32)


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


def check_intermediates(r, ref, want_pd):
    got = r.download("path_data", np.uint32)
    assert np.array_equal(got, want_pd) and np.array_equal(got, ref.download("path_data", np.uint32))
    for name in ("ptcl", "draw_bboxes"):
        assert np.array_equal(r.download(name, np.uint32), ref.download(name, np.uint32)), name


# ---- 1. equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_bound_equals_the_host_route(rr, aa):
    r, ref = rr
    packed = resolve(mixed().encoding)
    assert len(path_first(packed)) == packed.layout.n_paths + 1 and path_first(packed)[-1] == len(points(packed))
    r.upload(packed)
    rows = moved(packed, 1)
    r.bind_path_points(on_device(rows))
    img, _ = frame(r, aa)
    host = patched(packed, rows)
    ref.upload(host)
    want, _ = frame(ref, aa)
    check_intermediates(r, ref, path_data(host))
    same(img, want, aa)
    x = Renderer()  # the scene as encoded, on a renderer of its own: r and ref keep the same history of frames
    try:
        x.upload(packed)
        assert not (img == frame(x, aa)[0]).all()  # the points did move something
    finally:
        x.close()


# ---- 2. which rows are read ------------------------------------------------------------------------------------------------
def test_partial_non_finite_strided_and_far_rows(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    r.upload(packed)
    n = len(points(packed))
    rows = moved(packed, 2, 6.0)
    for j, (k, c, v) in enumerate([(0, 0, np.nan), (3, 1, np.inf), (7, 0, -np.inf), (12, 1, np.nan), (20, 0, np.inf)]):
        rows[k, c] = v
    rows[30] = (1e5, -1e5)  # far outside the frame
    rows[31] = (-9.5e4, 1e5)
    for m in (n, n - 17, 40, 1):
        r.bind_path_points(on_device(rows[:m]))
        img, _ = frame(r)
        host = patched(packed, rows[:m])
        ref.upload(host)
        assert np.array_equal(r.download("path_data", np.uint32), path_data(host)), m
        assert (img == frame(ref)[0]).all(), m
    # rows as columns 4:6 of a wider state tensor
    state = torch.randn((n, 7), dtype=torch.float32, device="cuda")
    state[:, 4:6] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    r.bind_path_points(state[:, 4:6])
    img, _ = frame(r)
    ref.upload(patched(packed, rows))
    assert (img == frame(ref)[0]).all()
    # every row non-finite: the scene as encoded
    r.bind_path_points(on_device(np.full((n, 2), np.nan, np.float32)))
    img, _ = frame(r)
    assert np.array_equal(r.download("path_data", np.uint32), path_data(packed))
    ref.upload(packed)
    assert (img == frame(ref)[0]).all()


# ---- 3. the rows are the encoder's points ----------------------------------------------------------------------------------
def test_translated_points_equal_the_translated_shape(rr):
    """Fills keep their tags under a translation by a dyadic offset of integral points, so moving a shape's rows equals
    encoding the moved shape, stream and pixels."""
    r, ref = rr
    shapes = [lambda x, y: Rect(x + 10, y + 10, x + 60, y + 45),
              lambda x, y: bez(("M", x + 100, y + 20), ("L", x + 160, y + 30), ("L", x + 130, y + 90), ("Z",)),
              lambda x, y: bez(("M", x + 200, y + 20), ("Q", x + 260, y + 10, x + 250, y + 70), ("C", x + 240, y + 110, x + 190, y + 90, x + 205, y + 60)),
              lambda x, y: bez(("M", x + 20, y + 150), ("L", x + 90, y + 150), ("L", x + 90, y + 220), ("L", x + 20, y + 150), ("Z",),
                               ("M", x + 40, y + 170), ("L", x + 70, y + 170), ("L", x + 70, y + 200))]
    offsets = [(3.25, -1.5), (-7.0, 12.75), (0.5, 0.125), (40.0, -22.25)]

    def scene(moves):
        s, spans = Scene(), []
        for j, sh in enumerate(shapes):
            a = s.n_points
            s.fill(FILL_NON_ZERO if j % 2 else FILL_EVEN_ODD, Affine.IDENTITY, Color(0.2 * j, 0.5, 0.9 - 0.2 * j, 0.9), None, sh(*moves[j]))
            spans.append((a, s.n_points))
        return s, spans

    s0, spans = scene([(0.0, 0.0)] * len(shapes))
    s1, spans1 = scene(offsets)
    assert spans == spans1
    packed0, packed1 = resolve(s0.encoding), resolve(s1.encoding)
    rows = points(packed0)
    for (a, b), d in zip(spans, offsets):
        rows[a:b] += np.float32(d)
    assert np.array_equal(patched(packed0, rows).scene, packed1.scene)
    r.upload(packed0)
    r.bind_path_points(on_device(rows))
    ref.upload(packed1)
    assert (frame(r)[0] == frame(ref)[0]).all()


# ---- 4. updates without calls ----------------------------------------------------------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [moved(packed, 100 + j, 3.0) for j in range(10)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(all_rows.shape[1:], dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_path_points(t)
    caps = None
    for j in range(len(seq)):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        assert st.kernel_launches == unbound + 1
        ref.upload(patched(packed, seq[j]))
        assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    # unbound again: the launches, config and graph of a renderer that never bound
    r.bind_path_points(None)
    ref.upload(packed)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)  # VbConfig's arena capacities, which only grow
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)
    caps = r.debug_graph_captures()
    r.render_resident(p)
    assert r.debug_graph_captures() == caps


# ---- 5. with other features ------------------------------------------------------------------------------------------------
def test_view_run_stages_and_rerun(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    rows = moved(packed, 5)
    r.upload(packed)
    r.bind_path_points(on_device(rows))
    ref.upload(patched(packed, rows))
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
    # split vb_run_stages ranges: the range with flatten reads the rows as they are then
    p = RenderParams(BASE, W, H, AA_MSAA16)
    t = on_device(moved(packed, 55))
    r.bind_path_points(t)
    r.run_stages(p, "pathtag", "pathtag")
    t.copy_(torch.from_numpy(rows))
    torch.cuda.synchronize()
    r.run_stages(p, "flatten", "flatten")
    t.copy_(torch.from_numpy(moved(packed, 56)))  # read by no later stage
    torch.cuda.synchronize()
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    t.copy_(torch.from_numpy(rows))
    torch.cuda.synchronize()
    # a blocking frame re-run after an arena overflow reads the same rows
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    st = r.render_resident(p)
    assert st.retries == 1
    assert (r.download_target(p) == want).all()
    assert np.array_equal(r.download("path_data", np.uint32), path_data(patched(packed, rows)))


def test_with_bound_instance_transforms_and_colours(rr):
    """A composed scene's points are global in instance order; all three bindings apply together."""
    r, ref = rr
    frags = [colour_mixed(seed=k) for k in range(3)]
    inst = [0, 1, 2, 1, 0]
    ids = [r.upload_fragment(f) for f in frags]
    lay, offs = r.compose([(ids[i], None) for i in inst])
    whole = Scene()
    for i in inst:
        whole.append(colour_mixed(seed=i))
    n_pts = whole.n_points
    xf = rand_rows(len(inst), 6, 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    cols = rand_colors(lay.n_draw_objects, 7)
    pts = moved(resolve(whole.encoding), 8, 5.0)
    pts[n_pts // 2] = np.nan
    r.bind_instance_transforms(on_device(xf))
    r.bind_draw_colors(on_device(cols))
    r.bind_path_points(on_device(pts))
    host = Scene()
    for k, i in enumerate(inst):
        solid = [offs[k] + d for d in solid_draws(colour_mixed(seed=i))]
        host.append(colour_mixed(recolor(cols, solid), seed=i, base=offs[k]), aff(xf[k]))
    packed = patched(resolve(host.encoding), pts)
    ref.upload(packed)
    img, _ = frame(r)
    want, _ = frame(ref)
    assert np.array_equal(r.download("path_data", np.uint32), path_data(packed))
    assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
    assert (img == want).all()
    r.bind_instance_transforms(None)  # colours and points stay bound
    r.bind_draw_colors(None)
    host = Scene()
    for i in inst:
        host.append(colour_mixed(seed=i))
    ref.upload(patched(resolve(host.encoding), pts))
    assert (frame(r)[0] == frame(ref)[0]).all()
    for f in ids:
        r.free_fragment(f)


def test_batch_global_points(rr):
    r, ref = rr
    cells = [mixed(seed=k) for k in range(3)]
    whole, offs = Scene(), [0]
    for c in cells:
        whole.append(c)
        offs.append(whole.n_draw_objects)
    packed = resolve(whole.encoding)
    rows = moved(packed, 9)
    r.upload(packed)
    r.bind_path_points(on_device(rows))
    r.set_cells(offs)  # the binding survives it
    ref.upload(patched(packed, rows))
    ref.set_cells(offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


# ---- 6. hit tests and hit maps ---------------------------------------------------------------------------------------------
def test_hit_tests_and_maps_follow_the_points(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    rows = moved(packed, 10, 12.0)
    r.upload(packed)
    r.bind_path_points(on_device(rows))
    ref.upload(patched(packed, rows))
    frame(r, AA_AREA)
    frame(ref, AA_AREA)
    pts = np.random.default_rng(10).uniform(0, [W, H], (5000, 2)).astype(np.float32)
    got = r.hit_test(pts)
    assert (got >= 0).sum() > 500 and (got == ref.hit_test(pts)).all()
    assert (r.hit_map() == ref.hit_map()).all()


def test_transform_launches_stop_at_their_region(rr):
    """The regions past the scene's streams lie in the order bound transforms, viewed transforms, bound draw data, bound path
    data. A range of vb_run_stages that starts at draw writes the transforms again, and not the path data: the bound path
    data must come through unchanged, so neither transform launch may reach past its own region."""
    r, ref = rr
    p = RenderParams(BASE, W, H, AA_MSAA16)
    view = Affine.translate(-20, 12) * Affine.scale(1.2)
    # a view over an uploaded scene, with points bound
    packed = resolve(mixed().encoding)
    rows = moved(packed, 60)
    host = patched(packed, rows)
    r.upload(packed)
    r.bind_path_points(on_device(rows))
    ref.upload(host)
    r.set_view(view)
    ref.set_view(view)
    try:
        want, _ = frame(ref)
        r.run_stages(p, "pathtag", "flatten")  # a frame split in two ranges; the second writes the transforms again
        out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        r.run_stages(p, "draw", "fine", out.data_ptr())
        assert np.array_equal(r.download("path_data", np.uint32), path_data(host))
        assert (out.cpu().numpy() == want).all()
    finally:
        r.set_view(None)
        ref.set_view(None)
    # a composed scene with instance transforms and points bound
    frags = [colour_mixed(seed=k) for k in range(2)]
    ids = [r.upload_fragment(f) for f in frags]
    inst = [0, 1, 0]
    r.compose([(ids[i], None) for i in inst])
    whole = Scene()
    for i in inst:
        whole.append(colour_mixed(seed=i))
    xf = rand_rows(len(inst), 61, 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    pts = moved(resolve(whole.encoding), 62)
    r.bind_instance_transforms(on_device(xf))
    r.bind_path_points(on_device(pts))
    host = Scene()
    for k, i in enumerate(inst):
        host.append(colour_mixed(seed=i), aff(xf[k]))
    host = patched(resolve(host.encoding), pts)
    ref.upload(host)
    want, _ = frame(ref)
    r.run_stages(p, "pathtag", "flatten")
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert np.array_equal(r.download("path_data", np.uint32), path_data(host))
    assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
    assert (out.cpu().numpy() == want).all()
    r.bind_instance_transforms(None)
    for f in ids:
        r.free_fragment(f)


# ---- 7. damage tracking ----------------------------------------------------------------------------------------------------
class Tracked:
    """`r` tracks damage into the device array `dst` with `rows` bound; `ref` renders the patched scene in full."""

    def __init__(self, r, ref, seed):
        self.r, self.ref = r, ref
        rec = Recording()
        mixed(s=rec)
        self.packed = resolve(rec.encoding)
        # each path's point rows as the encoder produced them (path d is draw object d)
        self.first = [rec.spans[d][0] for d in range(len(rec.spans))] + [rec.scene.n_points]
        assert all(rec.spans[d][1] == self.first[d + 1] for d in range(len(rec.spans)))
        assert self.first == path_first(self.packed)
        r.upload(self.packed)
        self.rows = moved(self.packed, seed, 2.0)
        self.t = on_device(self.rows)
        r.bind_path_points(self.t)
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
        self.ref.upload(patched(self.packed, self.rows) if self.bound else self.packed)
        assert (self.dst.cpu().numpy() == frame(self.ref)[0]).all()
        return self.r.last_damage()

    def span(self, d):
        return slice(self.first[d], self.first[d + 1])


def test_damage_follows_moved_points(rr):
    r, ref = rr
    d = Tracked(r, ref, 11)
    try:
        assert d.step().sum() == d.n_tiles  # the first tracked frame is full
        tags = d.packed.scene[d.packed.layout.draw_tag_base:d.packed.layout.draw_tag_base + d.packed.layout.n_draw_objects]
        clip = int(np.nonzero(tags == DRAWTAG_BEGIN_CLIP)[0][1])  # the inner BEGIN_CLIP: its clip path moves
        # every path with points alone (each entry of the device's table of first points is then checked against the encoder's
        # spans: a wrong entry marks a neighbouring path), then several at once
        alone = [[k] for k in range(len(d.first) - 1) if d.first[k + 1] > d.first[k]]
        assert [clip] in alone and len(alone) >= 14
        for paths in alone + [[1, 6, 9]]:
            before = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            new = d.rows.copy()
            for k in paths:
                assert d.first[k + 1] > d.first[k]
                new[d.span(k)] += np.float32([9.0, -6.0])
            got = d.step(new)
            after = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            want = box_tiles(before[paths]) | box_tiles(after[paths])
            assert got.any() and (got == want).all(), paths
        assert d.step().sum() == 0  # nothing changed
        # a path moved back to its encoded points, then the same words through non-finite rows: no change
        new = d.rows.copy()
        new[d.span(2)] = points(d.packed)[d.span(2)]
        assert d.step(new).any()
        same = new.copy()
        same[d.span(2), 0] = np.nan
        assert d.step(same).sum() == 0
        # bind, unbind and rebind each make the next frame full
        t2 = on_device(same)
        for bind in (t2, None, d.t):
            r.bind_path_points(bind)
            d.bound = bind is not None
            assert d.step().sum() == d.n_tiles
            assert d.step().sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_path_points(None)


def test_diffs_after_a_bound_base_are_full(rr):
    r, ref = rr
    d = Tracked(r, ref, 12)
    try:
        d.step()
        # an upload diffed against a bound base: full, and without points bound afterwards the scene as encoded
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
        fid = r.upload_fragment(mixed())
        r.compose([(fid, None)])
        r.bind_path_points(d.t)
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
    return r.lib.vb_bind_path_points(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding(rr):
    r, ref = rr
    s = mixed()
    packed = resolve(s.encoding)
    n = s.n_points
    r.upload(packed)
    rows = moved(packed, 13)
    t = on_device(rows)
    r.bind_path_points(t)
    before, _ = frame(r)

    def unchanged(what):
        assert r.lib.vb_last_error(r.handle), what
        assert (frame(r)[0] == before).all(), what

    ptr = t.data_ptr()
    host = np.zeros((n, 2), dtype=np.float32)
    for args in ((ptr, 0, 8), (ptr, n + 1, 8), (host.ctypes.data, n, 8), (ptr + 2, n, 8), (ptr, n, 4), (ptr, n, 6), (ptr, n, 10),
                 (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        unchanged(args)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    assert _bind_raw(r, ptr, n, 8) == VB_E_INVALID  # between enqueue and finish
    r.finish()
    assert (r.download_target(p) == before).all()
    with pytest.raises(ValueError):  # not (n, 2) float32 with 4-byte columns
        r.bind_path_points(torch.zeros((n, 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        r.bind_path_points(torch.zeros((2, n), dtype=torch.float32, device="cuda").t())
    unchanged("python checks")
    # a scene with 16-bit segments
    i16 = to_i16(resolve(integral_scene().encoding))
    r.upload(i16)
    assert _bind_raw(r, ptr, 1, 8) == VB_E_INVALID and b"16-bit" in r.lib.vb_last_error(r.handle)
    r.upload(packed)
    r.bind_path_points(t)
    # no scene installed, a renderer of a vb_group, and one with the exchange configured
    x = Renderer()
    try:
        assert _bind_raw(x, ptr, 1, 8) == VB_E_INVALID and b"scene" in x.lib.vb_last_error(x.handle)
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        assert _bind_raw(x, ptr, n, 8) == VB_E_INVALID and b"exchange" in x.lib.vb_last_error(x.handle)
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        assert _bind_raw(g.renderer(0), ptr, 1, 8) == VB_E_INVALID
    finally:
        g.close()
    assert (frame(r)[0] == before).all()
    # every installation unbinds; None unbinds
    from vello_b200.scene_native import NativeScene
    ref.upload(packed)
    encoded, _ = frame(ref)
    native = NativeScene()
    native.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.3, 0.6, 0.9, 1.0), None, star(100, 100, 30, 80))
    ref.upload(native.resolve())
    native_frame, _ = frame(ref)
    installs = [(lambda: r.upload(packed), encoded), (lambda: r.render_to_texture(packed, p), encoded),
                (lambda: list(r.render_stream([packed], p)), encoded), (lambda: r.recompose([(fid, None)]), encoded),
                (lambda: r.compose([(fid, None)]), encoded), (lambda: native.upload_device(r), native_frame)]
    for install, want in installs:
        fid = r.upload_fragment(s)
        r.compose([(fid, None)])
        r.bind_path_points(t)
        assert not (frame(r)[0] == encoded).all()
        install()
        assert (frame(r)[0] == want).all()
        r.free_fragment(fid)
    r.upload(packed)
    r.bind_path_points(t)
    r.bind_path_points(None)
    assert (frame(r)[0] == encoded).all()
