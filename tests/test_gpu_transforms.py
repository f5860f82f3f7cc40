"""Bound transforms (Renderer.bind_transforms, vb_bind_transforms): every frame reads transform-stream entry k of the scene from
row k of a device array, read when the frame runs. `r` binds; `ref` takes the host route, the packed scene with transform entry
k overwritten by the f32 bits of every finite row k and uploaded again, and every frame of `r` must equal it. Run on an H100
with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, EXTEND_REFLECT, EXTEND_REPEAT, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_MULTIPLY,
                                 MIX_SCREEN, Color, Gradient, Image, Packed, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Arc, Circle, Ellipse, Rect, RoundedRect

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_draw_colors import box_tiles, mixed as colour_mixed
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels
from .test_gpu_path_points import JOINS_CAPS, bez, star
from .test_transforms import transform_ranges

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
IMG = np.random.default_rng(22).integers(0, 256, (18, 22, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (0.6, Color(0.2, 0.9, 0.3, 0.8)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def image(q):
    im = Image(IMG)
    im.quality = q
    im.x_extend, im.y_extend = EXTEND_REPEAT, EXTEND_REFLECT
    return im


def mixed(seed=0, s=None):
    """Fills under both rules, strokes under rotation, non-uniform scale and shear with every join and cap and a dash, quads,
    cubics and arcs, gradients of every kind with brush transforms, images of the three qualities, blurred rectangles, nested
    clips with their own transforms, blend layers and a luminance mask; some calls share a transform entry."""
    g = np.random.default_rng(seed)

    def col():
        c = g.uniform(0, 1, 4)
        c[3] = g.choice([1.0, 0.8, 0.5])
        return Color(*map(float, c))

    s = Scene() if s is None else s
    s.fill(FILL_NON_ZERO, Affine.translate(60, 60), col(), None, star(0, 0, 20, 50))
    s.fill(FILL_EVEN_ODD, Affine.translate(60, 60), col(), None, star(0, 0, 8, 16, 5))  # shares the entry before
    s.fill(FILL_EVEN_ODD, Affine.translate(150, 60), col(), None, bez(("M", -30, -40), ("L", 50, 30), ("L", -40, 30), ("L", 40, -40),
                                                                      ("L", 5, 50), ("Z",)))
    shear = Affine((1.0, 0.0, 0.4, 1.0, 0.0, 0.0))
    for j, (join, cap) in enumerate(JOINS_CAPS):
        t = Affine.translate(230, 25 + 30 * j) * [Affine.rotate(0.3), Affine.scale(1.6, 0.7), shear][j]
        s.stroke(Stroke(6.0, join=join, start_cap=cap, end_cap=cap), t, col(), None, bez(("M", 0, 0), ("L", 25, 20), ("L", 50, 0), ("L", 80, 15)))
    s.stroke(Stroke(2.5, dash_pattern=(9.0, 4.0), dash_offset=2.0), Affine.translate(60, 170) * Affine.scale(1.2, 0.8), col(), None, Circle(0, 0, 40))
    s.fill(FILL_NON_ZERO, Affine.translate(120, 130), col(), None, bez(("M", 0, 0), ("Q", 80, -30, 90, 40), ("C", 100, 100, 30, 120, 10, 70), ("Z",)))
    s.stroke(Stroke(4.0), Affine.translate(290, 170), col(), None, Arc(0, 0, 50, 35, 0.3, 3.5, 0.2))
    s.fill(FILL_NON_ZERO, Affine.translate(20, 230), Gradient.linear((0, 0), (60, 30), STOPS, EXTEND_REPEAT), Affine.rotate(0.2),
           Ellipse(60, 35, 60, 30, 0.4))
    s.fill(FILL_NON_ZERO, Affine.translate(150, 240), Gradient.radial((0, 0), 2.0, (5, 3), 25.0, STOPS, EXTEND_REFLECT), Affine.scale(1.3, 0.8),
           Circle(0, 0, 35))
    s.stroke(Stroke(8.0), Affine.translate(220, 280), Gradient.sweep((0, 0), 0.0, 4.0, STOPS), Affine.translate(3, -2), Rect(-30, -20, 30, 20))
    for q in range(3):
        s.draw_image(image(q), Affine.translate(10 + 40 * q, 290) * Affine.rotate(0.1 * q))
    s.fill(FILL_NON_ZERO, Affine.translate(330, 110), image(1), Affine.scale(2.0) * Affine.rotate(0.3), star(0, 0, 10, 25, 6))
    s.draw_blurred_rounded_rect(Affine.translate(330, 50) * Affine.rotate(0.2), Rect(-20, -15, 20, 15), col(), 5.0, 4.0)
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.translate(250, 250), Circle(0, 0, 70))
    s.push_clip_layer(FILL_EVEN_ODD, Affine.translate(250, 220) * Affine.rotate(0.1), star(0, 0, 30, 60, 6))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, col(), None, RoundedRect(190, 190, 320, 300, 16))
    s.pop_layer()
    s.pop_layer()
    s.push_luminance_mask_layer(FILL_NON_ZERO, 0.9, Affine.translate(60, 110), Rect(-40, -25, 40, 25))
    s.fill(FILL_NON_ZERO, Affine.translate(60, 110), Gradient.linear((-40, 0), (40, 0), STOPS), None, Rect(-40, -25, 40, 25))
    s.pop_layer()
    s.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, Rect(300, 230, 380, 310))
    s.stroke(Stroke(3.0), Affine.IDENTITY, col(), None, Rect(310, 240, 370, 300))
    s.pop_layer()
    return s


def transforms(packed):
    L = packed.layout
    return packed.scene[L.transform_base:L.style_base].view(np.float32).reshape(-1, 6).copy()


def patched(packed, rows):
    """The host route: the packed scene with transform entry k replaced by the bits of every finite row k."""
    L = packed.layout
    scene = np.array(packed.scene, dtype=np.uint32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    ok = np.isfinite(rows).all(1)
    tr = scene[L.transform_base:L.transform_base + 6 * len(rows)].reshape(-1, 6)
    tr[ok] = rows[ok].view(np.uint32)
    return Packed(scene, L, packed.ramps, packed.atlas)


def moved(packed, seed, amp=0.15, shift=6.0):
    """Every entry rotated, scaled and sheared a little about its own origin, and moved."""
    g = np.random.default_rng(seed)
    t = transforms(packed).astype(np.float64)
    n = len(t)
    lin = np.eye(2)[None] + g.uniform(-amp, amp, (n, 2, 2))
    a, b, c, d = t[:, 0], t[:, 1], t[:, 2], t[:, 3]
    out = np.empty_like(t)
    out[:, 0] = lin[:, 0, 0] * a + lin[:, 0, 1] * b
    out[:, 1] = lin[:, 1, 0] * a + lin[:, 1, 1] * b
    out[:, 2] = lin[:, 0, 0] * c + lin[:, 0, 1] * d
    out[:, 3] = lin[:, 1, 0] * c + lin[:, 1, 1] * d
    out[:, 4:] = t[:, 4:] + g.uniform(-shift, shift, (n, 2))
    return out.astype(np.float32)


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


@pytest.fixture
def fresh():
    """Two new renderers: the ptcl holds offsets that depend on the arenas' capacities, which follow a renderer's history, so
    it is compared between renderers that rendered the same frames before."""
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def check_intermediates(r, ref, want_tr):
    got = r.download("transforms", np.uint32)
    assert np.array_equal(got, want_tr) and np.array_equal(got, ref.download("transforms", np.uint32))
    for name in ("ptcl", "draw_bboxes"):
        assert np.array_equal(r.download(name, np.uint32), ref.download(name, np.uint32)), name


def words(packed):
    L = packed.layout
    return np.asarray(packed.scene[L.transform_base:L.style_base], dtype=np.uint32)


# ---- 1. equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
@pytest.mark.parametrize("route", ["packed", "streams"])
def test_bound_equals_the_host_route(fresh, aa, route):
    r, ref = fresh
    s = mixed()
    packed = resolve(s.encoding)
    if route == "packed":
        r.upload(packed)
    else:
        r.upload_scene(s)
    rows = moved(packed, 1)
    r.bind_transforms(on_device(rows))
    img, _ = frame(r, aa)
    host = patched(packed, rows)
    ref.upload(host)
    want, _ = frame(ref, aa)
    check_intermediates(r, ref, words(host))
    same(img, want, aa)
    ref.upload(packed)
    assert not (img == frame(ref, aa)[0]).all()  # the rows did move something


def test_encoded_rows_give_the_unbound_frame(fresh):
    r, ref = fresh
    packed = resolve(mixed().encoding)
    r.upload(packed)
    ref.upload(packed)
    want, _ = frame(ref)
    r.bind_transforms(on_device(transforms(packed)))
    img, _ = frame(r)
    check_intermediates(r, ref, words(packed))
    assert (img == want).all()


def test_shared_rows_move_every_call_that_shares_them(rr):
    r, ref = rr
    s = Scene()
    for k in range(4):  # four fills, one entry
        s.fill(FILL_NON_ZERO, Affine.translate(100, 100), Color(0.2 * k, 0.5, 0.7, 0.8), None, Circle(30 * k - 45, 0, 12))
    packed = resolve(s.encoding)
    assert s.n_transforms == 1
    r.upload(packed)
    row = np.float32([[0.5, 0.3, -0.3, 1.2, 200, 150]])
    r.bind_transforms(on_device(row))
    ref.upload(patched(packed, row))
    s2 = Scene()
    for k in range(4):
        s2.fill(FILL_NON_ZERO, aff(row[0]), Color(0.2 * k, 0.5, 0.7, 0.8), None, Circle(30 * k - 45, 0, 12))
    assert np.array_equal(patched(packed, row).scene, resolve(s2.encoding).scene)
    assert (frame(r)[0] == frame(ref)[0]).all()


def test_singular_rows(rr):
    """A zero scale mid-animation: geometry collapses, and gradients and images whose brush transform is singular sample with
    an infinite inverse; the bound frame still equals the host route's."""
    r, ref = rr
    packed = resolve(mixed().encoding)
    r.upload(packed)
    rows = transforms(packed)
    n = len(rows)
    rows[1::2] = np.float32([0, 0, 0, 0, 40, 40])
    rows[2::5] = np.float32([0, 0, 0, 1.5, 10, 10])
    r.bind_transforms(on_device(rows))
    for aa in (AA_MSAA16, AA_AREA):
        img, _ = frame(r, aa)
        ref.upload(patched(packed, rows))
        same(img, frame(ref, aa)[0], aa)
    assert n > 10


# ---- 2. which rows are read ------------------------------------------------------------------------------------------------
def test_partial_non_finite_and_strided_rows(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    r.upload(packed)
    n = len(transforms(packed))
    rows = moved(packed, 2)
    for k, c, v in [(0, 0, np.nan), (3, 4, np.inf), (7, 2, -np.inf), (12, 5, np.nan)]:
        rows[k, c] = v
    for m in (n, n - 5, 9, 1):
        r.bind_transforms(on_device(rows[:m]))
        img, _ = frame(r)
        host = patched(packed, rows[:m])
        ref.upload(host)
        assert np.array_equal(r.download("transforms", np.uint32), words(host)), m
        assert (img == frame(ref)[0]).all(), m
    state = torch.randn((n, 9), dtype=torch.float32, device="cuda")
    state[:, 2:8] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    r.bind_transforms(state[:, 2:8])
    img, _ = frame(r)
    ref.upload(patched(packed, rows))
    assert (img == frame(ref)[0]).all()
    r.bind_transforms(on_device(np.full((n, 6), np.nan, np.float32)))
    img, _ = frame(r)
    assert np.array_equal(r.download("transforms", np.uint32), words(packed))
    ref.upload(packed)
    assert (img == frame(ref)[0]).all()


# ---- 3. updates without calls ----------------------------------------------------------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [moved(packed, 100 + j) for j in range(20)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(all_rows.shape[1:], dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_transforms(t)
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
    r.bind_transforms(None)
    ref.upload(packed)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)  # VbConfig's arena capacities, which only grow
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)


def test_enqueue_and_finish(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    rows = moved(packed, 3)
    r.upload(packed)
    r.bind_transforms(on_device(rows))
    ref.upload(patched(packed, rows))
    p = RenderParams(BASE, W, H, AA_MSAA16)
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.enqueue(p, out.data_ptr())
    r.finish()
    assert (out.cpu().numpy() == frame(ref)[0]).all()


# ---- 4. with other features ------------------------------------------------------------------------------------------------
def test_view_run_stages_and_rerun(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    rows = moved(packed, 5)
    r.upload(packed)
    r.bind_transforms(on_device(rows))
    ref.upload(patched(packed, rows))
    view = Affine.translate(-30, 20) * Affine.scale(1.3) * Affine.rotate(0.08)
    r.set_view(view)
    ref.set_view(view)
    try:
        assert (frame(r)[0] == frame(ref)[0]).all()
        assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
    finally:
        r.set_view(None)
        ref.set_view(None)
    want, _ = frame(ref)
    assert (frame(r)[0] == want).all(), "the binding survives the view"
    # split ranges: flatten's stage reads the rows, and a range that starts at draw reads them again
    p = RenderParams(BASE, W, H, AA_MSAA16)
    t = on_device(rows)
    r.bind_transforms(t)
    r.run_stages(p, "pathtag", "flatten")
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    assert np.array_equal(r.download("transforms", np.uint32), words(patched(packed, rows)))
    # a blocking frame re-run after an arena overflow reads the same rows
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    st = r.render_resident(p)
    assert st.retries == 1
    assert (r.download_target(p) == want).all()


def test_with_bound_instance_transforms(rr):
    """A composed scene's entries are global in instance order; a finite row replaces the instance product of its entry."""
    r, ref = rr
    frags = [colour_mixed(seed=k) for k in range(3)]
    inst = [0, 1, 2, 1]
    ids = [r.upload_fragment(f) for f in frags]
    r.compose([(ids[i], None) for i in inst])
    xf = rand_rows(len(inst), 6, 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    host = Scene()
    for k, i in enumerate(inst):
        host.append(colour_mixed(seed=i), aff(xf[k]))
    composed = resolve(host.encoding)
    n = len(transforms(composed))
    rows = moved(composed, 7)
    rows[1::3] = np.nan  # these keep the instance products
    r.bind_instance_transforms(on_device(xf))
    r.bind_transforms(on_device(rows[:n - 2]))
    want_packed = patched(composed, rows[:n - 2])
    ref.upload(want_packed)
    img, _ = frame(r)
    assert np.array_equal(r.download("transforms", np.uint32), words(want_packed))
    assert (img == frame(ref)[0]).all()
    r.bind_instance_transforms(None)  # the rows stay bound, over the composed scene's own transforms
    plain = Scene()
    for i in inst:
        plain.append(colour_mixed(seed=i))
    ref.upload(patched(resolve(plain.encoding), rows[:n - 2]))
    assert (frame(r)[0] == frame(ref)[0]).all()
    for f in ids:
        r.free_fragment(f)


def test_batch_global_rows(rr):
    r, ref = rr
    cells = [mixed(seed=k) for k in range(3)]
    whole, offs = Scene(), [0]
    for c in cells:
        whole.append(c)
        offs.append(whole.n_draw_objects)
    packed = resolve(whole.encoding)
    rows = moved(packed, 9)
    r.upload(packed)
    r.bind_transforms(on_device(rows))
    r.set_cells(offs)
    ref.upload(patched(packed, rows))
    ref.set_cells(offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


def test_hit_tests_and_maps_follow_the_transforms(rr):
    r, ref = rr
    packed = resolve(mixed().encoding)
    rows = moved(packed, 10, 0.3, 15.0)
    r.upload(packed)
    r.bind_transforms(on_device(rows))
    ref.upload(patched(packed, rows))
    frame(r, AA_AREA)
    frame(ref, AA_AREA)
    pts = np.random.default_rng(10).uniform(0, [W, H], (5000, 2)).astype(np.float32)
    got = r.hit_test(pts)
    assert (got >= 0).sum() > 500 and (got == ref.hit_test(pts)).all()
    assert (r.hit_map() == ref.hit_map()).all()


# ---- 5. damage tracking ----------------------------------------------------------------------------------------------------
def sprites():
    """Neighbouring sprites, each under its own transform: a filled star, a stroked outline and a gradient badge whose brush
    transform is an entry of its own."""
    s = Scene()
    for k in range(6):
        x, y = 40 + 60 * k, 60 + 90 * (k % 2)
        t = Affine.translate(x, y)
        s.fill(FILL_NON_ZERO, t, Color(0.9, 0.2 + 0.1 * k, 0.1, 1.0), None, star(0, 0, 8, 20, 5))
        s.stroke(Stroke(2.0), Affine.translate(x, y + 0.5), Color(0.1, 0.1, 0.1, 1.0), None, star(0, 0, 8, 20, 5))
        s.fill(FILL_NON_ZERO, Affine.translate(x, y + 40), Gradient.linear((-10, 0), (10, 0), STOPS), Affine.rotate(0.1 * k),
               Circle(0, 0, 12))
    return s


def test_damage_follows_the_exact_transform_ranges(rr):
    r, ref = rr
    s = sprites()
    packed = resolve(s.encoding)
    ranges = transform_ranges(packed)
    rows = transforms(packed)
    r.upload(packed)
    t = on_device(rows)
    r.bind_transforms(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)

    def step(new=None):
        nonlocal rows
        if new is not None:
            rows = new.astype(np.float32)
            t.copy_(torch.from_numpy(rows))
            torch.cuda.synchronize()
        r.render_resident(p, dst.data_ptr())
        ref.upload(patched(packed, rows))
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        return r.last_damage()

    try:
        assert step().sum() == n_tiles
        assert step().sum() == 0
        for k in list(range(len(rows))) + [None]:
            before = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            new = rows.copy()
            ks = [k] if k is not None else [0, 4, 9]
            for j in ks:
                new[j, 4:] += np.float32([7.0, -5.0])
                new[j, :4] = new[j, :4] * np.float32(0.9)
            got = step(new)
            after = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            paths = [d for d, (lo, hi) in enumerate(ranges) if any(lo <= j <= hi for j in ks)]
            assert paths, ks
            want = box_tiles(before[paths], W, H) | box_tiles(after[paths], W, H)
            assert (got == want).all(), (ks, paths)
        # the same words through non-finite rows: no change
        rows = rows.copy()
        rows[3, 2] = np.nan
        t = on_device(rows)
        r.bind_transforms(t)  # a new binding: full
        assert step().sum() == n_tiles
        assert step().sum() == 0
        fin = rows.copy()
        fin[3] = transforms(packed)[3]
        assert step(fin).sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_transforms(None)


def test_diff_after_a_bound_base_is_full(rr):
    r, ref = rr
    packed = resolve(sprites().encoding)
    r.upload(packed)
    r.bind_transforms(on_device(moved(packed, 12)))
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        r.render_resident(p, dst.data_ptr())
        r.set_upload_diff(True)
        r.upload(packed)  # diffed against a bound base: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        ref.upload(packed)
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload(packed)  # an unbound base: the same upload damages nothing
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == 0
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 6. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_transforms(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding_and_installations_unbind(rr):
    r, ref = rr
    s = mixed()
    packed = resolve(s.encoding)
    n = s.n_transforms
    r.upload(packed)
    t = on_device(moved(packed, 13))
    r.bind_transforms(t)
    before, _ = frame(r)

    def unchanged(what):
        assert r.lib.vb_last_error(r.handle), what
        assert (frame(r)[0] == before).all(), what

    ptr = t.data_ptr()
    host = np.zeros((n, 6), dtype=np.float32)
    for args in ((ptr, 0, 24), (ptr, n + 1, 24), (host.ctypes.data, n, 24), (ptr + 2, n, 24), (ptr, n, 20), (ptr, n, 26),
                 (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        unchanged(args)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    assert _bind_raw(r, ptr, n, 24) == VB_E_INVALID  # between enqueue and finish
    r.finish()
    assert (r.download_target(p) == before).all()
    x = Renderer()
    try:
        assert _bind_raw(x, ptr, 1, 24) == VB_E_INVALID and b"scene" in x.lib.vb_last_error(x.handle)
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        assert _bind_raw(x, ptr, n, 24) == VB_E_INVALID and b"exchange" in x.lib.vb_last_error(x.handle)
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        assert _bind_raw(g.renderer(0), ptr, 1, 24) == VB_E_INVALID
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
    fid = r.upload_fragment(s)
    installs = [(lambda: r.upload(packed), encoded), (lambda: r.upload_scene(s), encoded), (lambda: r.render_to_texture(packed, p), encoded),
                (lambda: list(r.render_stream([packed], p)), encoded), (lambda: r.recompose([(fid, None)]), encoded),
                (lambda: r.compose([(fid, None)]), encoded), (lambda: native.upload_device(r), native_frame)]
    for install, want in installs:
        r.compose([(fid, None)])
        r.bind_transforms(t)
        assert not (frame(r)[0] == encoded).all()
        install()
        assert (frame(r)[0] == want).all()
    r.free_fragment(fid)
    r.upload(packed)
    r.bind_transforms(t)
    r.bind_transforms(None)
    assert (frame(r)[0] == encoded).all()
