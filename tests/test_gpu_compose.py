"""Composition of resident fragments (Renderer.upload_fragment / compose, vb_fragment_upload / vb_compose): the renderer's
scene becomes `Scene()` with every fragment appended under its transform, built on the device. The reference of every case
is that appended scene resolved on the host (NativeScene.append + resolve, or Scene.append + encoding.resolve) and uploaded
from there. Run on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_SRC_OVER, Color, EXTEND_REFLECT, EXTEND_REPEAT, FILL_EVEN_ODD, FILL_NON_ZERO, FORMAT_BGRA8,
                                 Gradient, Image, MIX_MULTIPLY, Scene, Stroke, resolve, viewed)
from vello_b200.renderer import Renderer, RendererGroup, VelloB200Error, _Params, FrameStats
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Circle, Rect, RoundedRect

from .test_gpu_parity import assert_pixels

pytestmark = pytest.mark.gpu

BASE = Color.from_rgba8(12, 20, 30)
STOPS_A = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (0.6, Color(0.1, 0.8, 0.3, 0.5)), (1.0, Color(0.2, 0.3, 1.0, 1.0))]
STOPS_B = [(0.0, Color(0.9, 0.9, 0.1, 0.2)), (1.0, Color(0.1, 0.1, 0.9, 1.0))]
RNG = np.random.default_rng(7)
IMG = RNG.integers(0, 256, (20, 24, 4), dtype=np.uint8)
IMG_BGRA = RNG.integers(0, 256, (9, 13, 4), dtype=np.uint8)
TRANSFORMS = [None, Affine.IDENTITY, Affine.translate(40.5, 17.25) * Affine.rotate(0.7), Affine((-1.0, 0.0, 0.0, 1.0, 300.0, 10.0)),
              Affine((1.0, 0.3, -0.45, 1.0, 60.0, 80.0)), Affine.scale(1.7, 0.6)]


@pytest.fixture(scope="module")
def rr():
    """`r` composes; `ref` renders the host-resolved references."""
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


# ---- fragments -----------------------------------------------------------------------------------------------------------
def _frag_solid(k):
    s = NativeScene()
    for i in range(k + 1):  # a different number of paths, and so of tag bytes, per k
        s.fill(FILL_NON_ZERO, Affine.translate(10 * i, 5 * i), Color.from_rgba8(40 * i % 256, 200, 90, 230), None, Rect(0, 0, 30, 20))
    s.stroke(Stroke(3.0), Affine.IDENTITY, Color(0.9, 0.1, 0.4, 1.0), None, Circle(50, 40, 18 + k))
    return s


def _frag_gradients(stops):
    s = NativeScene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (100, 0), stops), None, Rect(0, 0, 100, 60))
    s.fill(FILL_EVEN_ODD, Affine.translate(20, 70), Gradient.radial((30, 30), 5, (35, 30), 40, STOPS_B, EXTEND_REFLECT, False), None,
           Circle(30, 30, 30))
    s.fill(FILL_NON_ZERO, Affine.translate(120, 0), Gradient.sweep((40, 40), 0.3, 5.0, stops, EXTEND_REPEAT), Affine.rotate(0.2),
           RoundedRect(0, 0, 80, 80, 12))
    return s


def _frag_images(img, bgra):
    s = NativeScene()
    s.draw_image(img, Affine.translate(4, 6))
    s.fill(FILL_NON_ZERO, Affine.translate(40, 0), img, Affine.scale(2.0), Rect(0, 0, 48, 40))
    if bgra is not None:
        s.draw_image(bgra, Affine.translate(0, 50) * Affine.scale(3.0))
    return s


def _frag_layers(open_clips):
    s = NativeScene()
    s.stroke(Stroke(4.0, dash_pattern=(9.0, 5.0), dash_offset=2.0), Affine.IDENTITY, Color(0.2, 0.6, 0.9, 1.0), None, Circle(60, 60, 40))
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Circle(60, 60, 45))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.5, 0.1, 1.0), None, Rect(10, 10, 110, 110))
    s.pop_layer()
    s.push_luminance_mask_layer(FILL_NON_ZERO, 0.9, Affine.translate(20, 20), Rect(0, 0, 60, 60))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (100, 100), STOPS_B), None, Rect(0, 0, 100, 100))
    s.pop_layer()
    for i in range(open_clips):  # left open: resolve closes them at the end of the whole scene
        s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Rect(5 * i, 5 * i, 150, 150))
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.3, 0.3, 0.8, 0.6), None, Circle(70, 70, 30 + 10 * i))
    return s


def mixed_fragments():
    # keyed images: every fragment that draws one refers to the same pixels, so the fragments share its atlas slot
    img = Image(IMG, key=IMG.ctypes.data)
    bgra = Image(IMG_BGRA, format=FORMAT_BGRA8, key=IMG_BGRA.ctypes.data)
    return [_frag_solid(0), _frag_solid(1), _frag_solid(2), _frag_solid(3),  # tag byte counts at several residues mod 4
            _frag_gradients(STOPS_A), _frag_gradients(STOPS_A),              # the same stops in two fragments
            _frag_images(img, bgra), _frag_images(img, None), _frag_images(img, bgra),  # one image key in three fragments
            _frag_layers(0), _frag_layers(2), NativeScene()]                 # layers, masks, dashes, open clips, empty


def host_packed(frags, instances):
    """The appended scene resolved on the host, and its draw offsets."""
    s = NativeScene()
    offs = [0]
    for fi, t in instances:
        s.append(frags[fi], t)
        offs.append(s.n_draw_objects)
    return s.resolve(), offs


def device_packed(r):
    return r.download("scene", np.uint32), r.download("ramps", np.uint32), r.download("atlas", np.uint8)


def assert_same_bytes(r, lay, offs, packed, ref_offs):
    scene, ramps, atlas = device_packed(r)
    assert (lay.as_array() == packed.layout.as_array()).all(), f"layout {lay} != {packed.layout}"
    assert offs == ref_offs
    assert scene.size == packed.scene.size and (scene == packed.scene).all(), \
        f"scene words differ at {np.nonzero(scene != packed.scene)[0][:8] if scene.size == packed.scene.size else 'size'}"
    assert (ramps == packed.ramps.reshape(-1)).all()
    assert atlas.size == packed.atlas.size and (atlas == packed.atlas.reshape(-1)).all()


def frame(r, w, h, aa):
    p = RenderParams(BASE, w, h, aa)
    r.render_resident(p)
    return r.download_target(p)


def ref_frame(ref, packed, w, h, aa):
    ref.upload(packed)
    return frame(ref, w, h, aa)


def upload_all(r, frags):
    return [r.upload_fragment(f) for f in frags]


def mixed_instances(n_frags):
    inst = []
    for i in range(n_frags):
        inst.append((i, TRANSFORMS[i % len(TRANSFORMS)]))
    inst += [(0, Affine.translate(7 * k, 3 * k)) for k in range(40)]  # one fragment instanced many times
    inst += [(n_frags - 1, None), (4, Affine.rotate(-0.3)), (7, None), (10, Affine.translate(200, 200))]
    return inst


# ---- 1. byte identity ----------------------------------------------------------------------------------------------------
def test_byte_identity_mixed(rr):
    r, _ = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    inst = mixed_instances(len(frags))
    tag_bytes = [(pk.scene[:pk.layout.path_data_base].view(np.uint8) != 0).sum() for pk in (f.resolve() for f in frags)]
    assert {int(n) % 4 for n in tag_bytes} == {0, 1, 2, 3}, "tag streams ending at every byte of a word"
    lay, offs = r.compose([(ids[i], t) for i, t in inst])
    packed, ref_offs = host_packed(frags, inst)
    assert_same_bytes(r, lay, offs, packed, ref_offs)
    assert packed.ramps.shape[0] == 3, "STOPS_A (shared by two fragments), and STOPS_B in both interpolation spaces"
    assert packed.atlas.shape == (20, 24 + 13, 4), "one slot for IMG (three fragments) and one for IMG_BGRA (two)"
    for i in ids:
        r.free_fragment(i)


def test_byte_identity_large_among_tiny(rr):
    """One paris-like fragment of 2,500 paths among 1,000 tiny ones (Python `Scene`s, resolved by encoding.resolve): the
    big one spans many windows and CTAs, the tiny ones share CTAs and tag words."""
    r, _ = rr
    big = scenes.paris_like(2500, 1024, seed=3)
    tiny = []
    for k in range(1000):
        s = Scene()
        for j in range(1 + k % 3):
            s.fill(FILL_NON_ZERO, Affine.translate(k % 40 * 20 + j, k // 40 * 20), Color.from_rgba8(k % 256, 99, j * 80, 255), None,
                   Rect(0, 0, 9 + j, 7))
        tiny.append(s)
    frags = tiny[:500] + [big] + tiny[500:]
    ids = upload_all(r, frags)
    inst = [(i, None if i % 3 == 0 else Affine.translate(i % 17, 0.5 * (i % 5))) for i in range(len(frags))]
    lay, offs = r.compose([(ids[i], t) for i, t in inst])
    app = Scene()
    ref_offs = [0]
    for i, t in inst:
        app.append(frags[i], t)
        ref_offs.append(app.n_draw_objects)
    assert_same_bytes(r, lay, offs, resolve(app.encoding), ref_offs)
    for i in ids:
        r.free_fragment(i)


# ---- 2. pixels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_pixels_equal_host_upload(rr, aa):
    r, ref = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    inst = mixed_instances(len(frags))
    r.compose([(ids[i], t) for i, t in inst])
    img = frame(r, 512, 384, aa)
    packed, _ = host_packed(frags, inst)
    want = ref_frame(ref, packed, 512, 384, aa)
    if aa == AA_AREA:
        assert_pixels(img, want, aa)
    else:
        assert (img == want).all()
    for i in ids:
        r.free_fragment(i)


@pytest.mark.parametrize("aa", [AA_MSAA16, AA_AREA])
def test_tile_grid_against_oracle(rr, oracle, aa):
    r, _ = rr
    tiles = [scenes.paris_like(60, 128, seed=k) for k in range(64)]
    ids = upload_all(r, tiles)
    inst = [(k, Affine.translate(128 * (k % 8), 128 * (k // 8))) for k in range(64)]
    r.compose([(ids[k], t) for k, t in inst])
    img = frame(r, 1024, 1024, aa)
    app = Scene()
    for k, t in inst:
        app.append(tiles[k], t)
    ref = oracle.render(resolve(app.encoding), 1024, 1024, BASE.premul_rgba8_u32(), aa)
    assert_pixels(img, ref, aa)
    for i in ids:
        r.free_fragment(i)


# ---- 3. recomposition ----------------------------------------------------------------------------------------------------
def test_recompose_sequence_and_graph_replay(rr):
    r, ref = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    seqs = [
        [(0, None), (4, Affine.translate(10, 10)), (6, None)],
        [(0, None), (4, Affine.translate(12, 9)), (6, Affine.rotate(0.1))],   # transforms only
        [(0, None), (4, Affine.translate(30, 2)), (6, Affine.rotate(0.2))],   # transforms only
        [(6, None), (0, None), (4, Affine.translate(30, 2))],                 # reordered
        [(6, None), (0, None), (4, Affine.translate(30, 2)), (10, None)],     # added
        [(10, Affine.scale(0.5)), (5, None)],                                 # removed
    ]
    caps = []
    for inst in seqs:
        r.compose([(ids[i], t) for i, t in inst])
        img = frame(r, 256, 256, AA_MSAA16)
        caps.append(r.debug_graph_captures())
        packed, _ = host_packed(frags, inst)
        assert (img == ref_frame(ref, packed, 256, 256, AA_MSAA16)).all()
    assert caps[1] == caps[0] and caps[2] == caps[0], f"only transforms changed, yet graphs were captured again: {caps}"
    assert caps[3] > caps[2] or caps[4] > caps[2], f"the layout changed and no graph was captured: {caps}"
    assert caps[4] > caps[3] and caps[5] > caps[4], caps
    for i in ids:
        r.free_fragment(i)


def test_compose_enqueue_finish_without_sync(rr):
    r, ref = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    p = RenderParams(BASE, 256, 256, AA_MSAA16)
    imgs, refs = [], []
    for k in range(6):
        inst = [(0, Affine.translate(5 * k, 3 * k)), (4, Affine.rotate(0.05 * k)), (6, None if k % 2 else Affine.translate(k, k))]
        r.compose([(ids[i], t) for i, t in inst])
        r.enqueue(p)
        r.finish()
        imgs.append(r.download_target(p))
        packed, _ = host_packed(frags, inst)
        refs.append(ref_frame(ref, packed, 256, 256, AA_MSAA16))
    for k, (a, b) in enumerate(zip(imgs, refs)):
        assert (a == b).all(), f"frame {k}"
    for i in ids:
        r.free_fragment(i)


# ---- 4. with views, hit testing, cells and device images -----------------------------------------------------------------
def test_view_on_top(rr):
    r, ref = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    inst = mixed_instances(len(frags))
    view = Affine.translate(-30, 12) * Affine.scale(1.3)
    r.set_view(view)
    try:
        r.compose([(ids[i], t) for i, t in inst])
        img = frame(r, 512, 384, AA_MSAA16)
    finally:
        r.set_view(None)
    packed, _ = host_packed(frags, inst)
    assert (img == ref_frame(ref, viewed(packed, view), 512, 384, AA_MSAA16)).all()
    for i in ids:
        r.free_fragment(i)


def test_hit_test_maps_to_instances(rr):
    r, ref = rr
    cell = NativeScene()
    cell.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.5, 0.5, 0.5, 1.0), None, Rect(0, 0, 40, 40))
    cell.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.1, 0.1, 1.0), None, Circle(20, 20, 10))
    fid = r.upload_fragment(cell)
    inst = [(0, Affine.translate(50 * (k % 6), 50 * (k // 6))) for k in range(24)]
    lay, offs = r.compose([(fid, t) for _, t in inst])
    frame(r, 300, 200, AA_AREA)
    pts = np.array([[50 * (k % 6) + 20.5, 50 * (k // 6) + 20.5] for k in range(24)] +
                   [[50 * (k % 6) + 3.5, 50 * (k // 6) + 3.5] for k in range(24)], dtype=np.float32)
    got = r.hit_test(pts)
    for k in range(24):
        assert offs[k] <= got[k] < offs[k + 1] and got[k] == offs[k] + 1, (k, got[k], offs[k:k + 2])
        assert got[24 + k] == offs[k], (k, got[24 + k])
    rand = np.random.default_rng(3).uniform(0, [300, 200], (4000, 2)).astype(np.float32)
    packed, _ = host_packed([cell], inst)
    ref.upload(packed)
    frame(ref, 300, 200, AA_AREA)
    assert (r.hit_test(rand) == ref.hit_test(rand)).all()
    r.free_fragment(fid)


def _render_cells(r, n, w, h, aa):
    out = np.zeros((n, h, w, 4), dtype=np.uint8)
    st = FrameStats()
    ps = _Params(BASE.premul_rgba8_u32(), w, h, aa, 0, 0, 0, 0)
    r._check(r.lib.vb_render_uploaded(r.handle, C.byref(ps), C.c_void_p(out.ctypes.data), 0, C.byref(st)), "vb_render_uploaded")
    return out


def test_set_cells_on_draw_offsets(rr):
    r, ref = rr
    frags = [_frag_solid(1), _frag_gradients(STOPS_A), _frag_images(Image(IMG), None), _frag_layers(0)]
    ids = upload_all(r, frags)
    inst = [(k, Affine.translate(10 + 3 * k, 5) * Affine.rotate(0.05 * k)) for k in range(4)]
    _, offs = r.compose([(ids[i], t) for i, t in inst])
    r.set_cells(offs)
    cells = _render_cells(r, 4, 200, 160, AA_MSAA16)
    for k, (i, t) in enumerate(inst):
        packed, _ = host_packed(frags, [(i, t)])
        assert (cells[k] == ref_frame(ref, packed, 200, 160, AA_MSAA16)).all(), f"cell {k}"
    for i in ids:
        r.free_fragment(i)


def test_override_refreshes_when_dirty(rr):
    torch = pytest.importorskip("torch")
    r, _ = rr
    t = torch.randint(0, 256, (16, 24, 4), dtype=torch.uint8, device="cuda")
    tex = r.register_texture(t)
    try:
        s = NativeScene()
        s.draw_image(tex, Affine.translate(10, 10))
        s.draw_image(Image(IMG), Affine.translate(60, 10))
        fid = r.upload_fragment(s)
        r.compose([(fid, None), (fid, Affine.translate(0, 50))])
        frame(r, 128, 128, AA_MSAA16)
        atlas = r.download("atlas", np.uint8)
        aw = atlas.size // 4 // 20
        a = atlas.reshape(-1, aw, 4)
        assert (a[:16, :24] == t.cpu().numpy()).all() and (a[:20, 24:48] == IMG).all()
        t.copy_(torch.randint(0, 256, (16, 24, 4), dtype=torch.uint8, device="cuda"))
        torch.cuda.synchronize()
        r.mark_override_image_dirty(tex)
        frame(r, 128, 128, AA_MSAA16)
        a = r.download("atlas", np.uint8).reshape(-1, aw, 4)
        assert (a[:16, :24] == t.cpu().numpy()).all(), "the dirty texture was not copied again"
        r.free_fragment(fid)
        s2 = NativeScene()
        s2.draw_image(tex, Affine.IDENTITY)
        fid2 = r.upload_fragment(s2)
        r.unregister_texture(tex)
        with pytest.raises(VelloB200Error):  # a registered texture without an override
            r.compose([(fid2, None)])
        r.free_fragment(fid2)
    finally:
        if tex.key in r._device_images:
            r.unregister_texture(tex)


# ---- 5. lifetime and errors ----------------------------------------------------------------------------------------------
def test_free_after_compose_keeps_the_frame(rr):
    r, _ = rr
    frags = mixed_fragments()
    ids = upload_all(r, frags)
    r.compose([(ids[i], t) for i, t in mixed_instances(len(frags))])
    before = frame(r, 384, 256, AA_MSAA16)
    for i in ids:
        r.free_fragment(i)
    assert (frame(r, 384, 256, AA_MSAA16) == before).all()
    with pytest.raises(VelloB200Error):
        r.free_fragment(ids[0])


def test_errors_leave_the_scene(rr):
    r, _ = rr
    frags = mixed_fragments()[:6]
    ids = upload_all(r, frags)
    good = [(ids[i], TRANSFORMS[i]) for i in range(6)]
    r.compose(good)
    before = frame(r, 256, 256, AA_MSAA16)
    gone = r.upload_fragment(frags[0])
    r.free_fragment(gone)
    bad = [
        [(ids[0], None), (987654, None)],                                       # unknown id
        [(gone, None)],                                                         # freed id
        [(ids[0], Affine((1e39, 0.0, 0.0, 1.0, 0.0, 0.0)))],                    # not finite in f32
        [(ids[0], Affine((1.0, 0.0, 0.0, 1.0, float("nan"), 0.0)))],
    ]
    for inst in bad:
        with pytest.raises(VelloB200Error, match="invalid"):
            r.compose(inst)
        assert (frame(r, 256, 256, AA_MSAA16) == before).all()
    assert r.lib.vb_compose(r.handle, None, 3, None, None) == -1  # NULL instances
    p = RenderParams(BASE, 256, 256, AA_MSAA16)
    r.enqueue(p)
    with pytest.raises(VelloB200Error, match="invalid"):  # between enqueue and finish
        r.compose(good)
    r.finish()
    assert (r.download_target(p) == before).all()
    g = RendererGroup([0, 0])
    try:
        gr = g.renderer(0)
        with pytest.raises(VelloB200Error, match="invalid"):  # a renderer of a vb_group
            gr.compose([])
    finally:
        g.close()
    for i in ids:
        r.free_fragment(i)


def test_empty_compose_shows_the_base_colour(rr):
    r, _ = rr
    lay, offs = r.compose([])
    assert offs == [0] and lay.n_draw_objects == 0
    img = frame(r, 64, 48, AA_AREA)
    want = np.array([round(c * 255) for c in (BASE.r, BASE.g, BASE.b, BASE.a)], dtype=np.int32)
    assert (np.abs(img.astype(np.int32) - want) <= 1).all()


def test_growing_scene_under_a_view(rr):
    r, ref = rr
    small = _frag_solid(0)
    big = scenes.paris_like(3000, 512, seed=9)
    fs, fb = r.upload_fragment(small), r.upload_fragment(big)
    view = Affine.translate(8, -6) * Affine.rotate(0.03)
    r.set_view(view)
    try:
        r.compose([(fs, None)])
        frame(r, 512, 512, AA_MSAA16)
        inst = [(fs, None), (fb, Affine.scale(0.9)), (fs, Affine.translate(100, 100))]
        r.compose(inst)
        img = frame(r, 512, 512, AA_MSAA16)
    finally:
        r.set_view(None)
    # the host reference: the same three instances appended in Python (the small fragment encoded again as a Python Scene)
    py_small = Scene()
    py_small.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(0, 200, 90, 230), None, Rect(0, 0, 30, 20))
    py_small.stroke(Stroke(3.0), Affine.IDENTITY, Color(0.9, 0.1, 0.4, 1.0), None, Circle(50, 40, 18))
    want_scene = Scene()
    for src, t in [(py_small, None), (big, Affine.scale(0.9)), (py_small, Affine.translate(100, 100))]:
        want_scene.append(src, t)
    packed = resolve(want_scene.encoding)
    assert (img == ref_frame(ref, viewed(packed, view), 512, 512, AA_MSAA16)).all()
    r.free_fragment(fs)
    r.free_fragment(fb)


# ---- image keys whose memory the caller reused, and overrides that come and go ---------------------------------------------
def test_reused_pixel_memory_keeps_images_apart(rr):
    """The caller's pixels are not needed after upload_fragment, so one buffer may hold another image in the next fragment;
    each fragment must still draw its own pixels. The reference keeps every scene and its pixels alive."""
    r, _ = rr
    icons = [np.random.default_rng(100 + k).integers(0, 256, (8, 8, 4), dtype=np.uint8) for k in range(12)]
    buf = np.zeros((8, 8, 4), dtype=np.uint8)
    ids = []
    for k in range(6):  # one buffer, refilled for every fragment: the same key pointer with other pixels each time
        buf[:] = icons[k]
        s = NativeScene()
        s.draw_image(Image(buf, key=buf.ctypes.data), Affine.translate(12 * k, 0))
        ids.append(r.upload_fragment(s))
    for k in range(6, 12):  # key-less images of scenes dropped right after their upload (their pixel copies die with them)
        s = NativeScene()
        s.draw_image(Image(icons[k].copy()), Affine.translate(12 * k, 0))
        ids.append(r.upload_fragment(s))
        del s
    kept = []
    for k in range(12):
        s = NativeScene()
        s.draw_image(Image(icons[k]), Affine.translate(12 * k, 0))
        kept.append(s)
    inst = [(k, Affine.translate(0, 3 * k)) for k in range(12)] + [(3, None), (9, None)]
    lay, offs = r.compose([(ids[i], t) for i, t in inst])
    packed, ref_offs = host_packed(kept, inst)
    assert packed.atlas.shape == (8, 12 * 8, 4)
    assert_same_bytes(r, lay, offs, packed, ref_offs)
    for i in ids:
        r.free_fragment(i)


def test_removed_override_gives_the_fragment_pixels_back(rr):
    torch = pytest.importorskip("torch")
    r, _ = rr
    img = Image(IMG, key=IMG.ctypes.data)
    s = NativeScene()
    s.draw_image(img, Affine.translate(5, 5))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.7, 0.3, 1.0), None, Rect(40, 0, 60, 20))
    fid = r.upload_fragment(s)
    inst = [(0, None), (0, Affine.translate(30, 30))]
    t = torch.randint(0, 256, IMG.shape, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r.override_image(img, t)
    try:
        r.compose([(fid, tr) for _, tr in inst])
        frame(r, 128, 128, AA_MSAA16)
        a = r.download("atlas", np.uint8).reshape(IMG.shape)
        assert (a == t.cpu().numpy()).all(), "the override fills the slot"
    finally:
        r.override_image(img, None)
    lay, offs = r.compose([(fid, tr) for _, tr in inst])  # the same instances, no override any more
    packed, ref_offs = host_packed([s], inst)
    assert_same_bytes(r, lay, offs, packed, ref_offs)
    r.free_fragment(fid)


def test_free_while_a_compose_is_enqueued(rr):
    """vb_fragment_free returns without waiting; the memory outlives the work already enqueued that reads it."""
    r, ref = rr
    frags = mixed_fragments()
    inst = mixed_instances(len(frags))
    p = RenderParams(BASE, 384, 256, AA_MSAA16)
    packed, _ = host_packed(frags, inst)
    want = ref_frame(ref, packed, 384, 256, AA_MSAA16)
    for _ in range(3):
        ids = upload_all(r, frags)
        r.compose([(ids[i], t) for i, t in inst])
        for i in ids:
            r.free_fragment(i)  # the compose above may not have run yet
        r.enqueue(p)
        r.finish()
        assert (r.download_target(p) == want).all()
