"""Images drawn from device memory (Renderer.register_texture / override_image / mark_override_image_dirty, vello/src/lib.rs:
536-603): the device resolve copies overridden images into the atlas with k_atlas_blit (k_atlas.cu), and a dirty image is copied
again in front of the next frame. Sources are torch CUDA tensors. Frames are compared byte for byte with the same scene drawn
from host pixels."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (ALPHA_PREMULTIPLIED, ALPHA_STRAIGHT, BLACK, Color, EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT,
                                 FILL_NON_ZERO, FORMAT_BGRA8, FORMAT_RGBA8, Image, QUALITY_HIGH, QUALITY_LOW, QUALITY_MEDIUM,
                                 Scene, resolve)
from vello_b200.shapes import Affine, Circle, Rect

from .test_gpu_parity import assert_pixels

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 256, 256
BASE = Color.from_rgba8(20, 30, 40)


@pytest.fixture(scope="module")
def renderers():
    """Two renderers: `r` draws from device memory, `ref` renders the host-pixel references (so that uploading a reference
    never touches r's scene)."""
    from vello_b200.renderer import Renderer
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def native(draw):
    from vello_b200.scene_native import NativeScene
    s = NativeScene()
    draw(s)
    return s


def frame(r, scene, p, out_ptr=0):
    """Resolve `scene` on r's device, render it resident and read the frame back."""
    scene.upload_device(r)
    return render(r, p, out_ptr)


def render(r, p, out_ptr=0):
    r.render_resident(p, out_ptr)
    return r.download_target(p, device_ptr=out_ptr)


def to_dev(a: np.ndarray, pad_cols: int = 0, col0: int = 0):
    """`a` as a CUDA tensor; with pad_cols, a column slice [col0, col0 + w) of a wider tensor (pitch != 4 * w)."""
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if not pad_cols:
        return t
    h, w, _ = a.shape
    big = torch.randint(0, 256, (h, w + pad_cols, 4), dtype=torch.uint8, device="cuda")
    big[:, col0:col0 + w] = t
    return big[:, col0:col0 + w]


def sampler_sweep(im: Image):
    """Every quality x extend mode, each filling a rectangle larger than the (rotated, scaled) image, plus one draw_image."""
    def draw(s):
        k = 0
        for q in (QUALITY_LOW, QUALITY_MEDIUM, QUALITY_HIGH):
            for e in (EXTEND_PAD, EXTEND_REPEAT, EXTEND_REFLECT):
                v = dataclasses.replace(im, quality=q, x_extend=e, y_extend=(e + k) % 3)
                x, y = 8 + 80 * (k % 3), 8 + 80 * (k // 3)
                s.fill(FILL_NON_ZERO, Affine.translate(x, y), v, Affine.translate(30, 10) * Affine.rotate(0.35) * Affine.scale(1.7, 1.3),
                       Rect(0, 0, 72, 72))
                k += 1
        s.draw_image(dataclasses.replace(im, quality=QUALITY_HIGH), Affine.translate(150, 120) * Affine.rotate(-0.5) * Affine.scale(2.3))
    return draw


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_device_image_equals_host_image(renderers, oracle, aa):
    r, ref = renderers
    rng = np.random.default_rng(11 + aa)
    data = rng.integers(0, 256, (21, 26, 4), dtype=np.uint8)
    p = RenderParams(BASE, W, H, aa)
    for fmt in (FORMAT_RGBA8, FORMAT_BGRA8):
        for at in (ALPHA_STRAIGHT, ALPHA_PREMULTIPLIED):
            host_im = Image(data, format=fmt, alpha_type=at)
            host_scene = native(sampler_sweep(host_im))
            want = frame(ref, host_scene, p)
            packed = host_scene.resolve()
            assert_pixels(want, oracle.render(packed, W, H, BASE.premul_rgba8_u32(), aa), aa)
            for pad in (0, 7):
                t = to_dev(data, pad_cols=pad, col0=3)
                tex = r.register_texture(t)
                got = frame(r, native(sampler_sweep(dataclasses.replace(tex, format=fmt, alpha_type=at))), p)
                assert np.array_equal(got, want), (fmt, at, pad)
                r.unregister_texture(tex)


def test_many_rectangles_one_launch(renderers):
    """~300 images of 1x1 .. 64x64 (odd widths, 4-byte aligned column slices) and one 2048x2048: the device atlas equals the
    host resolve's, and all of them are copied by one k_atlas_blit."""
    r, _ = renderers
    rng = np.random.default_rng(5)
    arrays = [rng.integers(0, 256, (int(rng.integers(1, 65)), int(rng.integers(1, 65)), 4), dtype=np.uint8) for _ in range(300)]
    arrays[:4] = [rng.integers(0, 256, s + (4,), dtype=np.uint8) for s in ((1, 1), (64, 64), (3, 63), (17, 1))]
    arrays.insert(150, rng.integers(0, 256, (2048, 2048, 4), dtype=np.uint8))
    tensors = [to_dev(a, pad_cols=5, col0=int(rng.integers(0, 6))) if i % 2 else to_dev(a) for i, a in enumerate(arrays)]
    texes = [r.register_texture(t) for t in tensors]

    def draw(images):
        def f(s):
            for i, im in enumerate(images):
                s.draw_image(im, Affine.translate(float(i % 20) * 12, float(i // 20) * 12) * Affine.scale(0.1))
        return f

    host = native(draw([Image(a) for a in arrays])).resolve()
    dev_scene = native(draw(texes))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev_scene.upload_device(r)
        torch.cuda.synchronize()
    blits = [e for e in prof.events() if "k_atlas_blit" in e.name]
    assert len(blits) == 1, [e.name for e in blits]
    atlas = r.download("atlas", np.uint8)
    assert atlas.tobytes() == host.atlas.tobytes()
    for tex in texes:
        r.unregister_texture(tex)


@pytest.mark.parametrize("graph", [True, False])
def test_dirty_protocol(renderers, graph):
    """Uploaded once and rendered resident: pixels A. The tensor changes: still A until the image is marked dirty (vello's
    documented behaviour), then B. The copy is not a frame launch: kernel_launches does not change."""
    r, ref = renderers
    r.set_cuda_graph(graph)
    rng = np.random.default_rng(3)
    a = rng.integers(0, 256, (40, 33, 4), dtype=np.uint8)
    b = rng.integers(0, 256, (40, 33, 4), dtype=np.uint8)
    p = RenderParams(BASE, W, H, AA_MSAA16)

    def draw(im):
        return lambda s: (s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 40, 90), None, Circle(128, 128, 90)),
                          s.draw_image(im, Affine.translate(40, 30) * Affine.rotate(0.2) * Affine.scale(4.0)))

    want_a, want_b = frame(ref, native(draw(Image(a))), p), frame(ref, native(draw(Image(b))), p)
    assert not np.array_equal(want_a, want_b)
    t = to_dev(a, pad_cols=3, col0=1)
    tex = r.register_texture(t)
    native(draw(tex)).upload_device(r)
    launches = []
    got = render(r, p)
    launches.append(int(r.last_stats.kernel_launches))
    assert np.array_equal(got, want_a)
    t.copy_(torch.from_numpy(b).cuda())
    torch.cuda.synchronize()
    got = render(r, p)
    launches.append(int(r.last_stats.kernel_launches))
    assert np.array_equal(got, want_a), "an override that is not marked dirty keeps the pixels copied last"
    r.mark_override_image_dirty(tex)
    got = render(r, p)
    launches.append(int(r.last_stats.kernel_launches))
    assert np.array_equal(got, want_b)
    got = render(r, p)  # clean again: the same pixels
    assert np.array_equal(got, want_b)
    assert len(set(launches)) == 1, launches
    r.unregister_texture(tex)
    r.set_cuda_graph(True)


def test_override_host_image_then_remove(renderers):
    r, ref = renderers
    rng = np.random.default_rng(4)
    h_px = rng.integers(0, 256, (30, 30, 4), dtype=np.uint8)
    d_px = rng.integers(0, 256, (30, 30, 4), dtype=np.uint8)
    p = RenderParams(BASE, W, H, AA_AREA)

    def draw(im):
        return lambda s: s.draw_image(im, Affine.translate(20, 20) * Affine.scale(6.5))

    want_h, want_d = frame(ref, native(draw(Image(h_px))), p), frame(ref, native(draw(Image(d_px))), p)
    img = Image(h_px)
    t = to_dev(d_px)
    r.override_image(img, t)
    assert img.key is not None
    scene = native(draw(img))
    assert np.array_equal(frame(r, scene, p), want_d)
    # the host resolve of the same scene reads the host pixels
    assert np.array_equal(scene.resolve().atlas, resolve(_py_scene(draw(img)).encoding).atlas)
    r.override_image(img, None)
    assert np.array_equal(render(r, p), want_d), "removing an override takes effect at the next device resolve"
    assert np.array_equal(frame(r, scene, p), want_h)


def _py_scene(draw):
    s = Scene()
    draw(s)
    return s


def test_frame_draws_its_own_destination(renderers):
    """Scene 2 draws the device buffer X (frame 1) scaled and is rendered into X itself: the copy into the atlas precedes the
    frame's kernels, so it reads frame 1. Marked dirty and rendered again, it reads frame 2 (the refresh path)."""
    r, ref = renderers
    p = RenderParams(BASE, W, H, AA_MSAA16)
    x = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")

    def scene1(s):
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(250, 200, 10), None, Circle(100, 130, 80))
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(10, 90, 250, 180), None, Rect(120, 20, 240, 200))

    def scene2(im):
        def f(s):
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(60, 220, 120), None, Rect(0, 0, 256, 40))
            s.draw_image(im, Affine.translate(30, 50) * Affine.rotate(0.1) * Affine.scale(0.6))
        return f

    frame(r, native(scene1), p, x.data_ptr())
    f1 = x.cpu().numpy().copy()
    tex = r.register_texture(x)
    f2 = frame(r, native(scene2(tex)), p, x.data_ptr())
    assert np.array_equal(f2, frame(ref, native(scene2(Image(f1))), p))
    assert np.array_equal(x.cpu().numpy(), f2)
    r.mark_override_image_dirty(tex)
    f3 = render(r, p, x.data_ptr())
    assert np.array_equal(f3, frame(ref, native(scene2(Image(f2))), p))
    r.unregister_texture(tex)


def test_errors(renderers):
    """Each misuse is VB_E_INVALID with a message, and leaves the renderer working."""
    from vello_b200.renderer import Renderer, VelloB200Error
    r, ref = renderers
    lib = r.lib
    VB_E_INVALID = -1
    t = torch.zeros((8, 8, 4), dtype=torch.uint8, device="cuda")
    host = np.zeros((8, 8, 4), dtype=np.uint8)
    key = C.c_void_p(host.ctypes.data)
    ov = lambda ptr, w, h, pitch: lib.vb_override_image(r.handle, key, w, h, C.c_void_p(ptr), pitch)
    assert ov(host.ctypes.data, 8, 8, 32) == VB_E_INVALID  # a host pointer
    assert b"device memory" in lib.vb_last_error(r.handle)
    assert ov(t.data_ptr(), 8, 8, 28) == VB_E_INVALID  # pitch below 4 * w
    assert ov(t.data_ptr(), 8, 8, 34) == VB_E_INVALID  # pitch not a multiple of 4
    assert ov(t.data_ptr() + 2, 7, 8, 32) == VB_E_INVALID  # pointer not a multiple of 4
    assert ov(t.data_ptr(), 0, 8, 32) == VB_E_INVALID and ov(t.data_ptr(), 8, 0, 32) == VB_E_INVALID
    assert lib.vb_mark_override_image_dirty(r.handle, key) == VB_E_INVALID  # nothing was set
    with pytest.raises(ValueError):
        r.register_texture(torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"))  # not (H, W, 4)

    class HostArray:  # claims to be a device array but points at host memory
        __cuda_array_interface__ = {"shape": (8, 8, 4), "typestr": "|u1", "data": (host.ctypes.data, False), "version": 3}
    with pytest.raises(VelloB200Error, match="device memory"):
        r.register_texture(HostArray())
    p = RenderParams(BASE, 64, 64, AA_MSAA16)
    draw = lambda im: (lambda s: s.draw_image(im, Affine.scale(3.0)))
    # a size mismatch at the device resolve
    img = Image(host)
    r.override_image(img, torch.zeros((8, 9, 4), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="-1"):
        native(draw(img)).upload_device(r)
    r.override_image(img, None)
    # a texture registered on another renderer
    other = Renderer()
    tex = other.register_texture(t)
    with pytest.raises(ValueError, match="-1"):
        native(draw(tex)).upload_device(r)
    assert b"no override" in lib.vb_last_error(r.handle)
    with pytest.raises(VelloB200Error):
        r.unregister_texture(tex)
    # the host resolve of a scene holding a registered texture: OK, zeros in its region, and the same bytes from Python
    rng = np.random.default_rng(9)
    side = Image(rng.integers(1, 256, (5, 6, 4), dtype=np.uint8))

    def both(s):
        s.draw_image(side, Affine.translate(2, 2))
        s.draw_image(tex, Affine.translate(20, 2))
    nat = native(both).resolve()
    py = resolve(_py_scene(both).encoding)
    assert nat.scene.tobytes() == py.scene.tobytes() and nat.atlas.tobytes() == py.atlas.tobytes()
    assert nat.atlas[0:8, 6:14].max() == 0 and nat.atlas[0:5, 0:6].min() >= 1
    other.unregister_texture(tex)
    other.close()
    # no fault: the renderer still renders
    assert np.array_equal(frame(r, native(draw(Image(host))), p), frame(ref, native(draw(Image(host))), p))
    torch.cuda.synchronize()
