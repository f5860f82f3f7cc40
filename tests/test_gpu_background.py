"""Backgrounds (vb_set_background; Renderer.set_background): frames drawn over the pixels of a device buffer or a CUDA array
instead of over the base colour. The reference is tests/oracle_bg.py: the oracle's own fine, its tiles started at the
background's values as the float32 numpy restatement of the load gives them (`start_values`), with the f32 output of
tests/oracle_f32.py. Exact, bit for bit, into RGBA32F premultiplied destinations and byte for byte into RGBA8: the whole oracle
pipeline in MSAA8 / MSAA16, its fine replayed on the frame's own command lists in Area (tests/parity.py's replay_fine). Then
the identities the header states, in-place frames, windows, bands, batches, graphs, damage tracking, the refusals and a layer
cache. Run on an H100 with `pytest -m gpu`."""
import ctypes as C
import os

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Scene, resolve
from vello_b200.renderer import Renderer, VelloB200Error, _Destination
from vello_b200.shapes import Affine, Circle, Rect

from . import oracle_bg
from .oracle_bg import start_values, store_rgba8_straight
from .parity import replay_fine
from .test_gpu_destination_formats import FArray, _blurred, _images, assert_bits
from .test_gpu_destinations import Array

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

AAS = [AA_AREA, AA_MSAA8, AA_MSAA16]
FORMATS = ["rgba8", "bgra8", "rgba16f", "rgba32f"]
TORCH = {"rgba8": torch.uint8, "bgra8": torch.uint8, "rgba16f": torch.float16, "rgba32f": torch.float32}
NP = {"rgba8": np.uint8, "bgra8": np.uint8, "rgba16f": np.float16, "rgba32f": np.float32}


def _mixed():
    """Nested clips, non-separable blend layers, a luminance mask, a gradient, an image and a blurred rectangle."""
    s = Scene()
    g, _, _ = scenes.gradient_extend()
    s.append(g, Affine.scale(0.5))
    im, _, _ = _images()
    s.append(im, Affine.translate(10.0, 150.0) * Affine.scale(0.6))
    bl, _, _ = _blurred()
    s.append(bl, Affine.translate(150.0, 20.0))
    s.push_layer(FILL_NON_ZERO, 14, 3, 0.9, Affine.IDENTITY, Circle(150, 150, 120))  # luminosity mix
    s.push_layer(FILL_NON_ZERO, 12, 3, 0.8, Affine.IDENTITY, Rect(40, 40, 260, 250))  # hue mix, nested clip
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.3, 0.1, 0.7), None, Rect(0, 0, 300, 300))
    s.pop_layer()
    s.pop_layer()
    s.push_luminance_mask_layer(FILL_NON_ZERO, 1.0, Affine.IDENTITY, Rect(180, 180, 300, 300))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.9, 0.4, 0.6), None, Circle(240, 240, 50))
    s.pop_layer()
    return s, 310, 290


SCENES = {
    "tiger": (lambda: (scenes.tiger(320, 240), 320, 240), Color(0.1, 0.2, 0.3, 1.0)),
    "mixed": (_mixed, Color(0.0, 0.0, 0.0, 0.0)),
}


def scene(name):
    build, base = SCENES[name]
    s, w, h = build()
    return resolve(s.encoding), w, h, base


def noise(h, w, fmt, seed=1, n=None):
    """Random texels whose alpha includes 0 and 255 (or 0.0 and 1.0), as a numpy array of the format's type."""
    rng = np.random.default_rng(seed)
    shape = (h, w, 4) if n is None else (n, h, w, 4)
    if NP[fmt] == np.uint8:
        t = rng.integers(0, 256, shape, dtype=np.uint8)
        t[..., 0, 0, 3] = 0
        t[..., 0, 1, 3] = 255
        t[..., 1::3, :, 3] = 255
        t[..., 2::5, :, 3] = 0
    else:
        t = rng.random(shape, dtype=np.float32).astype(NP[fmt])
        t[..., 1::3, :, 3] = 1.0
        t[..., 2::5, :, 3] = 0.0
    return t


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def r():
    rr = Renderer()
    yield rr
    rr.close()


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    lib = oracle_bg.build(str(tmp_path_factory.mktemp("oracle_bg")))
    return oracle_bg.F32BgOracle(lib, threads=max(1, os.cpu_count() or 1))


def into32(r, p, **kw):
    t = torch.full((p.height, p.width, 4), -7.0, dtype=torch.float32, device="cuda")
    key = r.register_destination(t, format="rgba32f", alpha="premultiplied")
    r.render_resident(p, key, **kw)
    r.unregister_destination(key)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def plain(r, p, **kw):
    buf = torch.zeros((p.height, p.width, 4), dtype=torch.uint8, device="cuda")
    r.render_resident(p, buf.data_ptr(), **kw)
    torch.cuda.synchronize()
    return buf.cpu().numpy()


def reference(r, o, packed, w, h, aa, base, start):
    """(f32 premultiplied, RGBA8 straight) of the oracle over `start` for the last frame of r."""
    f32 = np.zeros((h, w, 4), np.float32)
    o.f32(f32, False)
    o.bg(start)
    try:
        img = replay_fine(r, o, packed, w, h, aa, base) if aa == AA_AREA else o.render(packed, w, h, base.premul_rgba8_u32(), aa)
    finally:
        o.f32(None)
        o.bg(None)
    return f32, img


# ---- oracle parity ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("aa", AAS)
def test_oracle_parity(r, oracle, name, aa):
    packed, w, h, base = scene(name)
    r.upload(packed)
    p = RenderParams(base, w, h, aa)
    try:
        for k, fmt in enumerate(FORMATS):
            tex = noise(h, w, fmt, seed=k)
            t = dev(tex)
            for alpha in ("straight", "premultiplied"):
                start = start_values(tex, fmt, alpha == "premultiplied")
                r.set_background(t, format=fmt, alpha=alpha)
                got32 = into32(r, p)
                want32, want8 = reference(r, oracle, packed, w, h, aa, base, start)
                assert_bits(got32, want32, f"{name} aa={aa} {fmt} {alpha}: RGBA32F premultiplied vs the oracle")
                got8 = plain(r, p)
                if aa == AA_AREA:
                    _, want8 = reference(r, oracle, packed, w, h, aa, base, start)
                assert (got8 == want8).all(), f"{name} aa={aa} {fmt} {alpha}: RGBA8 differs in {int((got8 != want8).any(-1).sum())} pixels"
    finally:
        r.set_background()


# ---- identities and conversions --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", AAS)
def test_base_colour_background_is_the_plain_frame(r, aa):
    packed, w, h, base = scene("tiger")
    base = Color(0.1, 0.2, 0.3, 0.6)
    r.upload(packed)
    p = RenderParams(base, w, h, aa)
    want = plain(r, p)
    u = base.premul_rgba8_u32()
    bg = dev(np.broadcast_to(np.array([u & 255, (u >> 8) & 255, (u >> 16) & 255, u >> 24], np.uint8), (h, w, 4)))
    r.set_background(bg, alpha="premultiplied")
    try:
        assert (plain(r, p) == want).all()
        out = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        key = r.register_destination(out)
        r.render_resident(p, key)
        r.unregister_destination(key)
        assert (out.cpu().numpy() == want).all()
    finally:
        r.set_background()


def _empty(r, w, h):
    r.upload(resolve(Scene().encoding))
    return RenderParams(Color(0.5, 0.25, 0.75, 1.0), w, h, AA_MSAA16)


def test_every_byte_pair(r):
    """An empty scene over every (value, alpha) byte pair: the load and the store restated in float32 numpy."""
    v, a = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    tex = np.stack([v, 255 - v, v, a], axis=-1)
    p = _empty(r, 256, 256)
    try:
        for fmt in ("rgba8", "bgra8"):
            for alpha in ("straight", "premultiplied"):
                start = start_values(tex, fmt, alpha == "premultiplied")
                r.set_background(dev(tex), format=fmt, alpha=alpha)
                assert_bits(into32(r, p), start, f"{fmt} {alpha}: RGBA32F")
                assert (plain(r, p) == store_rgba8_straight(start)).all(), f"{fmt} {alpha}: RGBA8"
        # a premultiplied RGBA8 background into an RGBA8 premultiplied destination comes back as it was
        pre = np.minimum(tex, tex[..., 3:4])
        r.set_background(dev(pre), alpha="premultiplied")
        out = torch.zeros((256, 256, 4), dtype=torch.uint8, device="cuda")
        key = r.register_destination(out, alpha="premultiplied")
        r.render_resident(p, key)
        r.unregister_destination(key)
        assert (out.cpu().numpy() == pre).all()
    finally:
        r.set_background()


@pytest.mark.parametrize("fmt", ["rgba16f", "rgba32f"])
def test_float_edges(r, fmt):
    vals = np.array([np.nan, np.inf, -np.inf, -0.5, -0.0, 0.0, 0.25, 1.0, 1.5, 7.0, 1e-8, 0.999], np.float32)
    g = np.stack(np.meshgrid(vals, vals), -1).reshape(-1, 2)
    tex = np.stack([g[:, 0], g[:, 1], g[:, 0][::-1], g[:, 1]], -1).reshape(12, 12, 4).astype(NP[fmt])
    p = _empty(r, 12, 12)
    try:
        for alpha in ("straight", "premultiplied"):
            start = start_values(tex, fmt, alpha == "premultiplied")
            r.set_background(dev(tex), format=fmt, alpha=alpha)
            assert_bits(into32(r, p), start, f"{fmt} {alpha}")
            assert (plain(r, p) == store_rgba8_straight(start)).all()
        # values already in [0, 1] (-0 is read as +0), premultiplied: bit for bit through a destination of the same format
        inside = (np.clip(np.nan_to_num(tex.astype(np.float32)), 0, 1) + np.float32(0.0)).astype(NP[fmt])
        r.set_background(dev(inside), format=fmt, alpha="premultiplied")
        out = torch.zeros((12, 12, 4), dtype=TORCH[fmt], device="cuda")
        key = r.register_destination(out, format=fmt, alpha="premultiplied")
        r.render_resident(p, key)
        r.unregister_destination(key)
        assert_bits(out.cpu().numpy(), inside, "round trip")
    finally:
        r.set_background()


# ---- in place, culling, windows, bands, odd sizes --------------------------------------------------------------------------
def _tiger_params(r, w, h, aa=AA_MSAA16):
    r.upload(resolve(scenes.tiger(w, h).encoding))
    return RenderParams(Color(0.1, 0.2, 0.3, 0.6), w, h, aa)


@pytest.mark.parametrize("aa", AAS)
def test_in_place_and_culling(r, aa):
    w, h = 400, 300
    p = _tiger_params(r, w, h, aa)
    tex = noise(h, w, "rgba8", seed=9)
    try:
        r.set_background(dev(tex))
        want = plain(r, p)
        r.set_occlusion_cull(False)
        assert (plain(r, p) == want).all(), "occlusion culling off differs"
        r.set_occlusion_cull(True)
        buf = dev(tex)
        r.set_background(buf)
        r.render_resident(p, buf.data_ptr())
        assert (buf.cpu().numpy() == want).all(), "linear in place"
        a = Array(w + 5, h + 2)
        big = np.zeros((h + 2, w + 5, 4), np.uint8)
        big[1:1 + h, 3:3 + w] = tex
        a.write(big)
        r.set_background(array=a.handle.value, origin=(3, 1))
        key = r.register_destination(array=a.handle.value, origin=(3, 1))
        r.render_resident(p, key)
        r.unregister_destination(key)
        r.set_background()
        assert (a.read()[1:1 + h, 3:3 + w] == want).all(), "array in place"
        a.free()
    finally:
        r.set_occlusion_cull(True)
        r.set_background()


def test_windows_bands_and_odd_sizes(r):
    w, h = 1000, 333
    p = _tiger_params(r, w, h)
    tex = noise(h, w, "rgba32f", seed=4)
    try:
        r.set_background(dev(tex), format="rgba32f")
        want = plain(r, p)
        want32 = into32(r, p)
        assert not (want32 == -7.0).any()
        # a tile-row window reads its own rows
        out = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        key = r.register_destination(out)
        r.render_resident(p, key, tile_rows=(5, 11))
        r.unregister_destination(key)
        assert (out.cpu().numpy()[80:176] == want[80:176]).all()
        # read-back bands (a host destination) and a streamed frame
        r.upload(resolve(scenes.tiger(w, h).encoding))
        host = np.zeros((h, w, 4), np.uint8)
        from vello_b200.renderer import FrameStats, _params_struct
        st = FrameStats()
        r._check(r.lib.vb_render_uploaded(r.handle, C.byref(_params_struct(p)), host.ctypes.data, 0, C.byref(st)), "vb_render_uploaded")
        assert (host == want).all(), "banded read-back"
        frames = list(r.render_stream([scenes.tiger(w, h)] * 4, p))
        assert all((f == want).all() for f in frames), "streamed frames"
    finally:
        r.set_background()


def test_batch_annotated_in_place(r):
    n, w, h = 4, 200, 120
    ss = []
    for k in range(n):
        s = Scene()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.1 * k, 0.2, 0.7), None, Rect(10 + 20 * k, 10, 90 + 20 * k, 80))
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.1, 0.8, 0.3, 0.5), None, Circle(120, 60 + 5 * k, 30))
        ss.append(s)
    imgs = noise(h, w, "rgba8", seed=2, n=n)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    try:
        want = []
        for k in range(n):
            r.upload(resolve(ss[k].encoding))
            r.set_background(dev(imgs[k]))
            want.append(plain(r, p))
        t = dev(imgs)
        r.set_background(t)
        r.render_batch(ss, p, out=t)
        torch.cuda.synchronize()
        assert (t.cpu().numpy() == np.stack(want)).all()
        # an array cannot hold a batch
        a = Array(w, h * n)
        r.set_background(array=a.handle.value)
        with pytest.raises(VelloB200Error, match="batch"):
            r.render_batch(ss, p, out=torch.zeros((n, h, w, 4), dtype=torch.uint8, device="cuda"))
        r.set_background()
        a.free()
    finally:
        r.set_background()


# ---- graphs, overflow, damage, clearing, refusals --------------------------------------------------------------------------
def test_graphs_overflow_damage_and_clearing():
    r = Renderer()
    try:
        w, h = 320, 240
        p = _tiger_params(r, w, h)
        plain_frame = plain(r, p)
        launches = r.last_stats.kernel_launches
        tex = noise(h, w, "rgba8", seed=3)
        bg = dev(tex)
        r.set_background(bg)
        first = plain(r, p)
        caps = r.debug_graph_captures()
        bg.copy_(dev(noise(h, w, "rgba8", seed=8)))
        second = plain(r, p)
        assert r.debug_graph_captures() == caps, "new contents recaptured"
        assert (second != first).any()
        other = dev(tex)
        r.set_background(other)
        assert (plain(r, p) == first).all()
        assert r.debug_graph_captures() == caps + 1, "a new descriptor replayed an old graph"
        # a frame enqueued before set_background keeps its background
        out = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        r.enqueue(p, out.data_ptr())
        r.set_background()
        r.finish()
        assert (out.cpu().numpy() == first).all()
        # a re-run after an overflow reads the background it was issued with
        r.set_background(other)
        r.limit_arena("segments", 16)
        st = r.render_resident(p, out.data_ptr())
        assert st.retries >= 1 and (out.cpu().numpy() == first).all()
        # damage tracking: background frames are full and no base
        r.set_damage_tracking(True)
        n_tiles = ((w + 15) // 16) * ((h + 15) // 16)
        r.render_resident(p, out.data_ptr())
        assert int(r.last_damage().sum()) == n_tiles
        r.render_resident(p, out.data_ptr())
        assert int(r.last_damage().sum()) == n_tiles
        r.set_background()
        r.render_resident(p, out.data_ptr())
        assert int(r.last_damage().sum()) == n_tiles, "the first frame after a background frame is full"
        r.set_damage_tracking(False)
        # cleared: the plain frame and its launch count
        assert (plain(r, p) == plain_frame).all() and r.last_stats.kernel_launches == launches
    finally:
        r.close()


def test_refusals(r):
    w, h = 64, 48
    p = _tiger_params(r, w, h)
    try:
        t = torch.zeros((h, w - 1, 4), dtype=torch.uint8, device="cuda")
        r.set_background(t)
        with pytest.raises(ValueError, match="cannot hold 1 cell"):  # Python knows the target's shape
            plain(r, p)
        # the library's own check, for a caller that passes only the descriptor
        r._check(r.lib.vb_set_background(r.handle, C.byref(_Destination(0, 0, t.data_ptr(), (w - 1) * 4, None, 0, 0))), "vb_set_background")
        r._background_shape = None
        with pytest.raises(VelloB200Error, match="row pitch is below 4"):
            plain(r, p)
        a = Array(w, h)
        r.set_background(array=a.handle.value, origin=(1, 0))
        with pytest.raises(VelloB200Error, match="does not fit the array"):
            plain(r, p)
        r.set_background()
        with pytest.raises(VelloB200Error, match="cudaArraySurfaceLoadStore"):
            b = Array(w, h, flags=0)
            try:
                r.set_background(array=b.handle.value)
            finally:
                b.free()
        with pytest.raises(VelloB200Error, match="channels"):
            r.set_background(array=a.handle.value, format="rgba32f")
        a.free()
        with pytest.raises(VelloB200Error, match="ptr is not device"):
            r.set_background(_HostFake(h, w))
        key = r.register_destination(torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"))
        with pytest.raises(VelloB200Error, match="ptr is not device"):
            r.set_background(_HostFake(h, w, key))
        r.unregister_destination(key)
        f32 = torch.zeros((h, w + 1, 4), device="cuda", dtype=torch.float32)
        d = _Destination(0, 3, f32.data_ptr(), w * 16 + 4, None, 0, 0)  # Python refuses this pitch before the library sees it
        with pytest.raises(VelloB200Error, match="row_pitch_bytes is not a multiple of 16"):
            r._check(r.lib.vb_set_background(r.handle, C.byref(d)), "vb_set_background")
    finally:
        r.set_background()


class _HostFake:
    def __init__(self, h, w, ptr=None, pitch=None, typestr="|u1"):
        self._buf = np.zeros((h, w, 4), np.uint8)
        e = int(typestr[2:])
        self.__cuda_array_interface__ = {"shape": (h, w, 4), "typestr": typestr, "version": 3,
                                         "data": (ptr if ptr is not None else self._buf.ctypes.data, False),
                                         "strides": (pitch or w * 4 * e, 4 * e, e)}


# ---- a layer cache ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", AAS)
def test_layer_cache(r, aa):
    """P rendered once into an RGBA32F premultiplied buffer, then S over it, is within 1 LSB of P followed by S rendered whole."""
    w, h = 320, 240
    P = scenes.tiger(w, h)
    S = Scene()
    for k in range(40):
        S.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.5, 0.1 * (k % 10), 0.6), None, Circle(8 * k, 6 * k, 12))
    whole = Scene()
    whole.append(P)
    whole.append(S)
    base = Color(0.1, 0.2, 0.3, 1.0)
    p = RenderParams(base, w, h, aa)
    try:
        r.upload(resolve(P.encoding))
        layer = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        key = r.register_destination(layer, format="rgba32f", alpha="premultiplied")
        r.render_resident(p, key)
        r.unregister_destination(key)
        r.upload(resolve(S.encoding))
        r.set_background(layer, format="rgba32f", alpha="premultiplied")
        cached = plain(r, p)
        r.set_background()
        r.upload(resolve(whole.encoding))
        full = plain(r, p)
        d = np.abs(cached.astype(int) - full.astype(int))
        assert d.max() <= 1, f"aa={aa}: {d.max()}"
        print(f"layer cache aa={aa}: {int((d != 0).sum())} channel values differ")
    finally:
        r.set_background()


# ---- array backgrounds in every format ---------------------------------------------------------------------------------------
def _bg_array(img, fmt):
    """A CUDA array of img's texels in format fmt (surface load/store)."""
    h, w = img.shape[:2]
    if NP[fmt] == np.uint8:
        a = Array(w, h)
        a.write(img)
        return a
    a = FArray(w, h, fmt)
    img = np.ascontiguousarray(img, dtype=NP[fmt])
    assert a.rt.cudaMemcpy2DToArray(a.handle, 0, 0, img.ctypes.data, w * a.texel, w * a.texel, h, 1) == 0
    return a


@pytest.mark.parametrize("fmt", FORMATS)
def test_array_backgrounds_equal_linear_ones(r, fmt):
    """Over a 1000x333 frame (a partial edge tile in x and y): an array background at origin (0, 0), where the lanes read
    16-byte texel groups, and at (3, 1) and (1, 2), where they read texel by texel (odd columns for every format but RGBA32F),
    equals the same texels as a linear background, straight and premultiplied, into RGBA32F and RGBA8."""
    w, h = 1000, 333
    p = _tiger_params(r, w, h, AA_MSAA8)
    tex = noise(h, w, fmt, seed=11)
    try:
        for alpha in ("straight", "premultiplied"):
            r.set_background(dev(tex), format=fmt, alpha=alpha)
            want32, want8 = into32(r, p), plain(r, p)
            for ox, oy in ((0, 0), (3, 1), (1, 2)):
                big = np.zeros((h + oy + 2, w + ox + 5, 4), NP[fmt])
                big[oy:oy + h, ox:ox + w] = tex
                a = _bg_array(big, fmt)
                try:
                    r.set_background(array=a.handle.value, format=fmt, alpha=alpha, origin=(ox, oy))
                    assert_bits(into32(r, p), want32, f"{fmt} {alpha} array at ({ox}, {oy}), RGBA32F")
                    assert (plain(r, p) == want8).all(), f"{fmt} {alpha} array at ({ox}, {oy}), RGBA8"
                    r.set_background()
                finally:
                    a.free()
    finally:
        r.set_background()


# ---- a frame keeps its background -------------------------------------------------------------------------------------------
def _begin(r, packed, p, out):
    """vb_render_begin of `packed` into host `out`; returns the stats it reports (of the frame two before)."""
    from vello_b200.renderer import FrameStats, _Layout, _params_struct
    scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    st = FrameStats()
    r._check(r.lib.vb_render_begin(r.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None,
                                   512, ramps.shape[0], atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(_params_struct(p)),
                                   out.ctypes.data, C.byref(st)), "vb_render_begin")
    return st


@pytest.mark.parametrize("kind", ["linear", "array"])
def test_streamed_rerun_keeps_its_background(kind):
    """A streamed frame that overflows is re-run once the next frame has been issued. Between the two, set_background
    switches to another buffer; the re-run must read the background the frame was issued with (Frame::bg), not the
    renderer's. With an array, set_background instead completes that frame, re-run included, before it destroys the array's
    surface, so the frame reads the array whichever background it took."""
    r = Renderer()
    try:
        w, h = 320, 240
        packed = resolve(scenes.tiger(w, h).encoding)
        r.upload(packed)
        p = RenderParams(Color(0.1, 0.2, 0.3, 0.6), w, h, AA_MSAA16)
        tex_a, tex_b = noise(h, w, "rgba8", seed=21), noise(h, w, "rgba8", seed=22)
        bg_a, bg_b = dev(tex_a), dev(tex_b)
        r.set_background(bg_a)
        want_a = plain(r, p)
        r.set_background(bg_b)
        want_b = plain(r, p)
        assert (want_a != want_b).any()
        arr = _bg_array(tex_a, "rgba8") if kind == "array" else None
        if arr is not None:
            r.set_background(array=arr.handle.value)
        else:
            r.set_background(bg_a)
        outs = [np.zeros((h, w, 4), np.uint8) for _ in range(3)]
        r.limit_arena("segments", 16)
        _begin(r, packed, p, outs[0])
        r.set_background(bg_b)
        _begin(r, packed, p, outs[1])
        st = _begin(r, packed, p, outs[2])  # reports the first frame, complete
        r._check(r.lib.vb_readback_wait(r.handle), "vb_readback_wait")
        if arr is None:
            # with an array, set_background completed the first frame (and its re-run) itself, and no later call reports it
            assert st.retries >= 1, "the first streamed frame did not overflow"
        assert (outs[0] == want_a).all(), "the re-run did not read the background its frame was issued with"
        assert (outs[1] == want_b).all() and (outs[2] == want_b).all()
        if arr is not None:
            arr.free()
    finally:
        r.close()


# ---- refusals of grouped and exchanged renderers -----------------------------------------------------------------------------
def test_group_and_exchange_refuse_backgrounds():
    from vello_b200.renderer import RendererGroup
    t = torch.zeros((64, 64, 4), dtype=torch.uint8, device="cuda")
    d = _Destination(0, 0, t.data_ptr(), 256, None, 0, 0)
    g = RendererGroup([torch.cuda.current_device()])
    try:
        sub = C.c_void_p(g.lib.vb_group_renderer(g.handle, 0))
        assert g.lib.vb_set_background(sub, C.byref(d)) != 0
        assert b"vb_group" in g.lib.vb_last_error(sub)
    finally:
        g.close()
    r = Renderer()
    try:
        r.upload(resolve(scenes.tiger(64, 64).encoding))
        arena, nbytes = C.c_void_p(), C.c_size_t()
        r.set_background(t)
        assert r.lib.vb_exchange_configure(r.handle, 0, 1, C.byref(arena), C.byref(nbytes)) != 0
        assert b"background" in r.lib.vb_last_error(r.handle)
        r.set_background()
        r._check(r.lib.vb_exchange_configure(r.handle, 0, 1, C.byref(arena), C.byref(nbytes)), "vb_exchange_configure")
        with pytest.raises(VelloB200Error, match="exchange configured"):
            r.set_background(t)
    finally:
        r.close()
