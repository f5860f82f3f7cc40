"""Float and premultiplied destinations (vb_register_destination with VB_DEST_RGBA16F / VB_DEST_RGBA32F and
VB_DEST_PREMULTIPLIED; Renderer.register_destination(format=..., alpha=...)). Every relation here is exact, bit for bit:

1. RGBA32F premultiplied texels are the oracle's f32 output (fine's premultiplied pixel, clamped to [0, 1]; the oracle's
   own fine with its store extended to write it, tests/oracle_f32.py): its whole pipeline in MSAA8 / MSAA16, its fine
   replayed on the frame's own command lists in Area (tests/parity.py's replay_fine);
2. RGBA32F straight is the oracle's straight f32 output, and the straight formula applied in float32 to (1) wherever
   (1)'s alpha is below 1 (fine's alpha can sum to a little above 1, which (1) clamps); unorm8 of it is the RGBA8 frame;
3. RGBA16F is np.float16 (round to nearest even) of the matching f32 output;
4. RGBA8 / BGRA8 premultiplied are unorm8 of the premultiplied f32 output;
then where float frames land (slices, arrays at odd origins, windows), every entry point, graphs, damage tracking and the
refusals. Arrays are allocated, filled and read back through the CUDA runtime (`libcudart.so.12`). Run on an H100 with
`pytest -m gpu`."""
import ctypes as C
import os

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (BLACK, Color, FILL_NON_ZERO, Image, QUALITY_HIGH, QUALITY_LOW, QUALITY_MEDIUM, Scene,
                                 resolve)
from vello_b200.renderer import STAGES, FrameStats, Renderer, VelloB200Error, _Layout, _params_struct
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Circle, Rect

from . import oracle_f32 as f32_oracle
from .parity import replay_fine
from .test_gpu_destinations import KIND_FLOAT, KIND_UNSIGNED, SURFACE_LOAD_STORE, _Fmt, _bound_composition, cudart

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

H2D, D2H = 1, 2
SENT = -7.0  # a guard value fine can never store (texels are in [0, 1])
TEXEL = {"rgba16f": 8, "rgba32f": 16}
DTYPE = {"rgba16f": torch.float16, "rgba32f": torch.float32}
NP_DTYPE = {"rgba16f": np.float16, "rgba32f": np.float32}


# ---- references in float32 numpy --------------------------------------------------------------------------------------------
def straight(pre):
    """The straight texel of a clamped premultiplied f32 texel: clamp01(rgb * (1 / max(a, 1e-6))), a."""
    a_inv = np.float32(1.0) / np.fmax(pre[..., 3:], np.float32(1e-6))
    out = pre.copy()
    out[..., :3] = np.fmin(np.float32(1.0), np.fmax(np.float32(0.0), pre[..., :3] * a_inv))
    return out


def unorm8(v):
    return np.floor(np.float32(0.5) + np.float32(255.0) * v).astype(np.uint8)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint16)


def assert_bits(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = (g != w).any(axis=-1)
    assert not bad.any(), f"{what}: {int(bad.sum())} texels differ, first at {tuple(int(v) for v in np.argwhere(bad)[0])}: " \
                          f"{got[tuple(np.argwhere(bad)[0])]} vs {want[tuple(np.argwhere(bad)[0])]}"


# ---- float CUDA arrays -------------------------------------------------------------------------------------------------------
class FArray:
    """A 2-D CUDA array of w x h texels of four float16 or float32 channels (or `bits` / `kind` as given)."""

    def __init__(self, w, h, fmt="rgba32f", bits=None, kind=KIND_FLOAT, flags=SURFACE_LOAD_STORE):
        self.rt, self.w, self.h, self.fmt = cudart(), w, h, fmt
        self.texel = TEXEL.get(fmt, 4)
        b = bits or (self.texel * 2,) * 4
        self.handle = C.c_void_p()
        assert self.rt.cudaMallocArray(C.byref(self.handle), C.byref(_Fmt(*b, kind)), w, h, flags) == 0

    def fill(self, value=SENT):
        img = np.full((self.h, self.w, 4), value, NP_DTYPE[self.fmt])
        assert self.rt.cudaMemcpy2DToArray(self.handle, 0, 0, img.ctypes.data, self.w * self.texel, self.w * self.texel, self.h, H2D) == 0

    def read(self):
        torch.cuda.synchronize()
        out = np.zeros((self.h, self.w, 4), NP_DTYPE[self.fmt])
        assert self.rt.cudaMemcpy2DFromArray(out.ctypes.data, self.w * self.texel, self.handle, 0, 0, self.w * self.texel, self.h, D2H) == 0
        return out

    def free(self):
        if self.handle.value:
            self.rt.cudaFreeArray(self.handle)
            self.handle = C.c_void_p()


# ---- scenes ------------------------------------------------------------------------------------------------------------------
def _images():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (11, 13, 4), dtype=np.uint8)
    s = Scene()
    for i, q in enumerate((QUALITY_LOW, QUALITY_MEDIUM, QUALITY_HIGH)):
        t = Affine.translate(20.0 + 130.0 * i, 30.0) * Affine.rotate(0.15 * (i + 1)) * Affine.scale(7.3)
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Image(img, quality=q, alpha=0.8), t, Rect(10 + 130 * i, 20, 130 + 130 * i, 200))
    return s, 400, 230


def _blurred():
    s = Scene()
    s.draw_blurred_rounded_rect(Affine.translate(80.0, 70.0), Rect(-50, -30, 50, 30), Color.from_rgba8(250, 200, 30), 8.0, 5.0)
    s.draw_blurred_rounded_rect(Affine.translate(220.0, 80.0) * Affine.rotate(0.3), Rect(-60, -25, 60, 25),
                                Color.from_rgba8(30, 200, 250, 200), 0.0, 9.0)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.2, 0.4, 0.5), None, Circle(160, 90, 45))
    return s, 300, 170


def _tiger():
    return scenes.tiger(640, 480), 640, 480


SCENES = {  # name: (builder, base colour)
    "tiger": (_tiger, Color(0.1, 0.2, 0.3, 1.0)),
    "blend_grid": (scenes.blend_grid, BLACK),
    "compose_grid": (scenes.compose_grid, Color(0.0, 0.0, 0.0, 0.0)),
    "gradients": (scenes.gradient_extend, Color(1.0, 1.0, 1.0, 1.0)),
    "images": (_images, Color(0.2, 0.2, 0.2, 0.5)),
    "blurred": (_blurred, BLACK),
    "nested_clips": (lambda: scenes.many_clips(20, 8), BLACK),
    "tiger_clear": (_tiger, Color(0.0, 0.0, 0.0, 0.0)),
}
AAS = [AA_AREA, AA_MSAA8, AA_MSAA16]


def scene(name):
    build, base = SCENES[name]
    s, w, h = build()
    return resolve(s.encoding), w, h, base


@pytest.fixture(scope="module")
def r():
    rr = Renderer()
    yield rr
    rr.close()


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    """The CPU oracle with its f32 output (tests/oracle_f32.py)."""
    lib = f32_oracle.build(str(tmp_path_factory.mktemp("oracle_f32")))
    return f32_oracle.F32Oracle(lib, threads=max(1, os.cpu_count() or 1))


def into(r, p, fmt, alpha="straight", **kw):
    """A frame of r into a contiguous tensor of format fmt, registered as a destination: (h, w, 4) numpy."""
    if fmt in TEXEL:
        t = torch.full((p.height, p.width, 4), SENT, dtype=DTYPE[fmt], device="cuda")
    else:
        t = torch.zeros((p.height, p.width, 4), dtype=torch.uint8, device="cuda")
    key = r.register_destination(t, format=fmt, alpha=alpha)
    r.render_resident(p, key, **kw)
    r.unregister_destination(key)
    torch.cuda.synchronize()
    return t.cpu().numpy()


def plain(r, p, **kw):
    buf = torch.empty((p.height, p.width, 4), dtype=torch.uint8, device="cuda")
    r.render_resident(p, buf.data_ptr(), **kw)
    torch.cuda.synchronize()
    return buf.cpu().numpy()


def oracle_f32(r, o, packed, w, h, aa, base, straight_alpha=False):
    """The oracle's f32 output (premultiplied, or straight with `straight_alpha`) for the last frame of r: fine replayed on
    r's command lists in Area, the whole pipeline in MSAA (where the GPU's RGBA8 frames are exact against it)."""
    f32 = np.zeros((h, w, 4), np.float32)
    o.f32(f32, straight_alpha)
    try:
        if aa == AA_AREA:
            replay_fine(r, o, packed, w, h, aa, base)
        else:
            o.render(packed, w, h, base.premul_rgba8_u32(), aa)
    finally:
        o.f32(None)
    return f32


# ---- 1-5. values -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("aa", AAS)
def test_float_and_premultiplied_values(r, oracle, name, aa):
    """Each frame against the oracle's f32 output for that frame. In Area the oracle replays each frame's own command lists:
    the order of the segments in a tile's slice can differ from frame to frame, and with it the last bits of area sums, so
    there the formats are related through the oracle and not across frames. In MSAA every frame is the same."""
    packed, w, h, base = scene(name)
    r.upload(packed)
    p = RenderParams(base, w, h, aa)
    msaa = {}

    def refs(alpha):
        if aa != AA_AREA and alpha in msaa:
            return msaa[alpha]
        msaa[alpha] = oracle_f32(r, oracle, packed, w, h, aa, base, straight_alpha=alpha == "straight")
        return msaa[alpha]

    pre32 = into(r, p, "rgba32f", "premultiplied")
    want_pre = refs("premultiplied")
    assert_bits(pre32, want_pre, "RGBA32F premultiplied vs the oracle's f32 output")
    st32 = into(r, p, "rgba32f")
    want_st = refs("straight")
    assert_bits(st32, want_st, "RGBA32F straight vs the oracle's")
    # the straight formula on the premultiplied output is exact where alpha < 1; where that alpha is 1, fine's alpha may have
    # summed to a little above 1 (area coverage), and the straight colour is divided by that alpha before the clamp
    pre_same = oracle_f32(r, oracle, packed, w, h, aa, base) if aa == AA_AREA else want_pre  # of the straight frame
    below = pre_same[..., 3] < 1.0
    assert_bits(st32[below], straight(pre_same)[below], "RGBA32F straight vs the straight formula")
    if aa != AA_AREA:
        assert (unorm8(st32) == plain(r, p)).all(), "unorm8 of RGBA32F straight differs from the RGBA8 frame"
    assert_bits(into(r, p, "rgba16f", "premultiplied"), refs("premultiplied").astype(np.float16), "RGBA16F premultiplied")
    assert_bits(into(r, p, "rgba16f"), refs("straight").astype(np.float16), "RGBA16F straight")
    assert (into(r, p, "rgba8", "premultiplied") == unorm8(refs("premultiplied"))).all(), "RGBA8 premultiplied"
    assert (into(r, p, "bgra8", "premultiplied") == unorm8(refs("premultiplied"))[..., [2, 1, 0, 3]]).all(), "BGRA8 premultiplied"
    assert (into(r, p, "rgba8") == unorm8(refs("straight"))).all(), "RGBA8 straight"
    assert (into(r, p, "bgra8") == unorm8(refs("straight"))[..., [2, 1, 0, 3]]).all(), "BGRA8 straight"
    if aa == AA_AREA and name in ("images", "blurred"):
        x = pre32.astype(np.float64) * 255.0
        assert (np.abs(x - np.round(x)) > 1e-3).any(), "every RGBA32F value is a multiple of 1/255"


# ---- 6. where frames land ----------------------------------------------------------------------------------------------------
def _tiger_at(r, w, h, aa=AA_MSAA16):
    packed = resolve(scenes.tiger(w, h).encoding)
    r.upload(packed)
    return RenderParams(Color(0.1, 0.2, 0.3, 0.6), w, h, aa)


@pytest.mark.parametrize("fmt", ["rgba16f", "rgba32f"])
@pytest.mark.parametrize("size", [(1000, 517), (17, 33)])
def test_slices_and_arrays(r, fmt, size):
    w, h = size
    p = _tiger_at(r, w, h)
    for alpha in ("straight", "premultiplied"):
        want = into(r, p, fmt, alpha)
        assert (want != SENT).all()
        # column and row slices of wider tensors: texel-aligned only (odd column), and 16-byte aligned base and pitch
        for x0, extra in ((3, 5), (2, 6), (0, 1)):
            big = torch.full((h + 3, w + extra, 4), SENT, dtype=DTYPE[fmt], device="cuda")
            view = big[2:2 + h, x0:x0 + w]
            key = r.register_destination(view, format=fmt, alpha=alpha)
            r.render_resident(p, key)
            r.unregister_destination(key)
            b = big.cpu().numpy()
            assert_bits(b[2:2 + h, x0:x0 + w], want, f"{fmt} {alpha} slice at column {x0}")
            inside = np.zeros(b.shape[:2], bool)
            inside[2:2 + h, x0:x0 + w] = True
            assert (b[~inside] == SENT).all(), "a texel outside the slice was written"
        # arrays at origins with x % 4 != 0
        for ox, oy in ((3, 1), (6, 0), (1, 5)):
            a = FArray(w + ox + 2, h + oy + 3, fmt)
            a.fill()
            key = r.register_destination(array=a.handle.value, format=fmt, alpha=alpha, origin=(ox, oy))
            r.render_resident(p, key)
            r.unregister_destination(key)
            got = a.read()
            a.free()
            assert_bits(got[oy:oy + h, ox:ox + w], want, f"{fmt} {alpha} array at ({ox}, {oy})")
            inside = np.zeros(got.shape[:2], bool)
            inside[oy:oy + h, ox:ox + w] = True
            assert (got[~inside] == SENT).all(), "a texel outside the frame was written"


@pytest.mark.parametrize("fmt", ["rgba16f", "rgba32f"])
def test_windows_write_their_own_rows(r, fmt):
    w, h = 1000, 700
    p = _tiger_at(r, w, h, AA_MSAA8)
    want = into(r, p, fmt, "premultiplied")
    for kw, (y0, y1) in ((dict(tile_rows=(3, 9)), (48, 144)), (dict(bin_rows=(1, 2)), (256, 512))):
        big = torch.full((h, w + 2, 4), SENT, dtype=DTYPE[fmt], device="cuda")
        key = r.register_destination(big[:, 1:1 + w], format=fmt, alpha="premultiplied")
        r.render_resident(p, key, **kw)
        r.unregister_destination(key)
        b = big.cpu().numpy()
        assert_bits(b[y0:y1, 1:1 + w], want[y0:y1], f"{fmt} window {kw}")
        b[y0:y1, 1:1 + w] = SENT
        assert (b == SENT).all(), f"{fmt} window {kw}: a texel outside the window's rows was written"
        a = FArray(w, h, fmt)
        a.fill()
        key = r.register_destination(array=a.handle.value, format=fmt, alpha="premultiplied")
        r.render_resident(p, key, **kw)
        r.unregister_destination(key)
        got = a.read()
        a.free()
        assert_bits(got[y0:y1], want[y0:y1], f"{fmt} array window {kw}")
        got[y0:y1] = SENT
        assert (got == SENT).all(), f"{fmt} array window {kw}: a texel outside the window's rows was written"


# ---- 7. every entry point that takes a key -----------------------------------------------------------------------------------
def test_every_entry_point_into_a_float_key(r):
    packed = resolve(scenes.tiger(600, 400).encoding)
    w, h = 600, 400
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    r.upload(packed)
    want = into(r, p, "rgba16f")
    t = torch.full((h, w, 4), SENT, dtype=torch.float16, device="cuda")
    key = r.register_destination(t, format="rgba16f")
    lib, ps, st = r.lib, _params_struct(p), FrameStats()

    def check(expect=want):
        torch.cuda.synchronize()
        assert_bits(t.cpu().numpy(), expect, "entry point")
        t.fill_(SENT)

    r.render_resident(p, key)
    check()
    r.enqueue(p, key)
    r.finish()
    check()
    scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    assert lib.vb_render(r.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None,
                         512, ramps.shape[0], atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), C.c_void_p(key), 1,
                         C.byref(st)) == 0
    check()
    r.run_stages(p, STAGES[0], STAGES[-1], key)
    check()
    ns = NativeScene()
    ns.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 0.7), None, Rect(3, 5, 401, 300))
    ns.upload_device(r)
    want2 = into(r, p, "rgba16f")
    assert ns.lib.vb_render_scene(r.handle, ns.handle, C.byref(ps), C.c_void_p(key), 1, C.byref(st)) == 0
    check(want2)
    r.unregister_destination(key)


# ---- 8, 9. graphs and damage tracking into a float key ----------------------------------------------------------------------
def test_graph_replay_into_a_float_key():
    r, ref = Renderer(), Renderer()
    w, h = 640, 480
    t, t_ref = _bound_composition(r, w, h), _bound_composition(ref, w, h)
    p = RenderParams(Color(0.0, 0.0, 0.0, 0.0), w, h, AA_MSAA16)
    a = FArray(w, h, "rgba32f")
    key = r.register_destination(array=a.handle.value, format="rgba32f", alpha="premultiplied")
    r.render_resident(p, key)
    n0 = r.debug_graph_captures()
    for step in range(3):
        for tt in (t, t_ref):
            tt[5 + step, 4:] += 17.0
        torch.cuda.synchronize()
        r.render_resident(p, key)
        assert_bits(a.read(), into(ref, p, "rgba32f", "premultiplied"), f"replayed frame {step}")
    assert r.debug_graph_captures() == n0, "frames into the same float key captured again"
    r.unregister_destination(key)
    a.free()
    r.close()
    ref.close()


@pytest.mark.parametrize("fmt", ["rgba16f", "rgba32f"])
def test_damage_tracking_into_a_float_key(fmt):
    r, ref = Renderer(), Renderer()
    w, h = 640, 480
    t, t_ref = _bound_composition(r, w, h), _bound_composition(ref, w, h)
    p = RenderParams(Color(0.1, 0.1, 0.1, 0.5), w, h, AA_MSAA16)
    out = torch.full((h, w, 4), SENT, dtype=DTYPE[fmt], device="cuda")
    key = r.register_destination(out, format=fmt)
    r.set_damage_tracking(True)
    r.render_resident(p, key)
    torch.cuda.synchronize()
    assert_bits(out.cpu().numpy(), into(ref, p, fmt), "first (full) frame")
    for step in range(4):
        before = out.cpu().numpy()
        for tt in (t, t_ref):
            tt[3 + 7 * step, 4:] += 19.0
        torch.cuda.synchronize()
        r.render_resident(p, key)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert_bits(got, into(ref, p, fmt), f"incremental frame {step}")
        dmg = r.last_damage()
        assert dmg.any() and dmg.sum() < dmg.size // 4, "the frame was not incremental"
        changed = np.kron(dmg.astype(np.uint8), np.ones((16, 16), np.uint8)).astype(bool)[:h, :w]
        assert_bits(got[~changed], before[~changed], "texels outside the damaged tiles")
    r.set_damage_tracking(False)
    r.unregister_destination(key)
    r.close()
    ref.close()


# ---- 10. refusals ------------------------------------------------------------------------------------------------------------
def _refused(r, fn, *args, **kw):
    with pytest.raises(VelloB200Error):
        fn(*args, **kw)
    assert r.lib.vb_last_error(r.handle)


def test_refusals(r):
    w, h = 17, 33
    p = _tiger_at(r, w, h, AA_AREA)
    # array channels that do not match the format
    for arr_fmt, bits_, kind, fmt in (("rgba16f", None, KIND_FLOAT, "rgba32f"), ("rgba32f", None, KIND_FLOAT, "rgba16f"),
                                      ("rgba8", (8, 8, 8, 8), KIND_UNSIGNED, "rgba16f"),
                                      ("rgba8", (8, 8, 8, 8), KIND_UNSIGNED, "rgba32f"),
                                      ("rgba16f", None, KIND_FLOAT, "rgba8"),
                                      ("rgba16f", (16, 16, 16, 16), KIND_UNSIGNED, "rgba16f")):
        a = FArray(w, h, arr_fmt, bits=bits_, kind=kind)
        _refused(r, r.register_destination, array=a.handle.value, format=fmt)
        a.free()
    # misaligned ptr or pitch for the texel size, through the C ABI (Python views of float tensors are always aligned)
    from vello_b200.renderer import _Destination
    buf = torch.zeros((h, w + 2, 4), dtype=torch.float32, device="cuda")
    key = C.c_void_p()
    for fmt, off, pitch in ((3, 4, (w + 2) * 16), (3, 8, (w + 2) * 16), (3, 0, (w + 2) * 16 - 8), (2, 4, (w + 2) * 16),
                            (2, 0, w * 8 + 4), (3 | 0x200, 0, (w + 2) * 16), (4, 0, (w + 2) * 16), (0x100 | 7, 0, (w + 2) * 16)):
        d = _Destination(0, fmt, buf.data_ptr() + off, pitch, None, 0, 0)
        assert r.lib.vb_register_destination(r.handle, C.byref(d), C.byref(key)) == -1, (fmt, off, pitch)
        assert r.lib.vb_last_error(r.handle)
    # a pitch below texel size * width, checked at the frame
    d = _Destination(0, 3, buf.data_ptr(), 16 * w - 16, None, 0, 0)
    assert r.lib.vb_register_destination(r.handle, C.byref(d), C.byref(key)) == 0
    _refused(r, r.render_resident, p, key.value)
    r.unregister_destination(key.value)
    # a dtype that does not match the format
    for t, fmt in ((torch.zeros((h, w, 4), dtype=torch.float16, device="cuda"), "rgba32f"),
                   (torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"), "rgba16f"),
                   (torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"), "rgba32f"),
                   (torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"), "rgba8")):
        with pytest.raises(ValueError):
            r.register_destination(t, format=fmt)
    with pytest.raises(ValueError):
        r.register_destination(buf[:, :w], format="rgba32f", alpha="associated")
    # a batch into a float key
    packed = resolve(scenes.tiger(w, h).encoding)
    r.upload(packed)
    t = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    k = r.register_destination(t, format="rgba32f")
    r.set_cells([0, 3, int(packed.layout.n_draw_objects)])
    _refused(r, r.render_resident, p, k)
    r.upload(packed)
    r.render_resident(p, k)
    r.unregister_destination(k)
