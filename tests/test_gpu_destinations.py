"""Registered destinations (vb_register_destination / Renderer.register_destination): frames rendered straight into CUDA arrays
and pitched device buffers, in RGBA8 or BGRA8 order. Every frame must equal, byte for byte, the same renderer's frame into a
plain pointer (with R and B swapped for BGRA8), and every byte outside the frame must keep its sentinel. Arrays are allocated,
filled and read back through the CUDA runtime (`libcudart.so.12`, loaded after torch has initialised CUDA). Run on an H100 with
`pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, Color, FILL_NON_ZERO, Image, resolve
from vello_b200.renderer import STAGES, FrameStats, Renderer, VelloB200Error, _Layout, _params_struct
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Rect

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

SENT = 0x5A
SURFACE_LOAD_STORE, LAYERED = 0x02, 0x01
KIND_UNSIGNED, KIND_FLOAT = 1, 2
H2D, D2H = 1, 2
VB_E_INVALID = -1


class _Fmt(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


class _Extent(C.Structure):
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("depth", C.c_size_t)]


_RT = None


def cudart():
    global _RT
    if _RT is None:
        torch.zeros(1, device="cuda")  # torch's runtime first: the arrays live in the primary context the library uses too
        rt = C.CDLL("libcudart.so.12")
        vp, sz = C.c_void_p, C.c_size_t
        rt.cudaMallocArray.argtypes = [C.POINTER(vp), C.POINTER(_Fmt), sz, sz, C.c_uint]
        rt.cudaMalloc3DArray.argtypes = [C.POINTER(vp), C.POINTER(_Fmt), _Extent, C.c_uint]
        rt.cudaFreeArray.argtypes = [vp]
        rt.cudaMemcpy2DToArray.argtypes = [vp, sz, sz, vp, sz, sz, sz, C.c_int]
        rt.cudaMemcpy2DFromArray.argtypes = [vp, sz, vp, sz, sz, sz, sz, C.c_int]
        _RT = rt
    return _RT


class Array:
    """A 2-D CUDA array of w x h texels (RGBA8, surface load/store unless told otherwise)."""

    def __init__(self, w, h, bits=(8, 8, 8, 8), kind=KIND_UNSIGNED, flags=SURFACE_LOAD_STORE, layers=0):
        self.rt, self.w, self.h = cudart(), w, h
        self.handle = C.c_void_p()
        fmt = _Fmt(*bits, kind)
        if layers:
            e = self.rt.cudaMalloc3DArray(C.byref(self.handle), C.byref(fmt), _Extent(w, h, layers), flags | LAYERED)
        else:
            e = self.rt.cudaMallocArray(C.byref(self.handle), C.byref(fmt), w, h, flags)
        assert e == 0, f"cudaMallocArray: {e}"

    def fill(self, value=SENT):
        self.write(np.full((self.h, self.w, 4), value, np.uint8))

    def write(self, img):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        assert self.rt.cudaMemcpy2DToArray(self.handle, 0, 0, img.ctypes.data, self.w * 4, self.w * 4, self.h, H2D) == 0

    def read(self):
        torch.cuda.synchronize()
        out = np.zeros((self.h, self.w, 4), np.uint8)
        assert self.rt.cudaMemcpy2DFromArray(out.ctypes.data, self.w * 4, self.handle, 0, 0, self.w * 4, self.h, D2H) == 0
        return out

    def free(self):
        if self.handle.value:
            self.rt.cudaFreeArray(self.handle)
            self.handle = C.c_void_p()


def bgra(img):
    return img[..., [2, 1, 0, 3]]


def plain_frame(r, p, **kw):
    """The reference: the same renderer's frame into a plain device pointer."""
    buf = torch.empty((p.height, p.width, 4), dtype=torch.uint8, device="cuda")
    r.render_resident(p, buf.data_ptr(), **kw)
    torch.cuda.synchronize()
    return buf.cpu().numpy()


def pitched(h, w, pitch):
    """A device buffer of h rows `pitch` bytes apart, filled with the sentinel, and the (h, w, 4) view of its pixels."""
    big = torch.full((h, pitch), SENT, dtype=torch.uint8, device="cuda")
    return big, torch.as_strided(big, (h, w, 4), (pitch, 4, 1))


def check_linear(big, w, want):
    b = big.cpu().numpy()
    assert (b[:, :4 * w].reshape(want.shape) == want).all(), "the frame differs from the plain pointer's"
    assert (b[:, 4 * w:] == SENT).all(), "the row pitch's padding was written"


def check_array(a, x0, y0, want):
    got = a.read()
    h, w = want.shape[:2]
    assert (got[y0:y0 + h, x0:x0 + w] == want).all(), "the frame differs from the plain pointer's"
    outside = np.ones((a.h, a.w), bool)
    outside[y0:y0 + h, x0:x0 + w] = False
    assert (got[outside] == SENT).all(), "a texel outside the frame was written"


SCENES = {
    "tiger_1000x517": lambda: (resolve(scenes.tiger(1000, 517).encoding), 1000, 517),
    "brushes": lambda: (lambda s, w, h: (resolve(s.encoding), w, h))(*scenes.brushes()),
    "blend_grid": lambda: (lambda s, w, h: (resolve(s.encoding), w, h))(*scenes.blend_grid()),
    "tiger_1x1": lambda: (resolve(scenes.tiger(1, 1).encoding), 1, 1),
    "tiger_17x33": lambda: (resolve(scenes.tiger(17, 33).encoding), 17, 33),
}


@pytest.fixture(scope="module")
def r():
    rr = Renderer()
    yield rr
    rr.close()


# ---- 1. every destination gives the plain pointer's bytes ------------------------------------------------------------------
@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_destinations_equal_plain_frames(r, scene, aa):
    packed, w, h = SCENES[scene]()
    r.upload(packed)
    p = RenderParams(Color(0.1, 0.2, 0.3, 1.0), w, h, aa)
    want = plain_frame(r, p)
    for pitch, fmt in ((4 * w + 52, "rgba8"), (4 * w + 64, "rgba8"), (4 * w + 64, "bgra8"), (4 * w, "bgra8")):
        big, view = pitched(h, w, pitch)
        key = r.register_destination(view, format=fmt)
        r.render_resident(p, key)
        check_linear(big, w, want if fmt == "rgba8" else bgra(want))
        r.unregister_destination(key)
    for (x0, y0, dw, dh, fmt) in ((0, 0, 0, 0, "rgba8"), (3, 17, 7, 40, "bgra8"), (4, 1, 4, 1, "rgba8")):
        a = Array(w + dw, h + dh)
        a.fill()
        key = r.register_destination(array=a.handle.value, format=fmt, origin=(x0, y0))
        r.render_resident(p, key)
        check_array(a, x0, y0, want if fmt == "rgba8" else bgra(want))
        r.unregister_destination(key)
        a.free()


# ---- 2. every entry point ----------------------------------------------------------------------------------------------------
def test_every_entry_point_into_an_array(r):
    packed, w, h = SCENES["tiger_1000x517"]()
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    r.upload(packed)
    want = plain_frame(r, p)
    a = Array(w, h)
    key = r.register_destination(array=a.handle.value)
    lib, ps, st = r.lib, _params_struct(p), FrameStats()

    def fresh():
        a.fill()

    fresh()
    r.enqueue(p, key)
    r.finish()
    check_array(a, 0, 0, want)
    fresh()
    assert lib.vb_render_uploaded(r.handle, C.byref(ps), C.c_void_p(key), 1, C.byref(st)) == 0
    check_array(a, 0, 0, want)
    fresh()
    scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    rc = lib.vb_render(r.handle, scene.ctypes.data, scene.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None, 512,
                       ramps.shape[0], atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), C.c_void_p(key), 1, C.byref(st))
    assert rc == 0
    check_array(a, 0, 0, want)
    fresh()
    r.run_stages(p, STAGES[0], STAGES[-1], key)
    check_array(a, 0, 0, want)
    # the native front end: vb_render_scene
    ns = NativeScene()
    ns.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 0.7), None, Rect(3, 5, 601, 400))
    ns.upload_device(r)
    want2 = plain_frame(r, p)
    fresh()
    assert ns.lib.vb_render_scene(r.handle, ns.handle, C.byref(ps), C.c_void_p(key), 1, C.byref(st)) == 0
    check_array(a, 0, 0, want2)
    r.unregister_destination(key)
    a.free()


# ---- 3. whole-frame graphs are keyed by the key ------------------------------------------------------------------------------
def test_graphs_follow_the_key():
    r = Renderer()
    packed, w, h = SCENES["tiger_1000x517"]()
    r.upload(packed)
    p = RenderParams(BLACK, w, h, AA_AREA)
    a, b = Array(w, h), Array(w, h)
    ka, kb = r.register_destination(array=a.handle.value), r.register_destination(array=b.handle.value, format="bgra8")
    r.render_resident(p, ka)
    n0 = r.debug_graph_captures()
    for _ in range(3):
        r.render_resident(p, ka)
    assert r.debug_graph_captures() == n0, "repeated frames into one key captured again"
    r.render_resident(p, kb)
    assert r.debug_graph_captures() == n0 + 1, "another key did not capture its own graph"
    r.render_resident(p, ka)
    assert r.debug_graph_captures() == n0 + 1, "coming back to the first key did not replay"
    want = plain_frame(r, p)
    assert (a.read() == want).all() and (b.read() == bgra(want)).all()
    for k in (ka, kb):
        r.unregister_destination(k)
    a.free()
    b.free()
    r.close()


def _bound_composition(r, w, h, n=64, seed=3):
    frag = NativeScene()
    frag.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 1.0), None, Rect(0, 0, 20, 14))
    fid = r.upload_fragment(frag)
    r.compose([(fid, None)] * n)
    rows = np.zeros((n, 6), np.float32)
    rows[:, 0] = rows[:, 3] = 1.0
    rows[:, 4:] = np.random.default_rng(seed).uniform([0, 0], [w - 20, h - 14], (n, 2))
    t = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    r.bind_instance_transforms(t)
    return t


def test_moving_bound_rows_into_an_array_replays():
    r = Renderer()
    w, h = 640, 480
    t = _bound_composition(r, w, h)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    a = Array(w, h)
    key = r.register_destination(array=a.handle.value)
    r.render_resident(p, key)
    n0 = r.debug_graph_captures()
    t[5, 4:] += 17.0
    torch.cuda.synchronize()
    r.render_resident(p, key)
    assert r.debug_graph_captures() == n0
    assert (a.read() == plain_frame(r, p)).all()
    r.unregister_destination(key)
    a.free()
    r.close()


# ---- 4. damage tracking into an array key ------------------------------------------------------------------------------------
def test_damage_tracking_into_an_array():
    r, ref = Renderer(), Renderer()
    w, h = 640, 480
    t, t_ref = _bound_composition(r, w, h), _bound_composition(ref, w, h)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    a = Array(w, h)
    key = r.register_destination(array=a.handle.value, format="bgra8")
    r.set_damage_tracking(True)
    r.render_resident(p, key)
    assert (a.read() == bgra(plain_frame(ref, p))).all()
    a.fill()  # a frame without damage writes nothing
    r.render_resident(p, key)
    assert not r.last_damage().any() and (a.read() == SENT).all()
    r.set_damage_tracking(True)  # full again
    r.render_resident(p, key)
    before = a.read()
    for tt in (t, t_ref):
        tt[9, 4:] += 23.0
    torch.cuda.synchronize()
    r.render_resident(p, key)
    want = bgra(plain_frame(ref, p))
    got = a.read()
    assert (got == want).all(), "the incremental frame differs from a full frame"
    dmg = r.last_damage()
    assert dmg.any() and dmg.sum() < dmg.size // 4
    changed = np.kron(dmg.astype(np.uint8), np.ones((16, 16), np.uint8)).astype(bool)[:h, :w]
    assert (got[~changed] == before[~changed]).all(), "a texel outside the damaged tiles changed"
    # upload diff: a re-upload of a scene with one rectangle moved is incremental into the key
    r.set_upload_diff(True)
    s0 = NativeScene()
    for k in range(20):
        s0.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.1 * (k % 10), 0.5, 0.3, 1.0), None, Rect(20 * k, 10, 20 * k + 15, 30))
    s0.upload_device(r)
    r.render_resident(p, key)
    s1 = NativeScene()
    for k in range(20):
        y = 200 if k == 7 else 10
        s1.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.1 * (k % 10), 0.5, 0.3, 1.0), None, Rect(20 * k, y, 20 * k + 15, y + 20))
    s1.upload_device(r)
    r.render_resident(p, key)
    dmg = r.last_damage()
    assert dmg.any() and not dmg.all(), "the upload-diffed frame into the key was not incremental"
    s1.upload_device(ref)
    ref.render_resident(p)
    assert (a.read() == bgra(ref.download_target(p))).all()
    r.set_upload_diff(False)
    r.set_damage_tracking(False)
    r.unregister_destination(key)
    a.free()
    r.close()
    ref.close()


def test_recompose_into_an_array_is_incremental():
    r, ref = Renderer(), Renderer()
    w, h = 512, 384
    p = RenderParams(BLACK, w, h, AA_AREA)
    frags = []
    for k in range(3):
        f = NativeScene()
        f.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.3 * k, 0.6, 0.2, 1.0), None, Rect(0, 0, 30, 20))
        frags.append(f)
    ids, rids = [r.upload_fragment(f) for f in frags], [ref.upload_fragment(f) for f in frags]
    inst = [(k % 3, Affine.translate(40 * k, 30 * (k % 5))) for k in range(12)]
    a = Array(w, h)
    key = r.register_destination(array=a.handle.value)
    r.set_damage_tracking(True)
    r.compose([(ids[i], tr) for i, tr in inst])
    r.render_resident(p, key)
    inst[4] = (2, Affine.translate(300, 300))
    r.recompose([(ids[i], tr) for i, tr in inst])
    r.render_resident(p, key)
    dmg = r.last_damage()
    assert dmg.any() and not dmg.all(), "the recomposed frame into the key was not incremental"
    ref.compose([(rids[i], tr) for i, tr in inst])
    assert (a.read() == plain_frame(ref, p)).all()
    r.unregister_destination(key)
    a.free()
    r.close()
    ref.close()


# ---- 5. a window writes its rows at their own rows ---------------------------------------------------------------------------
def test_window_writes_its_own_rows(r):
    packed, w, h = SCENES["tiger_1000x517"]()
    r.upload(packed)
    p = RenderParams(BLACK, w, h, AA_MSAA8)
    want = plain_frame(r, p)
    a = Array(w, h)
    a.fill()
    key = r.register_destination(array=a.handle.value)
    r.render_resident(p, key, tile_rows=(3, 9))
    got = a.read()
    assert (got[48:144] == want[48:144]).all()
    assert (got[:48] == SENT).all() and (got[144:] == SENT).all()
    big, view = pitched(h, w, 4 * w + 52)
    k2 = r.register_destination(view, format="bgra8")
    r.render_resident(p, k2, tile_rows=(3, 9))
    b = big.cpu().numpy()
    assert (b[48:144, :4 * w].reshape(96, w, 4) == bgra(want[48:144])).all()
    assert (b[:48] == SENT).all() and (b[144:] == SENT).all() and (b[:, 4 * w:] == SENT).all()
    r.unregister_destination(key)
    r.unregister_destination(k2)
    a.free()


# ---- 6, 7. arena overflow re-runs, and hit tests ----------------------------------------------------------------------------
def test_overflow_and_hit_tests(r):
    packed, w, h = SCENES["tiger_1000x517"]()
    r.upload(packed)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    want = plain_frame(r, p)
    g = np.random.default_rng(2)
    pts = np.stack([g.uniform(0, w, 500), g.uniform(0, h, 500)], axis=1).astype(np.float32)
    hits = r.hit_test(pts)
    a = Array(w, h)
    key = r.register_destination(array=a.handle.value, format="bgra8")
    r.limit_arena("segments", 1000)
    st = r.render_resident(p, key)
    assert st.retries >= 1
    assert (a.read() == bgra(want)).all()
    assert (r.hit_test(pts) == hits).all()
    r.unregister_destination(key)
    a.free()


# ---- 8. refusals -------------------------------------------------------------------------------------------------------------
def _refused(fn, *args, **kw):
    with pytest.raises(VelloB200Error) as e:
        fn(*args, **kw)
    return str(e.value)


def test_refusals(r):
    packed, w, h = SCENES["tiger_17x33"]()
    r.upload(packed)
    p = RenderParams(BLACK, w, h, AA_AREA)
    want = plain_frame(r, p)
    lib = r.lib
    bad_arrays = [Array(w, h, bits=(32, 32, 32, 32), kind=KIND_FLOAT), Array(w, h, bits=(8, 8, 0, 0)), Array(w, h, flags=0),
                  Array(w, h, layers=2)]
    for arr in bad_arrays:
        _refused(r.register_destination, None, array=arr.handle.value)
        assert lib.vb_last_error(r.handle)
        arr.free()
    with pytest.raises(ValueError):
        r.register_destination(array=1, format="argb")
    host = np.zeros((h, w, 4), np.uint8)

    class HostArray:  # a host pointer dressed as a device array
        __cuda_array_interface__ = {"shape": (h, w, 4), "typestr": "|u1", "data": (host.ctypes.data, False), "strides": None, "version": 3}

    _refused(r.register_destination, HostArray())
    big, view = pitched(h, w, 4 * w + 8)
    narrow = torch.as_strided(big, (h, w, 4), (4 * w - 4, 4, 1))
    k_narrow = r.register_destination(narrow)
    assert "pitch" in _refused(r.render_resident, p, k_narrow)
    small = Array(w + 2, h + 2)
    k_small = r.register_destination(array=small.handle.value, origin=(3, 0))
    assert "fit" in _refused(r.render_resident, p, k_small)
    k_ok = r.register_destination(array=small.handle.value, origin=(2, 2))
    # a batch into a destination
    r.set_cells([0, 3, r_n_draw(packed)])
    _refused(r.render_resident, p, k_ok)
    r.upload(packed)
    # another renderer's key, an unregistered one, a texture key
    other = Renderer()
    other.upload(packed)
    k_other = other.register_destination(array=small.handle.value, origin=(1, 1))
    _refused(r.render_resident, p, k_other)
    other.unregister_destination(k_other)
    _refused(other.render_resident, p, k_other)
    other.close()
    tex = torch.zeros((4, 4, 4), dtype=torch.uint8, device="cuda")
    img = r.register_texture(tex)
    tkey = img.key
    _refused(r.render_resident, p, tkey)
    _refused(r.unregister_destination, tkey)
    r.unregister_texture(img)
    _refused(r.unregister_texture, Image(np.zeros((4, 4, 4), np.uint8), key=k_ok))
    # a key where a host pointer or a plain device pointer is needed
    ps, st = _params_struct(p), FrameStats()
    assert lib.vb_render_uploaded(r.handle, C.byref(ps), C.c_void_p(k_ok), 0, C.byref(st)) == VB_E_INVALID
    assert lib.vb_copy_to_host(r.handle, C.c_void_p(k_ok), host.ctypes.data, 16) == VB_E_INVALID
    assert lib.vb_override_image(r.handle, C.c_void_p(1234), 4, 4, C.c_void_p(k_ok), 16) == VB_E_INVALID
    ns = NativeScene()
    ns.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 1.0), None, Rect(0, 0, 5, 5))
    assert ns.lib.vb_render_scene(r.handle, ns.handle, C.byref(ps), C.c_void_p(k_ok), 0, C.byref(st)) == VB_E_INVALID
    scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
    lay = _Layout(*[int(v) for v in packed.layout.as_array()])
    atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
    ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
    args = (scene.ctypes.data, scene.nbytes, C.byref(lay), ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
            atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps))
    assert lib.vb_render(r.handle, *args, C.c_void_p(k_ok), 0, C.byref(st)) == VB_E_INVALID
    assert lib.vb_render_begin(r.handle, *args, C.c_void_p(k_ok), C.byref(st)) == VB_E_INVALID
    # a destination key as an image key: the host resolve leaves its region zero, the device resolve refuses it, as for an
    # unregistered texture key
    im = NativeScene()
    im.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 1.0), None, Rect(0, 0, 5, 5))
    im.draw_image(Image(np.full((4, 4, 4), 200, np.uint8), key=k_ok), Affine.IDENTITY)
    assert (im.resolve().atlas == 0).all()
    with pytest.raises(ValueError):
        im.upload_device(r)
    assert b"texture" in lib.vb_last_error(r.handle)
    # the renderer still renders correctly
    r.upload(packed)
    r.render_resident(p, k_ok)
    got = small.read()
    assert (got[2:2 + h, 2:2 + w] == want).all()
    assert (plain_frame(r, p) == want).all()
    for k in (k_narrow, k_small, k_ok):
        r.unregister_destination(k)
    _refused(r.unregister_destination, k_ok)
    small.free()


def r_n_draw(packed):
    return int(packed.layout.n_draw_objects)


# ---- 9. unregistering waits for the frames enqueued into the key -------------------------------------------------------------
def test_unregister_after_enqueued_frame(r):
    packed, w, h = SCENES["tiger_1000x517"]()
    r.upload(packed)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    want = plain_frame(r, p)
    a = Array(w, h)
    a.fill()
    key = r.register_destination(array=a.handle.value)
    r.enqueue(p, key)
    r.unregister_destination(key)
    st = r.finish()
    assert st.failed == 0
    assert (a.read() == want).all()
    a.free()
