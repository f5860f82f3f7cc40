"""The paint edge cases of test_paint_ref.py on the GPU, and the atlas's 16-bit place limit on every resolve path.

Each paint case renders in area AA and MSAA16 and is checked stage by stage against the oracle (`compare_all`), pixel for
pixel against the oracle's fine replayed on the GPU's buffers (`assert_replay`), and against the float64 reference
(test_paint_ref.check_pixels). Ramps: the device resolve's ramp equals the host resolve's byte for byte, and both are within
1 LSB of the reference ramp."""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import FILL_NON_ZERO, TRANSPARENT, Image, Scene, resolve
from vello_b200.shapes import Affine, Rect

from . import paint_ref as P
from . import parity
from .test_paint_ref import CASES, RAMP_CASES, check_pixels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_paint_edges(renderer, oracle, case, aa):
    packed = resolve(case.scene().encoding)
    img = renderer.render_to_texture(packed, RenderParams(TRANSPARENT, case.w, case.h, aa))
    oracle.render(packed, case.w, case.h, 0, aa)  # compare_all reads the oracle's buffers of this scene
    # nan_info: the paint's info words hold NaNs (p0 == p1), whose payload the GPU and the host compiler produce differently
    parity.compare_all(renderer, oracle, packed.layout, case.w, case.h, info_nan=case.nan_info)
    parity.assert_replay(renderer, oracle, packed, img, case.w, case.h, aa, TRANSPARENT)
    check_pixels(case, img, packed.ramps)


@pytest.mark.parametrize("case", RAMP_CASES, ids=[c.name for c in RAMP_CASES])
def test_device_ramps(renderer, case):
    """k_make_ramps (device resolve) == the native host resolve byte for byte, both within 1 LSB of the float64 ramp."""
    from vello_b200.encoding import Gradient
    from vello_b200.scene_native import NativeScene
    ns = NativeScene()
    g = Gradient(case.kind, tuple(case.params), list(case.stops), case.extend, case.premul)
    ns.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), g, None, Rect(0, 0, case.w, case.h))
    host = ns.resolve().ramps
    ns.upload_device(renderer)
    dev = renderer.download("ramps", np.uint32)[: host.size].reshape(host.shape)
    assert np.array_equal(dev, host), "device ramps differ from the host resolve's"
    want = P.ramp([(o, (c.r, c.g, c.b, c.a)) for o, c in case.stops], case.premul).astype(np.int32)
    got = np.ascontiguousarray(host[0]).view(np.uint8).reshape(-1, 4).astype(np.int32)
    assert np.abs(got - want).max() <= 1


# ---- the atlas's 16-bit places ------------------------------------------------------------------------------------------------
def _tall_then(width2):
    """A 1 x 65535 image, then a width2 x 1 image: the second starts a new shelf at y = 65535 when width2 > 2047."""
    tall = Image(np.broadcast_to(np.array([9, 8, 7, 255], np.uint8), (65535, 1, 4)))
    rng = np.random.default_rng(7)
    low = Image(rng.integers(0, 256, size=(1, width2, 4), dtype=np.uint8), quality=0)
    return tall, low


def test_image_at_row_65535_renders(renderer, oracle):
    """An image placed at y = 65535 (the last row a place can hold) renders from its own texels. The atlas is 2048 x 65536
    texels: about 0.5 GB of host memory for the resolve and as much device memory for the frame."""
    tall, low = _tall_then(2048)
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), tall, None, Rect(-8, -8, -4, -4))
    m = (0.125, 0.0, 0.0, 16.0, 0.0, 0.0)  # 2048 texels over 256 pixels, the one row over 16
    s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), low, Affine(m), Rect(0, 0, 256, 16))
    packed = resolve(s.encoding)
    assert packed.atlas.shape[:2] == (65536, 2048)
    img = renderer.render_to_texture(packed, RenderParams(TRANSPARENT, 256, 16, AA_AREA))
    x, y = P.centre_grid(256, 16)
    ref = P.image_sample(low.data, x, y, m, quality=0)
    assert np.abs(img.astype(np.float64) - P.stored(ref)).max() <= 1.0


def test_places_past_row_65535_are_refused_on_the_device(renderer):
    """The device resolve, fragment upload, compose, recompose and register_texture refuse a place past row 65535 or a side
    over 65535, with the renderer's last error set, and leave the renderer's scene as it was: the same frame renders
    afterwards."""
    import torch
    from vello_b200.renderer import VelloB200Error
    from vello_b200.scene_native import NativeScene
    tall, low = _tall_then(2048)
    second = Image(np.zeros((1, 2048, 4), np.uint8))

    def build(s):
        s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), tall, None, Rect(-8, -8, -4, -4))
        s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), low, None, Rect(0, 0, 8, 8))
        s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), second, None, Rect(0, 0, 8, 8))  # a new shelf at y = 65536
        return s

    known = Scene()
    rng = np.random.default_rng(11)
    known.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), Image(rng.integers(0, 256, size=(5, 7, 4), dtype=np.uint8)),
               Affine.scale(3.0), Rect(0, 0, 21, 15))
    params = RenderParams(TRANSPARENT, 32, 32, AA_AREA)
    before = renderer.render_to_texture(resolve(known.encoding), params)
    assert before.any()

    def last_error():
        return renderer.lib.vb_last_error(renderer.handle).decode()

    ns = build(NativeScene())
    with pytest.raises(ValueError):
        ns.upload_device(renderer)
    assert "65535" in last_error()
    wide = NativeScene()
    wide.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), Image(np.zeros((1, 65536, 4), np.uint8)), None, Rect(0, 0, 8, 8))
    with pytest.raises(ValueError):
        wide.upload_device(renderer)
    assert "65535" in last_error()
    with pytest.raises(VelloB200Error, match="65535"):
        renderer.upload_fragment(wide)
    f1 = renderer.upload_fragment(build(Scene()))
    with pytest.raises(VelloB200Error, match="65535"):
        renderer.compose([(f1, None)])
    with pytest.raises(VelloB200Error, match="65535"):
        renderer.recompose([(f1, None)])
    renderer.free_fragment(f1)
    t = torch.zeros((1, 65536, 4), dtype=torch.uint8, device="cuda")
    with pytest.raises(VelloB200Error, match="65535"):
        renderer.register_texture(t)
    renderer.render_resident(params)
    after = renderer.download_target(params)
    assert np.array_equal(after, before), "a refused call changed the renderer's scene"
