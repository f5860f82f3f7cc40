"""CPU-side checks of device-image support: the (H, W, 4) uint8 device-array check of Renderer.register_texture /
override_image, and images named by a key in both resolves (Python and native: identical bytes)."""
import numpy as np
import pytest

from vello_b200.encoding import FILL_NON_ZERO, Image, Scene, resolve
from vello_b200.renderer import _device_image
from vello_b200.shapes import Affine, Rect


class FakeDeviceArray:
    def __init__(self, shape, strides=None, typestr="|u1", ptr=0x7F0000001000):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": typestr, "data": (ptr, False), "version": 3}


def test_device_array_interface():
    assert _device_image(FakeDeviceArray((3, 5, 4))) == (0x7F0000001000, 3, 5, 20)
    assert _device_image(FakeDeviceArray((3, 5, 4), (36, 4, 1))) == (0x7F0000001000, 3, 5, 36)  # a column slice
    for bad in (FakeDeviceArray((3, 5, 3)), FakeDeviceArray((3, 5, 4), typestr="<f4"), FakeDeviceArray((3, 5, 4), (22, 4, 1)),
                FakeDeviceArray((3, 5, 4), (80, 16, 1)), FakeDeviceArray((15, 4))):
        with pytest.raises(ValueError):
            _device_image(bad)
    with pytest.raises(TypeError):
        _device_image(np.zeros((3, 5, 4), np.uint8))


def test_keyed_images_resolve_identically():
    """Images with a key share one atlas slot whatever their data object; a zero-strided image leaves its region zero."""
    from vello_b200.scene_native import NativeScene
    rng = np.random.default_rng(2)
    a = np.ascontiguousarray(rng.integers(1, 256, (7, 9, 4), dtype=np.uint8))
    keyed = Image(a, key=int(a.ctypes.data))
    same_key = Image(a.copy(), quality=2, key=keyed.key)  # a second Image of the same key
    plain = Image(rng.integers(1, 256, (4, 3, 4), dtype=np.uint8))
    zeros = Image(np.lib.stride_tricks.as_strided(np.zeros(4, np.uint8), shape=(6, 5, 4), strides=(0, 0, 1)))

    def draw(s):
        for i, im in enumerate((keyed, plain, same_key, zeros, keyed)):
            s.fill(FILL_NON_ZERO, Affine.translate(10.0 * i, 3.0), im, None, Rect(0, 0, 9, 9))
    py, nat = Scene(), NativeScene()
    draw(py)
    draw(nat)
    want, got = resolve(py.encoding), nat.resolve()
    assert got.scene.tobytes() == want.scene.tobytes()
    assert got.atlas.tobytes() == want.atlas.tobytes()
    assert want.atlas.shape == (7, 9 + 3 + 5, 4)  # three slots: keyed (shared), plain, zeros
    assert want.atlas[:6, 12:17].max() == 0


def test_short_lived_image_variants():
    """Sampler variants made on the fly (dataclasses.replace) and dropped right after drawing: each keeps its own sampler
    bits in the native scene, although Python may give a new Image the id of a dropped one."""
    import dataclasses
    from vello_b200.scene_native import NativeScene
    im = Image(np.random.default_rng(1).integers(0, 256, (6, 7, 4), dtype=np.uint8))

    def draw(s):
        for k in range(9):
            v = dataclasses.replace(im, quality=k % 3, x_extend=k // 3, y_extend=(k + 1) % 3)
            s.fill(FILL_NON_ZERO, Affine.translate(8.0 * k, 0.0), v, None, Rect(0, 0, 8, 8))
    py, nat = Scene(), NativeScene()
    draw(py)
    draw(nat)
    assert nat.resolve().scene.tobytes() == resolve(py.encoding).scene.tobytes()
