"""Renderer.register_destination reads a linear destination from `__cuda_array_interface__` without torch (the conversion
device images use too): (pointer, height, width, row pitch). No GPU needed: the arrays here are fakes."""
import pytest

from vello_b200.renderer import _device_image


class Fake:
    def __init__(self, shape, strides=None, typestr="|u1", data=0x7000_0000):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (data, False), "strides": strides, "version": 3}


def test_contiguous():
    assert _device_image(Fake((517, 1000, 4))) == (0x7000_0000, 517, 1000, 4000)
    assert _device_image(Fake((1, 1, 4), strides=(4, 4, 1))) == (0x7000_0000, 1, 1, 4)


def test_rows_of_a_wider_buffer():
    # columns 16..16+300 of a (200, 1024, 4) buffer with 512-byte aligned rows of 4352 bytes
    base, pitch = 0x7000_0000, 4352
    assert _device_image(Fake((200, 300, 4), strides=(pitch, 4, 1), data=base + 16 * 4)) == (base + 64, 200, 300, pitch)
    # a pitch that is 4-byte aligned only (4w + 52)
    assert _device_image(Fake((33, 17, 4), strides=(4 * 17 + 52, 4, 1)))[3] == 120


@pytest.mark.parametrize("shape,strides,typestr", [
    ((10, 10, 4), None, "<f4"),          # wrong dtype
    ((10, 10, 4), None, "<u2"),
    ((10, 10, 3), None, "|u1"),          # wrong shape
    ((10, 40), None, "|u1"),
    ((10, 10, 4), (40, 8, 1), "|u1"),    # texels not 4 bytes apart
    ((10, 10, 4), (40, 4, 2), "|u1"),    # channels not 1 byte apart
    ((10, 10, 4), (42, 4, 1), "|u1"),    # rows not a multiple of 4 bytes apart
])
def test_refused(shape, strides, typestr):
    with pytest.raises(ValueError):
        _device_image(Fake(shape, strides, typestr))


def test_not_an_array():
    with pytest.raises(TypeError):
        _device_image(object())
