"""CPU-side checks of bound visibility (Renderer.bind_draw_visibility): the Python row checks, with a stub
`__cuda_array_interface__` and a stub library, and the snapshot kernel's resources. The frames are tested on the GPU in
test_gpu_visibility.py."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")


class _NoLib:
    """A library stub: the argument checks must refuse before any call reaches it."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


class _Cai:
    def __init__(self, shape, typestr="|u1", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "strides": strides, "data": (1 << 20, False),
                                         "version": 3}


@pytest.mark.parametrize("t, err", [
    (np.ones(4, np.uint8), TypeError),        # host memory: no __cuda_array_interface__
    (_Cai((5, 1)), ValueError),               # 2-D
    (_Cai(()), ValueError),                   # a scalar
    (_Cai((0,)), ValueError),                 # no rows
    (_Cai((5,), "<i4"), ValueError),          # int32
    (_Cai((5,), "<f4"), ValueError),          # float32
    (_Cai((5,), "|i1"), ValueError),          # int8
    (_Cai((5,), strides=(0,)), ValueError),   # every row the same byte
    (_Cai((5,), strides=(-1,)), ValueError),  # reversed
])
def test_python_checks_refuse_before_the_library(t, err):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(err):
        r.bind_draw_visibility(t)


def test_python_messages():
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(TypeError) as e:
        r.bind_draw_visibility(np.ones(2, np.uint8))
    assert str(e.value) == "ndarray has no __cuda_array_interface__: device flags are needed"
    with pytest.raises(ValueError) as e:
        r.bind_draw_visibility(_Cai((2, 3)))
    assert str(e.value) == "bind_draw_visibility: flags must be (n,) bool or uint8, not (2, 3) |u1"


def test_python_accepts_bool_uint8_and_strided_rows():
    """A bool or uint8 vector, or a column of a wider uint8 state tensor, reaches the library with its byte stride."""
    from vello_b200.renderer import Renderer
    got = []

    class Lib:
        def vb_bind_draw_visibility(self, handle, ptr, n, pitch):
            got.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = Renderer._borrowed(Lib(), 1, owner=object())
    t = _Cai((7,), strides=(10,))  # state[:, 3] of a (7, 10) uint8 tensor
    r.bind_draw_visibility(t)
    assert got == [(1 << 20, 7, 10)] and r._visibility is t
    r.bind_draw_visibility(_Cai((9,), "|b1"))  # bool, contiguous: no strides
    assert got[-1] == (1 << 20, 9, 1)
    r.bind_draw_visibility(_Cai((1,), strides=(5,)))  # one row: its pitch is never used
    assert got[-1] == (1 << 20, 1, 1)
    r.bind_draw_visibility(_Cai((4,), "<u1", strides=(4,)))
    assert got[-1] == (1 << 20, 4, 4)
    r.bind_draw_visibility(None)
    assert got[-1] == (None, 0, 0) and r._visibility is None


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@needs_cuobjdump
def test_snapshot_kernel_stays_in_registers(built):
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(BUILD, "k_visibility.o")], capture_output=True, text=True, check=True).stdout
    fns = dict((fn, (int(st), int(loc))) for fn, st, loc in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res))
    assert [re.match(r"_Z\d+(\w+?)P", fn).group(1) for fn in fns] == ["k_draw_visibility"], sorted(fns)
    for fn, (stack, local) in fns.items():
        assert stack == 0 and local == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
