"""Bound draw colours without a GPU: the conversion the tests hold k_draw_data to is the encoder's, Renderer.bind_draw_colors
refuses what the library would refuse before calling it, and the compiled kernel rounds each step of its conversions on its
own (its registers: test_compiled_kernels.py)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import Color, FILL_NON_ZERO
from vello_b200.shapes import Affine, Rect

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")


def premul_np(rows):
    """`premultiply().to_rgba8().to_u32()` of float32 (n, 4) rows, in float32: p = (r a, g a, b a, a), then
    clamp(floor(p * 255 + 0.5), 0, 255) with the product and the sum rounded separately; r in the low byte."""
    rows = np.asarray(rows, dtype=np.float32)
    a = rows[:, 3]
    with np.errstate(over="ignore", invalid="ignore"):
        p = np.stack([rows[:, 0] * a, rows[:, 1] * a, rows[:, 2] * a, a], 1)
        v = np.floor(p * np.float32(255.0) + np.float32(0.5))
    v = np.where(v > 0, v, 0)
    v = np.minimum(v, 255).astype(np.uint32)
    return v[:, 0] | v[:, 1] << 8 | v[:, 2] << 16 | v[:, 3] << 24


def tie_rows():
    """Rows at the float32 neighbours (up to 2 ulp either side) of every (k + 0.5) / 255, under alpha 0, 1, tiny and at ties;
    values outside [0, 1], +-3e38 and -0.0."""
    f = np.float32
    ties = []
    for k in range(256):
        t = f((k + 0.5) / 255)
        for d in (-2, -1, 0, 1, 2):
            x = t
            for _ in range(abs(d)):
                x = np.nextafter(x, f(np.inf) if d > 0 else f(-np.inf), dtype=np.float32)
            ties.append(x)
    ties = np.array(ties, dtype=np.float32)
    n = len(ties)
    rows = [np.stack([ties, ties[::-1], np.roll(ties, 7), np.ones(n, np.float32)], 1),  # alpha 1: the ties themselves
            np.stack([np.ones(n, np.float32), ties, np.roll(ties, 3), ties], 1)]       # alpha at the ties
    odd = [0.0, -0.0, 1.0, 1e-30, 1.4e-45, 0.5, 2.0, -0.5, 3e38, -3e38, 255.5, 1.0000001]
    rows.append(np.array([[x, y, z, a] for a in odd for x, y, z in ((1.0, 0.5, 0.25), (3e38, -3e38, -0.0), (2.0, -1.0, 0.999))],
                         dtype=np.float32))
    return np.concatenate(rows)


def test_restatement_is_the_encoders_conversion():
    rows = tie_rows()
    with np.errstate(over="ignore"):
        p = np.concatenate([rows[:, :3] * rows[:, 3:], rows[:, 3:]], 1)
        finite = np.isfinite(p * np.float32(255)).all(1)
    assert finite.sum() > 2500 and (~finite).sum() > 0
    want = premul_np(rows)
    # the Python encoder (math.floor raises on inf, so rows whose products overflow are left to the restatement)
    for k in np.nonzero(finite)[0]:
        assert Color(*map(float, rows[k])).premul_rgba8_u32() == want[k], rows[k]
    # the native encoder, through a scene of one fill per row
    from vello_b200.scene_native import NativeScene
    s = NativeScene()
    for x in rows:
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(*map(float, x)), None, Rect(0, 0, 1, 1))
    packed = s.resolve()
    L = packed.layout
    assert np.array_equal(packed.scene[L.draw_data_base:L.transform_base], want)


def test_ties_are_ties():
    """The rows do sit on both sides of the rounding boundaries, so that a contracted multiply-add would show."""
    rows = tie_rows()
    words = premul_np(rows[:1280])
    r = words & 0xff
    assert len(np.unique(r)) == 256
    # at each tie the five neighbours straddle it: the middle three rows of every group of five hold two values
    groups = r.reshape(256, 5)
    assert (groups[:, 0] != groups[:, 4]).sum() > 200


class _NoLib:
    """A library stub: the argument checks must refuse before any call reaches it."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


class _Cai:
    def __init__(self, shape, typestr="<f4", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "strides": strides, "data": (1 << 20, False),
                                         "version": 3}


@pytest.mark.parametrize("t, err", [
    (np.zeros((4, 4), np.float32), TypeError),                 # host memory: no __cuda_array_interface__
    (_Cai((5, 3)), ValueError),                                # not 4 columns
    (_Cai((5, 4, 1)), ValueError),                             # not 2-D
    (_Cai((0, 4)), ValueError),                                # no rows
    (_Cai((5, 4), "<f8"), ValueError),                         # float64
    (_Cai((5, 4), "<f2"), ValueError),                         # float16
    (_Cai((5, 4), strides=(16, 8)), ValueError),               # columns not 4 bytes apart
    (_Cai((5, 4), strides=(4, 20)), ValueError),               # a transposed array
    (_Cai((5, 4), strides=(18, 4)), ValueError),               # a row pitch that is not a multiple of 4
    (_Cai((5, 4), strides=(12, 4)), ValueError),               # rows that overlap
])
def test_python_checks_refuse_before_the_library(t, err):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(err):
        r.bind_draw_colors(t)


def test_python_accepts_column_slices():
    """A column slice of a wider state tensor passes the checks and reaches the library with its row pitch."""
    from vello_b200.renderer import Renderer
    calls = []

    class Lib:
        def vb_bind_draw_colors(self, handle, ptr, n, pitch):
            calls.append((ptr.value, n, pitch))
            return 0

    r = Renderer._borrowed(Lib(), 1, owner=object())
    t = _Cai((7, 4), strides=(40, 4))
    r.bind_draw_colors(t)
    assert calls == [(1 << 20, 7, 40)] and r._colors is t
    r.bind_draw_colors(_Cai((1, 4), strides=(4, 4)))  # one row: its pitch is never used
    assert calls[-1] == (1 << 20, 1, 16)


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@needs_cuobjdump
def test_draw_data_conversions_have_no_fused_multiply_add(built):
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(built, "k_colors.o")], capture_output=True, text=True, check=True).stdout
    body = sass[sass.index("Function : _Z11k_draw_data"):]
    body = body[:body.index("..........")] if ".........." in body else body
    ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9.]+)", body)
    # a colour: three premultiplications and four scalings by 255, each its own rounding, floored and truncated per byte; an
    # image's alpha byte (bound opacity): one scaling by 255 and one + 0.5, each its own rounding, then a truncation
    assert ops.count("FRND.FLOOR") == 4 and ops.count("FMUL") == 8 and ops.count("FADD") == 5, ops
    assert sum(op.startswith("F2I") for op in ops) == 5, ops
    assert not any(op.startswith(("FFMA", "HFMA", "DFMA")) for op in ops), "the conversion contracts a multiply and an add"
