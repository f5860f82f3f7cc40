"""CPU-side checks of bound stroke widths (Renderer.bind_stroke_widths): the Python row checks, with a stub
`__cuda_array_interface__` and a stub library; the other bindings' messages; the snapshot kernel's resources; and the encoder
facts the GPU tests (test_gpu_stroke_widths.py) rely on, in both scene front ends."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import (FILL_NON_ZERO, STYLE_CAP_BUTT, STYLE_CAP_SQUARE, STYLE_FLAGS_STYLE_BIT, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER,
                                 TAG_PATH, TAG_STYLE, Color, Scene, Stroke, resolve)
from vello_b200.shapes import Affine, Circle, Rect

from .test_visibility import _Cai, _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")


def _renderer(lib=None):
    from vello_b200.renderer import Renderer
    return Renderer._borrowed(lib or _NoLib(), 1, owner=object())


# ---- the Python row checks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t, err", [
    (np.ones(4, np.float32), TypeError),              # host memory: no __cuda_array_interface__
    (_Cai((5, 2), "<f4"), ValueError),                # two columns
    (_Cai((), "<f4"), ValueError),                    # a scalar
    (_Cai((0,), "<f4"), ValueError),                  # no rows
    (_Cai((0, 1), "<f4"), ValueError),
    (_Cai((5,), "<f8"), ValueError),                  # float64
    (_Cai((5,), "<f2"), ValueError),                  # float16
    (_Cai((5,), "|u1"), ValueError),                  # uint8
    (_Cai((5,), "<f4", strides=(0,)), ValueError),    # every row the same float
    (_Cai((5,), "<f4", strides=(-4,)), ValueError),   # reversed
    (_Cai((5,), "<f4", strides=(6,)), ValueError),    # not a multiple of 4 bytes
    (_Cai((5, 1), "<f4", strides=(8, 2)), ValueError),
])
def test_python_checks_refuse_before_the_library(t, err):
    with pytest.raises(err):
        _renderer().bind_stroke_widths(t)


def test_python_messages():
    r = _renderer()
    with pytest.raises(TypeError) as e:
        r.bind_stroke_widths(np.ones(2, np.float32))
    assert str(e.value) == "ndarray has no __cuda_array_interface__: device widths are needed"
    with pytest.raises(ValueError) as e:
        r.bind_stroke_widths(_Cai((2, 3), "<f4"))
    assert str(e.value) == "bind_stroke_widths: widths must be (n,) or (n, 1) float32, not (2, 3) <f4"
    with pytest.raises(ValueError) as e:
        r.bind_stroke_widths(_Cai((4,), "<f4", strides=(6,)))
    assert str(e.value) == "bind_stroke_widths: columns 4 bytes apart and rows a multiple of 4 bytes, at least 4, apart; not strides (6, 4)"


def test_other_bindings_messages_are_unchanged():
    r = _renderer()
    for name, what, cols in [("bind_instance_transforms", "transforms", 6), ("bind_draw_colors", "colours", 4),
                             ("bind_path_points", "points", 2), ("bind_gradient_stops", "stops", 5), ("bind_transforms", "transforms", 6)]:
        with pytest.raises(TypeError) as e:
            getattr(r, name)(np.ones((2, cols), np.float32))
        assert str(e.value) == f"ndarray has no __cuda_array_interface__: device {what} are needed"
        with pytest.raises(ValueError) as e:
            getattr(r, name)(_Cai((3,), "<f4"))  # 1-D: only widths take a vector
        assert str(e.value) == f"{name}: {what} must be (n, {cols}) float32, not (3,) <f4"
        with pytest.raises(ValueError) as e:
            getattr(r, name)(_Cai((3, cols), "<f4", strides=(4 * cols + 2, 4)))
        assert str(e.value) == (f"{name}: columns 4 bytes apart and rows a multiple of 4 bytes, at least {4 * cols}, apart; "
                                f"not strides ({4 * cols + 2}, 4)")
    with pytest.raises(ValueError) as e:
        r.bind_draw_visibility(_Cai((2, 3)))
    assert str(e.value) == "bind_draw_visibility: flags must be (n,) bool or uint8, not (2, 3) |u1"


def test_python_accepts_vectors_columns_and_strided_rows():
    """A float32 vector, an (n, 1) array, or a column of a wider float32 state tensor reaches the library with its row pitch."""
    got = []

    class Lib:
        def vb_bind_stroke_widths(self, handle, ptr, n, pitch):
            got.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = _renderer(Lib())
    t = _Cai((7,), "<f4", strides=(40,))  # state[:, 5] of a (7, 10) float32 tensor
    r.bind_stroke_widths(t)
    assert got == [(1 << 20, 7, 40)] and r._widths is t
    r.bind_stroke_widths(_Cai((9,), "<f4"))  # contiguous: no strides
    assert got[-1] == (1 << 20, 9, 4)
    r.bind_stroke_widths(_Cai((9, 1), "<f4"))
    assert got[-1] == (1 << 20, 9, 4)
    r.bind_stroke_widths(_Cai((6, 1), "<f4", strides=(24, 4)))  # state[:, 2:3] of a (6, 6) tensor
    assert got[-1] == (1 << 20, 6, 24)
    r.bind_stroke_widths(_Cai((1,), "<f4", strides=(12,)))  # one row: its pitch is never used
    assert got[-1] == (1 << 20, 1, 4)
    r.bind_stroke_widths(None)
    assert got[-1] == (None, 0, 0) and r._widths is None


# ---- the snapshot kernel -----------------------------------------------------------------------------------------------------
needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@needs_cuobjdump
def test_snapshot_kernel_stays_in_registers(built):
    from .test_compiled_kernels import Usage, _key, _label
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, "k_widths.o")], capture_output=True, text=True, check=True).stdout
    fns = {_key(fn): Usage(*map(int, v)) for fn, *v in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)}
    assert sorted(map(_label, fns)) == ["k_stroke_widths"], sorted(map(_label, fns))
    for key, u in fns.items():
        assert u.stack == 0 and u.local == 0, f"{_label(key)}: {u.stack} bytes of stack, {u.local} bytes of local memory"


# ---- encoder facts -----------------------------------------------------------------------------------------------------------
def draw_styles(packed):
    """Per draw object (path k is draw object k), the style entry in effect at its path's end tag, as pathtag's path table
    gives it, and whether that entry is a stroke's."""
    L = packed.layout
    scene = np.asarray(packed.scene, dtype=np.uint32)
    tags = scene[L.path_tag_base:L.path_data_base].view(np.uint8)
    styles = scene[L.style_base:L.style_base + 2 * int((tags & TAG_STYLE != 0).sum())]
    entry, out = -1, []
    for t in tags:
        entry += 1 if t & TAG_STYLE else 0
        if t & TAG_PATH:
            out.append(entry)
    out = np.array(out, dtype=np.int64)
    assert len(out) == L.n_paths
    stroke = np.array([e >= 0 and (int(styles[2 * e]) & STYLE_FLAGS_STYLE_BIT) != 0 for e in out], dtype=bool)
    return out, stroke


def width_word(packed, entry):
    return np.asarray(packed.scene, dtype=np.uint32)[packed.layout.style_base + 2 * entry + 1].view(np.float32)


def stroke_ops(widths):
    """One stroke per width (the join follows the width), then a fill; every call encodes one draw object."""
    ops = []
    for i, w in enumerate(widths):
        s = Stroke(w, join=STYLE_JOIN_MITER if w > 4 else STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_SQUARE, end_cap=STYLE_CAP_BUTT)
        ops.append(lambda sc, i=i, s=s: sc.stroke(s, Affine.IDENTITY, Color(0.2, 0.3, 0.9, 1.0), None, Circle(30 + 20 * i, 40, 12)))
    ops.append(lambda sc: sc.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.9, 0.3, 0.1, 1.0), None, Rect(5, 5, 30, 30)))
    return ops


def front_ends():
    from vello_b200.scene_native import NativeScene
    return [("python", Scene, lambda s: resolve(s.encoding)), ("native", NativeScene, lambda s: s.resolve())]


@pytest.mark.parametrize("front", front_ends(), ids=lambda f: f[0])
def test_encoders_give_one_draw_object_per_stroke_and_share_equal_styles(front):
    _, make, packed_of = front
    widths = [3.0, 3.0, 5.0, 2.0, 2.0, 2.0, 7.5]
    s = make()
    for k, op in enumerate(stroke_ops(widths)):
        op(s)
        assert s.n_draw_objects == k + 1
    packed = packed_of(s)
    entry, stroke = draw_styles(packed)
    assert packed.layout.n_draw_objects == packed.layout.n_paths == len(widths) + 1
    assert stroke.tolist() == [True] * len(widths) + [False]
    # consecutive equal widths share one entry; a different width (or a fill between) starts another
    assert entry[0] == entry[1] and entry[3] == entry[4] == entry[5]
    assert len({entry[0], entry[2], entry[3], entry[6], entry[7]}) == 5
    assert [float(width_word(packed, e)) for e in entry[:-1]] == widths


@pytest.mark.parametrize("front", front_ends(), ids=lambda f: f[0])
def test_distinct_widths_give_distinct_entries(front):
    _, make, packed_of = front
    widths = [1.0 + 0.5 * k for k in range(9)]
    s = make()
    for op in stroke_ops(widths)[:-1]:
        op(s)
    # a dashed stroke is one draw object too: its dashes are subpaths of one path
    s.stroke(Stroke(11.0, dash_pattern=(6.0, 4.0)), Affine.IDENTITY, Color(0.1, 0.8, 0.2, 1.0), None, Circle(100, 100, 30))
    assert s.n_draw_objects == len(widths) + 1
    packed = packed_of(s)
    entry, stroke = draw_styles(packed)
    assert stroke.all() and len(set(entry.tolist())) == len(widths) + 1
    assert [float(width_word(packed, e)) for e in entry] == widths + [11.0]
