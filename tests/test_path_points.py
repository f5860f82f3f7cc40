"""Bound path points without a GPU: Scene.n_points counts the rows a call produced, equally in the Python and the native encoder;
Renderer.bind_path_points refuses what the library would refuse before calling it; the compiled kernels keep their data in
registers."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import (COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_MULTIPLY, STYLE_CAP_BUTT, STYLE_CAP_ROUND,
                                 STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Color, Scene, Stroke, resolve)
from vello_b200.shapes import Affine, Arc, BezPath, Circle, Ellipse, Line, Rect, RoundedRect

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
RED = Color(0.9, 0.2, 0.1, 1.0)


def path(*els):
    p = BezPath()
    p.els = list(els)
    return p


# one shape of every kind the encoders lay points out for: (name, shape)
SHAPES = [
    ("rect", Rect(10, 12, 70, 50)),
    ("rounded_rect", RoundedRect(5, 6, 90, 70, 12)),
    ("circle", Circle(50, 40, 30)),
    ("ellipse", Ellipse(60, 50, 40, 20, 0.3)),
    ("arc", Arc(50, 50, 30, 20, 0.2, 2.5, 0.1)),
    ("line", Line(3, 4, 80, 60)),
    ("quads_and_cubics", path(("M", 0, 0), ("Q", 20, 40, 60, 10), ("C", 70, 0, 90, 50, 40, 70), ("L", 10, 60))),
    ("repeated_move_to", path(("M", 1, 1), ("M", 5, 5), ("M", 10, 10), ("L", 40, 10), ("L", 40, 40))),
    ("closed_last_equals_first", path(("M", 10, 10), ("L", 50, 10), ("L", 50, 50), ("L", 10, 10), ("Z",))),
    ("closed_last_differs", path(("M", 10, 10), ("L", 50, 10), ("L", 50, 50), ("Z",))),
    ("open_last_differs", path(("M", 10, 10), ("L", 50, 10), ("L", 50, 50))),
    ("two_subpaths", path(("M", 0, 0), ("L", 30, 0), ("L", 30, 30), ("Z",), ("M", 40, 40), ("Q", 60, 40, 60, 60))),
    ("zero_length", path(("M", 5, 5), ("L", 5, 5), ("L", 30, 5), ("L", 30, 5))),
    ("empty", path()),
]
STROKES = [
    Stroke(4.0),
    Stroke(3.0, join=STYLE_JOIN_MITER, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_SQUARE),
    Stroke(2.5, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_SQUARE, end_cap=STYLE_CAP_ROUND),
    Stroke(2.0, join=STYLE_JOIN_ROUND, dash_pattern=(7.0, 3.0), dash_offset=1.5),
]


def calls():
    """(name, call(scene)): fills under both rules, strokes of every join, cap and a dash, and clip layers, of every shape."""
    out = []
    for name, shape in SHAPES:
        out.append((f"fill_{name}", lambda s, sh=shape: s.fill(FILL_NON_ZERO, Affine.translate(3, 2), RED, None, sh)))
        out.append((f"even_odd_{name}", lambda s, sh=shape: s.fill(FILL_EVEN_ODD, Affine.IDENTITY, RED, None, sh)))
        for j, st in enumerate(STROKES):
            out.append((f"stroke{j}_{name}", lambda s, sh=shape, st=st: s.stroke(st, Affine.rotate(0.1), RED, None, sh)))
    for name, shape in SHAPES[:4]:
        def layer(s, sh=shape):
            s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.7, Affine.IDENTITY, sh)
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, RED, None, Circle(40, 40, 20))
            s.pop_layer()
        out.append((f"layer_{name}", layer))
    return out


def _path_data(packed):
    L = packed.layout
    return packed.scene[L.path_data_base:L.draw_tag_base]


def test_n_points_counts_path_data_and_the_encoders_agree():
    from vello_b200.scene_native import NativeScene
    s, ns = Scene(), NativeScene()
    assert s.n_points == ns.n_points == 0
    kinds = set()
    for name, call in calls():
        a = s.n_points
        call(s)
        call(ns)
        assert s.n_points == ns.n_points, name
        assert s.n_points * 2 == len(s.encoding.path_data), name
        kinds.add(s.n_points - a > 0)
    assert kinds == {True, False}  # some calls (the empty path) add no point
    py, nat = resolve(s.encoding), ns.resolve()
    assert np.array_equal(_path_data(py), _path_data(nat))
    assert len(_path_data(py)) == 2 * s.n_points


@pytest.mark.parametrize("name, els, fill_points, stroke_points", [
    # a move-to is 1 point, a line-to 1; a closed fill adds its start point when the last one differs; a stroke ends a closed
    # subpath with a line-to (1 point) and an open one with a quad-to (2 points)
    ("triangle_open", [("M", 0, 0), ("L", 10, 0), ("L", 10, 10)], 4, 5),
    ("triangle_closed_equal", [("M", 0, 0), ("L", 10, 0), ("L", 10, 10), ("L", 0, 0), ("Z",)], 4, 5),
    ("triangle_closed_differs", [("M", 0, 0), ("L", 10, 0), ("L", 10, 10), ("Z",)], 4, 5),
    ("quad", [("M", 0, 0), ("Q", 10, 0, 10, 10)], 4, 5),
    ("cubic", [("M", 0, 0), ("C", 10, 0, 10, 10, 0, 10)], 5, 6),
    ("repeated_move_to", [("M", 3, 3), ("M", 0, 0), ("L", 10, 0)], 3, 4),
])
def test_point_layout(name, els, fill_points, stroke_points):
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, RED, None, path(*els))
    assert s.n_points == fill_points, name
    t = Scene()
    t.stroke(Stroke(1.0), Affine.IDENTITY, RED, None, path(*els))
    assert t.n_points == stroke_points, name


class _NoLib:
    """A library stub: the argument checks must refuse before any call reaches it."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


class _Cai:
    def __init__(self, shape, typestr="<f4", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "strides": strides, "data": (1 << 20, False),
                                         "version": 3}


@pytest.mark.parametrize("t, err", [
    (np.zeros((4, 2), np.float32), TypeError),                 # host memory: no __cuda_array_interface__
    (_Cai((5, 3)), ValueError),                                # not 2 columns
    (_Cai((5, 2, 1)), ValueError),                             # not 2-D
    (_Cai((10,)), ValueError),                                 # flat
    (_Cai((0, 2)), ValueError),                                # no rows
    (_Cai((5, 2), "<f8"), ValueError),                         # float64
    (_Cai((5, 2), "<f2"), ValueError),                         # float16
    (_Cai((5, 2), "<i4"), ValueError),                         # int32
    (_Cai((5, 2), strides=(16, 8)), ValueError),               # columns not 4 bytes apart
    (_Cai((5, 2), strides=(4, 20)), ValueError),               # a transposed array
    (_Cai((5, 2), strides=(10, 4)), ValueError),               # a row pitch that is not a multiple of 4
    (_Cai((5, 2), strides=(4, 4)), ValueError),                # rows that overlap
])
def test_python_checks_refuse_before_the_library(t, err):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(err):
        r.bind_path_points(t)


def test_python_accepts_column_slices():
    """A column slice of a wider state tensor passes the checks and reaches the library with its row pitch."""
    from vello_b200.renderer import Renderer
    got = []

    class Lib:
        def vb_bind_path_points(self, handle, ptr, n, pitch):
            got.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = Renderer._borrowed(Lib(), 1, owner=object())
    t = _Cai((7, 2), strides=(24, 4))  # state[:, 4:6] of a (7, 6) float32 tensor
    r.bind_path_points(t)
    assert got == [(1 << 20, 7, 24)] and r._points is t
    r.bind_path_points(_Cai((1, 2), strides=(4, 4)))  # one row: its pitch is never used
    assert got[-1] == (1 << 20, 1, 8)
    r.bind_path_points(_Cai((3, 2)))  # contiguous: no strides
    assert got[-1] == (1 << 20, 3, 8)
    r.bind_path_points(None)
    assert got[-1] == (None, 0, 0) and r._points is None


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@needs_cuobjdump
def test_point_kernels_stay_in_registers(built):
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, "k_points.o")], capture_output=True, text=True, check=True).stdout
    fns = dict((fn, (int(st), int(loc))) for fn, st, loc in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res))
    names = sorted(re.match(r"_Z\d+(\w+?)P", fn).group(1) for fn in fns)
    assert names == ["k_path_point_slots", "k_path_points"], names
    for fn, (stack, local) in fns.items():
        assert stack == 0 and local == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"


@needs_cuobjdump
def test_damage_kernels_stay_in_registers(built):
    """k_damage_mark compares the bound points beside the transforms."""
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, "k_damage.o")], capture_output=True, text=True, check=True).stdout
    fns = dict((fn, (int(st), int(loc))) for fn, st, loc in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res))
    assert any("k_damage_mark" in fn for fn in fns), sorted(fns)
    for fn, (stack, local) in fns.items():
        assert stack == 0 and local == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"


def test_an_empty_clip_adds_the_empty_path():
    """A fill of a shape that encodes nothing adds no point; a layer whose clip encodes nothing adds the 2 points of the empty
    path that stands in for the clip, in both encoders."""
    from vello_b200.scene_native import NativeScene
    for s in (Scene(), NativeScene()):
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, RED, None, path())
        assert s.n_points == 0 and s.n_draw_objects == 0
        s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, path())
        assert s.n_points == 2 and s.n_draw_objects == 1
        s.pop_layer()
        assert s.n_points == 2
        pd = _path_data(resolve(s.encoding) if isinstance(s, Scene) else s.resolve())
        assert np.array_equal(pd.view(np.float32), np.zeros(4, np.float32))
