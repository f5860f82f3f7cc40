"""Bound transforms without a GPU: Scene.n_transforms counts the transform-stream entries a call produced, equally in the Python
and the native encoder; each path's transform range [t_lo, t_hi], restated from the tag bytes, is the one the encoder's own calls
give; Renderer.bind_transforms refuses what the library would refuse before calling it, with the same messages as the other
bindings; the new kernel copies bits only and keeps everything in registers."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import (COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_MULTIPLY, STYLE_CAP_ROUND, STYLE_JOIN_BEVEL, Color,
                                 Gradient, Image, Scene, Stroke, resolve)
from vello_b200.shapes import Affine, BezPath, Circle, Rect, RoundedRect

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
IMG = np.random.default_rng(3).integers(0, 256, (6, 5, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]


def path(*els):
    p = BezPath()
    p.els = list(els)
    return p


def random_calls(seed):
    """(call(scene)) of fills, strokes, layers, images, blurred rectangles and shapes that encode nothing, with transforms that
    often repeat (shared entries) and brush transforms."""
    g = np.random.default_rng(seed)
    xfs = [Affine.IDENTITY, Affine.translate(3, 2), Affine.rotate(0.2) * Affine.scale(1.5), Affine.translate(-4, 9)]
    shapes = [Rect(1, 2, 30, 40), Circle(20, 20, 9), RoundedRect(0, 0, 20, 10, 3), path(("M", 0, 0), ("L", 10, 5), ("L", 3, 9)),
              path()]
    brushes = [Color(0.2, 0.4, 0.6, 1.0), Gradient.linear((0, 0), (10, 5), STOPS), Gradient.radial((5, 5), 1.0, (5, 5), 8.0, STOPS),
               Gradient.sweep((5, 5), 0.0, 3.0, STOPS), Image(IMG)]

    def pick(xs):
        return xs[int(g.integers(len(xs)))]

    calls, depth = [], 0
    for _ in range(40):
        k = int(g.integers(7))
        t, sh, br = pick(xfs), pick(shapes), pick(brushes)
        bt = pick([None, None, Affine.scale(0.5), Affine.translate(1, 1), Affine.IDENTITY])
        if k == 0:
            calls.append(lambda s, t=t, sh=sh, br=br, bt=bt: s.fill(FILL_NON_ZERO, t, br, bt, sh))
        elif k == 1:
            calls.append(lambda s, t=t, sh=sh, br=br, bt=bt: s.fill(FILL_EVEN_ODD, t, br, bt, sh))
        elif k == 2:
            st = pick([Stroke(2.0), Stroke(0.0), Stroke(3.0, join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_ROUND, end_cap=STYLE_CAP_ROUND),
                       Stroke(1.5, dash_pattern=(4.0, 2.0))])
            calls.append(lambda s, t=t, sh=sh, br=br, bt=bt, st=st: s.stroke(st, t, br, bt, sh))
        elif k == 3:
            calls.append(lambda s, t=t: s.draw_image(Image(IMG), t))
        elif k == 4:
            calls.append(lambda s, t=t: s.draw_blurred_rounded_rect(t, Rect(2, 3, 20, 15), Color(0.9, 0.1, 0.2, 0.8), 3.0, 2.0))
        elif k == 5 and depth < 3:
            clip = pick([sh, Stroke(2.0)])
            if isinstance(clip, Stroke):
                calls.append(lambda s, t=t, sh=sh: s.push_layer(Stroke(2.0), MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.7, t, sh))
            else:
                calls.append(lambda s, t=t, sh=sh: s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.7, t, sh))
            depth += 1
        elif depth > 0:
            calls.append(lambda s: s.pop_layer())
            depth -= 1
    calls += [lambda s: s.pop_layer()] * depth
    return calls


@pytest.mark.parametrize("seed", range(6))
def test_n_transforms_counts_the_stream_and_the_encoders_agree(seed):
    from vello_b200.scene_native import NativeScene
    s, ns = Scene(), NativeScene()
    assert s.n_transforms == ns.n_transforms == 0
    for call in random_calls(seed):
        call(s)
        call(ns)
        assert s.n_transforms == ns.n_transforms == len(s.encoding.transforms)
    # append, with and without a transform, of a scene built the same way
    other, nother = Scene(), NativeScene()
    for call in random_calls(seed + 100):
        call(other)
        call(nother)
    s.append(other, Affine.translate(5, 5))
    ns.append(nother, Affine.translate(5, 5))
    assert s.n_transforms == ns.n_transforms
    s.append(other)
    ns.append(nother)
    assert s.n_transforms == ns.n_transforms
    py, nat = resolve(s.encoding), ns.resolve()
    L = py.layout
    assert (L.style_base - L.transform_base) // 6 == s.n_transforms
    assert np.array_equal(py.scene[L.transform_base:L.style_base], nat.scene[nat.layout.transform_base:nat.layout.style_base])


def test_shared_entries_brush_transforms_and_empty_shapes():
    s = Scene()
    red = Color(1, 0, 0, 1)
    s.fill(FILL_NON_ZERO, Affine.translate(1, 2), red, None, Rect(0, 0, 5, 5))
    s.fill(FILL_NON_ZERO, Affine.translate(1, 2), red, None, Circle(3, 3, 2))  # the same transform: one shared entry
    assert s.n_transforms == 1
    s.fill(FILL_NON_ZERO, Affine.translate(1, 2), Gradient.linear((0, 0), (5, 0), STOPS), Affine.scale(2.0), Rect(0, 0, 5, 5))
    assert s.n_transforms == 2  # the brush transform, transform * brush_transform, is an entry of its own
    assert s.encoding.transforms[-1] == tuple(np.float32(v) for v in (Affine.translate(1, 2) * Affine.scale(2.0)).coeffs)
    s.fill(FILL_NON_ZERO, Affine.translate(7, 7), red, None, path())  # encodes nothing, still pushes its transform
    assert s.n_transforms == 3 and s.n_draw_objects == 3
    s.stroke(Stroke(0.0), Affine.translate(9, 9), red, None, Rect(0, 0, 5, 5))  # a stroke of width 0 pushes nothing
    assert s.n_transforms == 3
    s.draw_image(Image(IMG), Affine.translate(8, 8))  # one entry places the rectangle and the image
    assert s.n_transforms == 4


class Recording:
    """A Scene that notes, for every draw object a call adds, the transform in effect after the call's first and last
    encode_transform (the geometry's and the brush's): the encoder's own account of each path's [t_lo, t_hi]."""

    def __init__(self):
        self.scene = Scene()
        self.ranges = {}
        self._seen = []
        enc = self.scene.encoding
        push = enc.encode_transform

        def encode_transform(t):
            r = push(t)
            self._seen.append(len(enc.transforms) - 1)
            return r
        enc.encode_transform = encode_transform

    def __getattr__(self, name):
        f = getattr(self.scene, name)
        if not callable(f):
            return f

        def call(*a, **k):
            d = self.scene.n_draw_objects
            self._seen = []
            f(*a, **k)
            if self.scene.n_draw_objects > d:
                assert self.scene.n_draw_objects == d + 1
                now = len(self.scene.encoding.transforms) - 1
                self.ranges[d] = (self._seen[0], self._seen[-1]) if self._seen else (now, now)
        return call


def transform_ranges(packed):
    """[t_lo, t_hi] of every path from the tag bytes: the transform in effect at a byte is the TRANSFORM bytes before it minus 1;
    t_lo is the one at the path's first segment byte, t_hi the one at its TAG_PATH (t_hi for a path without a segment)."""
    L = packed.layout
    tags = packed.scene[L.path_tag_base:L.path_data_base].view(np.uint8)
    out, t, lo = [], -1, None
    for b in tags.tolist():
        if b & 3 and lo is None:
            lo = t
        if b & 0x10:
            out.append((t if lo is None else lo, t))
            lo = None
        if b & 0x20:
            t += 1
    return out[:L.n_paths]


@pytest.mark.parametrize("seed", range(6))
def test_transform_ranges_from_the_tags_equal_the_encoder_calls(seed):
    rec = Recording()
    for call in random_calls(seed):
        call(rec)
    got = transform_ranges(resolve(rec.scene.encoding))
    assert len(got) == rec.scene.n_draw_objects == len(rec.ranges)  # path d is draw object d
    assert got == [rec.ranges[d] for d in range(len(got))]
    assert any(lo < hi for lo, hi in got)  # brush transforms widen some ranges


class _NoLib:
    """A library stub: the argument checks must refuse before any call reaches it."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


class _Cai:
    def __init__(self, shape, typestr="<f4", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "strides": strides, "data": (1 << 20, False),
                                         "version": 3}


@pytest.mark.parametrize("t, err", [
    (np.zeros((4, 6), np.float32), TypeError),                 # host memory: no __cuda_array_interface__
    (_Cai((5, 4)), ValueError),                                # not 6 columns
    (_Cai((5, 6, 1)), ValueError),                             # not 2-D
    (_Cai((36,)), ValueError),                                 # flat
    (_Cai((0, 6)), ValueError),                                # no rows
    (_Cai((5, 6), "<f8"), ValueError),                         # float64
    (_Cai((5, 6), "<f2"), ValueError),                         # float16
    (_Cai((5, 6), "<i4"), ValueError),                         # int32
    (_Cai((5, 6), strides=(48, 8)), ValueError),               # columns not 4 bytes apart
    (_Cai((5, 6), strides=(4, 20)), ValueError),               # a transposed array
    (_Cai((5, 6), strides=(26, 4)), ValueError),               # a row pitch that is not a multiple of 4
    (_Cai((5, 6), strides=(20, 4)), ValueError),               # rows that overlap
])
def test_python_checks_refuse_before_the_library(t, err):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(err):
        r.bind_transforms(t)


def test_python_accepts_column_slices():
    """A column slice of a wider state tensor passes the checks and reaches the library with its row pitch."""
    from vello_b200.renderer import Renderer
    got = []

    class Lib:
        def vb_bind_transforms(self, handle, ptr, n, pitch):
            got.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = Renderer._borrowed(Lib(), 1, owner=object())
    t = _Cai((7, 6), strides=(40, 4))  # state[:, 2:8] of a (7, 10) float32 tensor
    r.bind_transforms(t)
    assert got == [(1 << 20, 7, 40)] and r._xforms is t
    r.bind_transforms(_Cai((1, 6), strides=(4, 4)))  # one row: its pitch is never used
    assert got[-1] == (1 << 20, 1, 24)
    r.bind_transforms(_Cai((3, 6)))  # contiguous: no strides
    assert got[-1] == (1 << 20, 3, 24)
    r.bind_transforms(None)
    assert got[-1] == (None, 0, 0) and r._xforms is None


# the five bindings share one parser of device rows; each keeps its own messages
MESSAGES = [
    ("bind_instance_transforms", 6, "transforms"),
    ("bind_draw_colors", 4, "colours"),
    ("bind_path_points", 2, "points"),
    ("bind_gradient_stops", 5, "stops"),
    ("bind_transforms", 6, "transforms"),
]


@pytest.mark.parametrize("method, cols, what", MESSAGES)
def test_every_binding_keeps_its_messages(method, cols, what):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    bind = getattr(r, method)
    with pytest.raises(TypeError) as e:
        bind(np.zeros((2, cols), np.float32))
    assert str(e.value) == f"ndarray has no __cuda_array_interface__: device {what} are needed"
    with pytest.raises(ValueError) as e:
        bind(_Cai((2, cols + 1)))
    assert str(e.value) == f"{method}: {what} must be (n, {cols}) float32, not (2, {cols + 1}) <f4"
    with pytest.raises(ValueError) as e:
        bind(_Cai((2, cols), strides=(4 * cols - 4, 4)))
    assert str(e.value) == (f"{method}: columns 4 bytes apart and rows a multiple of 4 bytes, at least {4 * cols}, apart; "
                            f"not strides ({4 * cols - 4}, 4)")


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


def _usage(obj):
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(BUILD, obj)], capture_output=True, text=True, check=True).stdout
    return dict((fn, (int(st), int(loc))) for fn, st, loc in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res))


@needs_cuobjdump
def test_bound_transforms_kernel_stays_in_registers_and_copies_bits(built):
    fns = _usage("k_transforms.o")
    assert [re.match(r"_Z\d+(\w+?)P", fn).group(1) for fn in fns] == ["k_bound_transforms"], sorted(fns)
    for fn, (stack, local) in fns.items():
        assert stack == 0 and local == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(BUILD, "k_transforms.o")], capture_output=True, text=True, check=True).stdout
    ops = set(re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", sass))
    assert "LDG" in ops and "STG" in ops, sorted(ops)
    floating = {op for op in ops if op.startswith(("F", "H", "D", "MUFU"))}  # FFMA, FADD, FMUL, FSETP, HADD2, DFMA, MUFU ...
    assert not floating, f"k_bound_transforms does float arithmetic: {sorted(floating)}"
    assert "LDL" not in ops and "STL" not in ops


@needs_cuobjdump
def test_tag_walk_and_damage_kernels_stay_in_registers(built):
    """k_path_point_slots also finds the transform ranges; k_damage_mark and k_damage also follow the transforms."""
    for obj in ("k_points.o", "k_damage.o"):
        for fn, (stack, local) in _usage(obj).items():
            assert stack == 0 and local == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
