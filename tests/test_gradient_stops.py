"""Bound gradient stops without a GPU: both encoders count the rows vb_bind_gradient_stops reads alike, the ramp walk the tests
hold k_bound_ramps to is the encoders' make_ramp at its edges, Renderer.bind_gradient_stops refuses what the library would
refuse before calling it, and the compiled kernels keep their data in registers and their arithmetic unfused."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import COMPOSE_SRC_OVER, MIX_MULTIPLY, Color, FILL_NON_ZERO, Gradient, Scene, Stroke, batch, make_ramp
from vello_b200.shapes import Affine, Rect

from .test_draw_colors import _Cai, _NoLib, premul_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
f32 = np.float32


def ramp_np(stops, premul):
    """make_ramp (vb_scene.cpp, encoding.make_ramp) of float32 (n, 5) offset r g b a rows, every product, sum and quotient
    rounded to float32 on its own: 512 premultiplied RGBA8 words."""
    st = np.asarray(stops, dtype=f32)
    out = np.zeros((512, 4), dtype=f32)
    for i in range(512):
        u = f32(i) / f32(511)
        last_u = this_u = f32(0)
        last = this = st[0, 1:]
        j = 0
        while u > this_u:
            last_u, last = this_u, this
            if j + 1 < len(st):
                this_u, this = st[j + 1, 0], st[j + 1, 1:]
                j += 1
            else:
                break
        du = f32(this_u - last_u)
        if du < f32(1e-9):
            c = this
        else:
            t = f32((u - last_u) / du)
            if premul:
                pa = np.array([last[0] * last[3], last[1] * last[3], last[2] * last[3], last[3]], dtype=f32)
                pb = np.array([this[0] * this[3], this[1] * this[3], this[2] * this[3], this[3]], dtype=f32)
                pc = (pa + ((pb - pa) * t).astype(f32)).astype(f32)
                if pc[3] == 0 or pc[3] == 1:
                    c = pc
                else:
                    inv = f32(1) / pc[3]
                    c = np.array([pc[0] * inv, pc[1] * inv, pc[2] * inv, pc[3]], dtype=f32)
            else:
                c = (last + ((this - last) * t).astype(f32)).astype(f32)
        out[i] = c
    return premul_np(out)


def edge_ramps():
    """(stops, premul) at make_ramp's edges: du below 1e-9, equal and out-of-order offsets, offsets outside [0, 1], alpha 0,
    1 and tiny under premultiplied interpolation, and colours on the .5 rounding ties."""
    tie = [f32((k + 0.5) / 255) for k in (0, 77, 128, 254)]
    cases = [
        [[0.0, 1, 0, 0, 1], [1e-10, 0, 1, 0, 1], [1.0, 0, 0, 1, 1]],                  # du < 1e-9
        [[0.3, 1, 0, 0, 1], [0.3, 0, 1, 0, 0.5], [0.3, 0, 0, 1, 1], [0.9, 1, 1, 1, 1]],  # equal offsets
        [[0.8, 1, 0.5, 0, 1], [0.2, 0, 1, 0.5, 0.7], [0.6, 0.2, 0.2, 1, 1]],          # out of order
        [[-0.5, 1, 0, 0, 1], [1.5, 0, 0, 1, 0.25]],                                   # outside [0, 1]
        [[0.0, 1, 0.2, 0.3, 0.0], [0.5, 0.1, 0.9, 0.4, 1.0], [1.0, 0.7, 0.7, 0.1, 1e-30]],  # alpha 0, 1, tiny
        [[0.0, tie[0], tie[1], tie[2], 1.0], [1.0, tie[3], tie[2], tie[1], 1.0]],     # the ties
        [[0.1, 0.25, 0.5, 0.75, 1.0 / 3.0], [0.1, 0.9, 0.1, 0.2, 0.6], [0.95, 0.0, 0.0, 0.0, 0.0]],
    ]
    return [(np.array(c, dtype=f32), premul) for c in cases for premul in (True, False)]


@pytest.mark.parametrize("k", range(len(edge_ramps())))
def test_restatement_is_make_ramp(k):
    stops, premul = edge_ramps()[k]
    want = ramp_np(stops, premul)
    pairs = [(float(s[0]), Color(*map(float, s[1:]))) for s in stops]
    assert np.array_equal(make_ramp(pairs, premul), want)
    # the native host resolve: one gradient, one ramp
    from vello_b200.scene_native import NativeScene
    s = NativeScene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (10, 0), pairs, premul_interp=premul), None, Rect(0, 0, 10, 10))
    packed = s.resolve()
    assert packed.ramps.shape[0] == 1
    assert np.array_equal(packed.ramps[0], want)


STOPS3 = [(0.0, Color(1, 0, 0, 1)), (0.4, Color(0, 1, 0, 0.5)), (1.0, Color(0, 0, 1, 1))]
STOPS2 = [(0.2, Color(0.5, 0.5, 0.1, 1)), (0.7, Color(0.2, 0.1, 0.9, 0.8))]


def stop_scene(cls, with_layer=True):
    """Linear, radial and sweep gradients in both alpha spaces, the gradients that encode a colour (no stop, one stop,
    degenerate radial and sweep), a solid fill and a gradient stroke in a blend layer."""
    s = cls()
    r = Rect(0, 0, 20, 20)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (20, 0), STOPS3), None, r)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.radial((5, 5), 1.0, (10, 10), 9.0, STOPS2), None, r)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.sweep((10, 10), 0.0, 4.0, STOPS3, premul_interp=False), None, r)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (20, 0), STOPS2[:1]), None, r)        # one stop: a colour
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (20, 0), []), None, r)                # no stop: a colour
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.radial((5, 5), 3.0, (5, 5), 3.0, STOPS3), None, r)   # degenerate radial
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.sweep((10, 10), 1.0, 1.0, STOPS3), None, r)          # degenerate sweep
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.3, 0.2, 0.1, 1), None, r)
    if with_layer:
        s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.5, Affine.IDENTITY, r)
        s.stroke(Stroke(2.0), Affine.IDENTITY, Gradient.linear((0, 0), (20, 20), STOPS3), None, r)
        s.pop_layer()
    return s


def test_n_stops_agrees_between_the_encoders():
    from vello_b200.scene_native import NativeScene
    py, nat = stop_scene(Scene), stop_scene(NativeScene)
    assert py.n_stops == nat.n_stops == 3 + 2 + 3 + 3
    assert sum(len(p["stops"]) for p in py.encoding.ramp_patches) == py.n_stops
    # a gradient adds its stops and nothing else does
    for cls in (Scene, NativeScene):
        s = cls()
        before = s.n_stops
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (9, 0), STOPS3), None, Rect(0, 0, 9, 9))
        assert (before, s.n_stops) == (0, 3)
    # append and batch concatenate in stream order
    a, b = stop_scene(Scene), stop_scene(Scene, False)
    na, nb = stop_scene(NativeScene), stop_scene(NativeScene, False)
    a.append(b, Affine.translate(3, 4))
    na.append(nb, Affine.translate(3, 4))
    assert a.n_stops == na.n_stops == 11 + 8
    pb, _ = batch([stop_scene(Scene), stop_scene(Scene, False)])
    nbatch = NativeScene()
    nbatch.batch([stop_scene(NativeScene), stop_scene(NativeScene, False)])
    assert pb.n_stops == nbatch.n_stops == 19


def test_python_ramp_patches_hold_the_rows():
    """Row k of a binding is stop k of the patches in order, after the brush alpha."""
    s = stop_scene(Scene)
    rows = [(o, c.r, c.g, c.b, c.a) for p in s.encoding.ramp_patches for (o, c) in p["stops"]]
    assert len(rows) == s.n_stops
    assert rows[:3] == [(o, c.r, c.g, c.b, c.a) for o, c in STOPS3]


@pytest.mark.parametrize("t, err", [
    (np.zeros((4, 5), np.float32), TypeError),                 # host memory: no __cuda_array_interface__
    (_Cai((5, 4)), ValueError),                                # not 5 columns
    (_Cai((5, 5, 1)), ValueError),                             # not 2-D
    (_Cai((0, 5)), ValueError),                                # no rows
    (_Cai((5, 5), "<f8"), ValueError),                         # float64
    (_Cai((5, 5), "<f2"), ValueError),                         # float16
    (_Cai((5, 5), strides=(40, 8)), ValueError),               # columns not 4 bytes apart
    (_Cai((5, 5), strides=(4, 20)), ValueError),               # a transposed array
    (_Cai((5, 5), strides=(22, 4)), ValueError),               # a row pitch that is not a multiple of 4
    (_Cai((5, 5), strides=(16, 4)), ValueError),               # rows that overlap
])
def test_python_checks_refuse_before_the_library(t, err):
    from vello_b200.renderer import Renderer
    r = Renderer._borrowed(_NoLib(), 1, owner=object())
    with pytest.raises(err):
        r.bind_gradient_stops(t)


def test_python_accepts_column_slices():
    from vello_b200.renderer import Renderer
    calls = []

    class Lib:
        def vb_bind_gradient_stops(self, handle, ptr, n, pitch):
            calls.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = Renderer._borrowed(Lib(), 1, owner=object())
    t = _Cai((7, 5), strides=(36, 4))  # state[:, 2:7] of a (7, 9) float32 array
    r.bind_gradient_stops(t)
    assert calls == [(1 << 20, 7, 36)] and r._stops is t
    r.bind_gradient_stops(_Cai((1, 5), strides=(4, 4)))  # one row: its pitch is never used
    assert calls[-1] == (1 << 20, 1, 20)
    r.bind_gradient_stops(None)
    assert calls[-1] == (None, 0, 0) and r._stops is None


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


def _functions(sass):
    """{mangled name: [opcodes]} of a cuobjdump -sass listing."""
    out = {}
    for part in sass.split("Function : ")[1:]:
        name = part.split()[0]
        body = part[:part.index("..........")] if ".........." in part else part
        out[name] = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9.]+)", body)
    return out


@needs_cuobjdump
def test_bound_ramps_run_the_resolves_arithmetic(built):
    """k_bound_ramps and k_make_ramps share one walk: the same floating-point operations, and the only FFMAs are those of the
    correctly rounded divisions (u = i / 511 and 1 / alpha), which the compiler expands the same way in both."""
    fns = _functions(subprocess.run(["cuobjdump", "-sass", os.path.join(built, "k_resolve.o")], capture_output=True, text=True,
                                    check=True).stdout)
    bound = next(v for k, v in fns.items() if "k_bound_ramps" in k)
    make = next(v for k, v in fns.items() if "k_make_ramps" in k)
    for op in ("FMUL", "FADD", "FFMA", "FRND.FLOOR", "MUFU.RCP"):
        assert bound.count(op) == make.count(op), (op, bound.count(op), make.count(op))
    assert bound.count("FRND.FLOOR") == 4 and bound.count("MUFU.RCP") >= 2


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not installed")
def test_ramp_arithmetic_is_not_contracted(tmp_path):
    """The PTX of k_resolve.cu, built with the library's flags, holds no fused multiply-add: every product and sum of the ramp
    walk and the conversion is rounded on its own, as on the host."""
    src = os.path.join(ROOT, "vello_b200", "csrc", "k_resolve.cu")
    out = tmp_path / "k_resolve.ptx"
    subprocess.run(["nvcc", "-O3", "-std=c++17", "-arch=sm_90a", "-fmad=false", "-ptx", src, "-o", str(out)], check=True,
                   cwd=os.path.dirname(src))
    ptx = out.read_text()
    assert ".entry _Z13k_bound_ramps" in ptx
    assert "fma." not in ptx and "div.rn.f32" in ptx
