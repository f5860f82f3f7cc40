"""Fragments from device arrays, without a GPU: the argument checks of `Renderer.upload_device_paths`, which raise before the
library is called, and the worst-case stream lengths vb_fragment_from_device_paths allocates a fragment for, against the host
encoder's lengths on random and degenerate inputs."""
import numpy as np
import pytest

from vello_b200.encoding import FILL_NON_ZERO, Scene, Stroke
from vello_b200.renderer import Renderer
from vello_b200.shapes import Affine
from vello_b200.encoding import Color

from .test_compiled_kernels import built, usage  # noqa: F401  (fixtures)


class Dev:
    """A stand-in device array: only its __cuda_array_interface__."""

    def __init__(self, shape, typestr, strides=None, ptr=0x10000):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, strides=strides, data=(ptr, False), version=2)


class Lib:
    """Fails the test if the library is reached."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


@pytest.fixture
def r():
    r = Renderer.__new__(Renderer)
    r.lib, r.handle = Lib(), None
    return r


PTS, ROFF, COLS = Dev((4, 2), "<f4"), Dev((2,), "<i4"), Dev((1, 4), "<f4")


@pytest.mark.parametrize("args, kw, match", [
    ((Dev((4, 3), "<f4"), ROFF, COLS), {}, "points must be"),
    ((Dev((4, 2), "<f8"), ROFF, COLS), {}, "points must be"),
    ((Dev((4, 2), "<f4", strides=(6, 4)), ROFF, COLS), {}, "strides"),
    ((PTS, Dev((2,), "<i8"), COLS), {}, "int64; convert them to int32"),
    ((PTS, ROFF, COLS), dict(path_offsets=Dev((2,), "<i8")), "int64; convert them to int32"),
    ((PTS, Dev((2, 1), "<i4"), COLS), {}, "1-D int32"),
    ((PTS, Dev((3,), "<i4", strides=(8,)), COLS), {}, "contiguous"),
    ((PTS, Dev((0,), "<i4"), COLS), {}, "at least 1"),
    ((PTS, ROFF, Dev((1, 3), "<f4")), {}, "colours must be"),
    ((PTS, ROFF, Dev((2, 4), "<f4")), {}, "2 colours for 1 paths"),
    ((PTS, ROFF, COLS), dict(path_offsets=Dev((3,), "<i4")), "1 colours for 2 paths"),
    ((PTS, ROFF, COLS), dict(draw_index=Dev((2,), "<i4")), "draw_index has 2 entries"),
    ((PTS, ROFF, COLS), dict(draw_index=Dev((1,), "<i8")), "int64"),
    ((PTS, ROFF, COLS), dict(style=Stroke(1.0, dash_pattern=(2.0, 1.0))), "dashed"),
    ((object(), ROFF, COLS), {}, "__cuda_array_interface__"),
])
def test_argument_checks(r, args, kw, match):
    with pytest.raises((ValueError, TypeError), match=match):
        r.upload_device_paths(*args, **kw)


def worst_case(n_points, n_rings, n_paths):
    """The stream lengths vb_fragment_from_device_paths sizes a fragment for (vb_compose.cu): tag bytes, path-data words, draw
    tags, draw-data words, transforms, style words. tests/test_gpu_device_paths.py::test_allocation_is_the_worst_case ties it
    to the library: a fragment's allocation is exactly the one these lengths ask for."""
    if n_paths == 0:
        return (0, 2 * n_points + 4 * n_rings, 0, 0, 0, 0)
    return (2 + n_points + 2 * n_rings + n_paths, 2 * n_points + 4 * n_rings, n_paths, n_paths, 1, 2)


def encoded(pts, roff, poff, style, closed):
    s = Scene()
    stroke = isinstance(style, Stroke)
    for i in range(len(poff) - 1):
        els = []
        for k in range(poff[i], poff[i + 1]):
            a, b = roff[k], roff[k + 1]
            if a == b:
                continue
            els.append(("M", *pts[a]))
            els += [("L", *p) for p in pts[a + 1:b]]
            if closed or not stroke:
                els.append(("Z",))
        if stroke:
            s.stroke(style, Affine.IDENTITY, Color(1, 0, 0, 1), None, els)
        else:
            s.fill(style, Affine.IDENTITY, Color(1, 0, 0, 1), None, els)
    e = s.encoding
    return (len(e.path_tags), len(e.path_data), len(e.draw_tags), len(e.draw_data), len(e.transforms), 2 * len(e.styles))


@pytest.mark.parametrize("seed", range(12))
def test_worst_case_bounds_the_encoder(seed):
    rng = np.random.default_rng(seed)
    n_paths = int(rng.integers(0, 12))
    roff, poff, pts = [0], [0], []
    for _ in range(n_paths):
        for _ in range(int(rng.integers(0, 4))):
            k = int(rng.integers(0, 7))
            # few distinct values: duplicates, rings of one repeated point, closing points equal or not, -0 beside +0
            pool = [0.0, -0.0, 1.0, 5.0, 2e-12, 7.5]
            pts += [(float(rng.choice(pool)), float(rng.choice(pool))) for _ in range(k)]
            roff.append(len(pts))
        poff.append(len(roff) - 1)
    for style in (FILL_NON_ZERO, Stroke(1.0)):
        for closed in (False, True):
            got = encoded(pts, roff, poff, style, closed)
            bound = worst_case(len(pts), len(roff) - 1, n_paths)
            assert all(g <= b for g, b in zip(got, bound)), (got, bound)
            assert got[4:] == bound[4:], "one transform and one style exactly when there are paths"


@pytest.mark.skipif(__import__("shutil").which("cuobjdump") is None, reason="CUDA binary utilities not installed")
def test_kernels_have_no_stack_or_local_memory(usage):  # noqa: F811
    """k_device_paths.o holds exactly the four kernels of the build, each in registers only."""
    fns = usage["k_device_paths.o"]
    names = {"k_device_paths_points", "k_device_paths_rings", "k_device_paths_count", "k_device_paths_emit"}
    assert {k[0] for k in fns} == names and len(fns) == 4, sorted(fns)
    for key, u in fns.items():
        assert u.stack == 0 and u.local == 0, f"{key[0]}: {u.stack} bytes of stack, {u.local} bytes of local memory"
