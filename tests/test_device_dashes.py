"""Dashed fragments from device arrays, without a GPU: the facts of the host dasher that the device's per-ring walk relies on,
the translation of each ring's dashes into sub-rings (tests/device_dashes_ref.py) against `Scene.stroke`'s words on thousands
of random rings, the worst-case bound of the intermediate, the argument checks of `Renderer.upload_device_dashes`, and the
compiled dash kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.encoding import Stroke
from vello_b200.shapes import Arc, Circle, Ellipse, RoundedRect, dash, path_elements

from . import device_curves_ref as curves
from . import device_dashes_ref as ref
from .test_device_curves import random_curved
from .test_device_paths import Dev, Lib, worst_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POOLS = {"values": [0.0, -0.0, 1.0, 5.0, 2e-12, 7.5, 13.25], "wide": [0.0, 3.0, 9.5, 30.0, 40.0, -4.0],
         "eps": [0.0, -0.0, 4e-13, 8e-13, -8e-13, 1e-12, 2e-12, -2e-12, 3e-12, 1.0]}
PATTERNS = [(10.0, 5.0), (0.0, 8.0), (6.0, 3.0, 2.0), (100.0, 1.0), (4.0, 0.0), (1.0, 1.0), (3.0, 0.0, 2.0, 4.0), (1000.0, 0.5)]
OFFSETS = [0.0, 2.5, -3.0, 15.0, 17.0, 1000.5, -0.0, 5.0]


def cases(seed, n):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        pool = POOLS[list(POOLS)[int(rng.integers(0, len(POOLS)))]]
        pts, kinds, roff, poff = random_curved(rng, int(rng.integers(1, 4)), pool)
        pattern = PATTERNS[int(rng.integers(0, len(PATTERNS)))]
        offsets = [OFFSETS[int(rng.integers(0, len(OFFSETS)))] for _ in range(len(poff) - 1)]
        yield pts, kinds, roff, poff, bool(rng.random() < 0.6), pattern, offsets


@pytest.mark.parametrize("seed", range(8))
def test_rings_dash_independently(seed):
    """Fact 1: a path's dashes are its rings' dashes joined, for rings of two or more points."""
    for pts, kinds, roff, poff, closed, pattern, offsets in cases(seed, 150):
        for i in range(len(poff) - 1):
            whole = dash(ref.shape(pts, kinds, roff, poff, i, closed), offsets[i], pattern)
            parts = []
            for k in range(poff[i], poff[i + 1]):
                if roff[k + 1] - roff[k] >= 2:
                    parts += dash(ref.ring_elements(pts, kinds, roff[k], roff[k + 1], closed), offsets[i], pattern)
            assert whole == parts


def test_one_point_rings_are_the_exception():
    """A closed one-point ring gives Z and a segment that depends on the rings before it: the contract leaves it out."""
    assert dash([("M", 1.0, 2.0), ("Z",)], 0.0, (3.0, 1.0)) == [("Z",), ("L", 0.0, 0.0)]
    after = dash([("M", 5.0, 5.0), ("L", 6.0, 5.0), ("M", 1.0, 2.0), ("Z",)], 0.0, (3.0, 1.0))
    assert after[-1] == ("L", 6.0, 5.0)


@pytest.mark.parametrize("seed", range(8))
def test_ring_dashes_have_the_walk_structure(seed):
    """Facts 2 and 3: a ring's dashes start with M, and a Z comes only when the closed ring never leaves its first dash: M p0,
    then the segments, Z, then exactly one segment."""
    z_rings = 0
    for pts, kinds, roff, poff, closed, pattern, offsets in cases(100 + seed, 150):
        for i in range(len(poff) - 1):
            for k in range(poff[i], poff[i + 1]):
                a, b = roff[k], roff[k + 1]
                if b - a < 2:
                    continue
                out = dash(ref.ring_elements(pts, kinds, a, b, closed), offsets[i], pattern)
                if not out:
                    continue
                assert out[0][0] == "M"
                zs = [j for j, e in enumerate(out) if e[0] == "Z"]
                if zs:
                    z_rings += 1
                    assert closed and zs == [len(out) - 2] and out[-1][0] in "LQC"
                    assert [e[0] for e in out].count("M") == 1 and out[0][1:] == (float(pts[a][0]), float(pts[a][1]))
    assert z_rings > 0


def test_curved_tail_after_the_close():
    """The closed ring of the issue that stays inside one dash: M, Q, Z, Q; the last quad is drawn again from p0."""
    els = [("M", 7.5, 9.5), ("Q", 40.0, 30.0, 5.0, 3.0), ("Q", 5.0, 3.0, 7.5, 9.5), ("Z",)]
    assert [e[0] for e in dash(els, 0.0, (100.0, 1.0))] == ["M", "Q", "Z", "Q"]
    pts = np.array([(7.5, 9.5), (40, 30), (5, 3), (5, 3), (7.5, 9.5)], np.float32)
    kinds = np.array([0, 1, 0, 1, 0], np.uint8)
    mid = ref.intermediate(pts, kinds, [0, 5], [0, 1], True, (100.0, 1.0), [0.0])
    assert mid[4] == [ref.CLOSED, ref.CONDITIONAL]
    tags, data = ref.encode(mid)
    want_tags, want_data = ref.host(pts, kinds, [0, 5], [0, 1], True, (100.0, 1.0), [0.0])
    assert tags == want_tags and (data.view(np.uint32) == want_data.view(np.uint32)).all()


@pytest.mark.parametrize("seed", range(12))
def test_sub_rings_encode_as_the_dashed_stroke(seed):
    """The intermediate's sub-rings under the device's rules give Scene.stroke's words for the dashed paths, and its counts
    bound the encoding by the worst case the fragment is allocated for."""
    flags = set()
    for pts, kinds, roff, poff, closed, pattern, offsets in cases(200 + seed, 120):
        mid = ref.intermediate(pts, kinds, roff, poff, closed, pattern, offsets)
        flags.update(mid[4])
        tags, data = ref.encode(mid)
        want_tags, want_data = ref.host(pts, kinds, roff, poff, closed, pattern, offsets)
        assert tags == want_tags, (pts.tolist(), kinds.tolist(), roff, poff, closed, pattern, offsets)
        assert data.view(np.uint32).tolist() == want_data.view(np.uint32).tolist()
        n_paths = len(poff) - 1
        bound = worst_case(len(mid[0]), len(mid[2]) - 1, n_paths)
        got = (len(want_tags) + (2 if n_paths else 0), len(want_data), want_tags.count(curves.TAG_PATH))
        assert got[0] <= bound[0] and got[1] <= bound[1] and got[2] <= bound[2], (got, bound)
    assert {0, ref.CLOSED, ref.CONDITIONAL} <= flags


@pytest.mark.parametrize("shape", [Circle(50, 60, 20), Ellipse(40, 40, 30, 10, 0.4), RoundedRect(10, 10, 90, 60, 12),
                                   Arc(50, 50, 30, 20, 0.3, 4.0)], ids=["circle", "ellipse", "rounded_rect", "arc"])
@pytest.mark.parametrize("pattern", [(10.0, 5.0), (0.0, 8.0), (6.0, 3.0, 2.0), (1000.0, 1.0)])
def test_kurbo_shapes(shape, pattern):
    els = list(path_elements(shape, 0.1))
    pts, kinds, roff = curves.points_of(els)
    closed = els[-1][0] == "Z"
    for off in (0.0, 3.5, -7.25):
        mid = ref.intermediate(pts, kinds, roff, [0, len(roff) - 1], closed, pattern, [off])
        tags, data = ref.encode(mid)
        want_tags, want_data = ref.host(pts, kinds, roff, [0, len(roff) - 1], closed, pattern, [off])
        assert tags == want_tags and data.view(np.uint32).tolist() == want_data.view(np.uint32).tolist()


# ---- the argument checks of Renderer.upload_device_dashes, which raise before the library is called ------------------------
@pytest.fixture
def r():
    from vello_b200.renderer import Renderer
    r = Renderer.__new__(Renderer)
    r.lib, r.handle = Lib(), None
    return r


PTS, ROFF, COLS = Dev((4, 2), "<f4"), Dev((2,), "<i4"), Dev((1, 4), "<f4")
DASHED = Stroke(2.0, dash_pattern=(4.0, 2.0))


@pytest.mark.parametrize("kw, match", [
    (dict(stroke=Stroke(2.0)), "dash pattern"),
    (dict(stroke=0), "dash pattern"),
    (dict(dash_offsets=Dev((2,), "<f4")), "2 dash offsets for 1 paths"),
    (dict(dash_offsets=Dev((1,), "<f8")), "float32"),
    (dict(dash_offsets=np.zeros(1, np.float32)), "__cuda_array_interface__"),
    (dict(point_kinds=Dev((3,), "|u1")), "3 entries for 4 points"),
    (dict(draw_index=Dev((2,), "<i4")), "2 entries for 1 paths"),
    (dict(colors=Dev((2, 4), "<f4")), "2 colours for 1 paths"),
    (dict(ring_offsets=Dev((2,), "<i8")), "int32"),
])
def test_argument_checks(r, kw, match):
    args = dict(points=PTS, ring_offsets=ROFF, colors=COLS, stroke=DASHED)
    args.update(kw)
    with pytest.raises((ValueError, TypeError), match=match):
        r.upload_device_dashes(args.pop("points"), args.pop("ring_offsets"), args.pop("colors"), args.pop("stroke"), **args)


def test_upload_device_paths_still_refuses_dashes(r):
    with pytest.raises(ValueError, match="dashed"):
        r.upload_device_paths(PTS, ROFF, COLS, style=DASHED)


# ---- the compiled kernels ---------------------------------------------------------------------------------------------------
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_device_dashes.o")


@pytest.mark.skipif(not shutil.which("cuobjdump") or not os.path.exists(OBJ), reason="needs cuobjdump and a build")
def test_dash_kernels_use_no_stack_or_local_memory():
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", OBJ], capture_output=True, text=True, check=True).stdout
    names = re.findall(r"Function (\w+):", out)
    assert sorted(names) == sorted(f"_Z{len(n)}{n}6DdArgs" for n in
                                   ("k_device_dashes_phase", "k_device_dashes_count", "k_device_dashes_scan", "k_device_dashes_emit"))
    for m in re.finditer(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out):
        assert m.group(3) == "0" and m.group(4) == "0", m.group(0)
