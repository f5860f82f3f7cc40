"""The lean partitions' lines, written by k_flatten_emit straight to their final positions.

k_flatten_lean only counts a lean partition (line counts, path boxes, deferred arc jobs); after the scan k_flatten_emit
plans its tags again and writes their literal lines at part_dst + tag_off + rel, leaving gaps for the deferred arcs that
k_flatten_place expands. So a frame of lean partitions leaves no literal record (flatten counter [0]) and no work-list
entry (counter [2]), and its `lines` and `path_bboxes` must still equal the oracle's byte for byte: with straight
strokes and fills only, with round joins and caps whose arcs are deferred between literal lines of the same warp (also
with `lines` limited to exactly what the frame needs), and on the headline scene at the size that is timed.
"""
import math

import numpy as np
import pytest

from vello_b200.encoding import STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND

from .test_flatten_geometry import EPS_FILL, Case, fill, polyline, stroke
from .test_gpu_flatten_geometry import FJ_ARC, gpu_flatten, guarded, n_of, renderer  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def polygon(rng, cx, cy, extent, n):
    ang = np.sort(rng.uniform(0.0, 2.0 * math.pi, n))
    rad = rng.uniform(0.35, 1.0, n) * extent
    return [(float(cx + r * math.cos(a)), float(cy + r * math.sin(a))) for r, a in zip(rad, ang)]


def walk(rng, x, y, n, step, turn_deg):
    """A polyline of n segments of length `step` whose heading changes by a random angle of up to +-turn_deg."""
    pts, h = [(x, y)], rng.uniform(0.0, 2.0 * math.pi)
    for _ in range(n):
        h += math.radians(rng.uniform(-turn_deg, turn_deg))
        x, y = x + step * math.cos(h), y + step * math.sin(h)
        pts.append((float(x), float(y)))
    return pts


def straight_scene(s):
    rng = np.random.default_rng(7)
    for k in range(160):
        fill(polyline(polygon(rng, *rng.uniform(20.0, 236.0, 2), rng.uniform(4.0, 30.0), int(rng.integers(5, 40))), close=True))(s)
        if k % 2 == 0:
            join = (STYLE_JOIN_BEVEL, STYLE_JOIN_MITER)[k % 4 // 2]
            cap = (STYLE_CAP_BUTT, STYLE_CAP_SQUARE)[k % 8 // 4]
            stroke(polyline(walk(rng, *rng.uniform(60.0, 196.0, 2), int(rng.integers(5, 30)), 6.0, 50.0)),
                   width=float(rng.uniform(0.5, 5.0)), join=join, miter_limit=10.0, start_cap=cap, end_cap=cap)(s)


def round_scene(s):
    """Width 12: a round join's arc has 1-2 lines below about 65 degrees of turn and is deferred as a job of 3 or more
    lines above it; a round cap's half turn is a job of 6 lines."""
    rng = np.random.default_rng(11)
    for k in range(90):
        stroke(polyline(walk(rng, *rng.uniform(40.0, 216.0, 2), int(rng.integers(4, 24)), 9.0, 120.0)), width=12.0,
               join=STYLE_JOIN_ROUND, start_cap=STYLE_CAP_ROUND, end_cap=STYLE_CAP_ROUND)(s)
        fill(polyline(polygon(rng, *rng.uniform(20.0, 236.0, 2), 10.0, 9), close=True))(s)


def test_gpu_emit_straight_lines(renderer, oracle):  # noqa: F811
    """Line-to fills and bevel / miter strokes with butt / square caps over many partitions: every line is a literal
    line of a lean partition, none leaves as a record."""
    case = Case("emit-straight", straight_scene, EPS_FILL, w=256, h=256)
    _, st = gpu_flatten(renderer, oracle, case)
    ctr = st["counters"]
    assert int(st["bump"]["lines"]) > 32 * 100
    assert int(ctr[0]) == 0 and int(ctr[1]) == 0 and int(ctr[2]) == 0, ctr[:3]


def test_gpu_emit_around_deferred_arcs(renderer, oracle):  # noqa: F811
    """Round joins and caps: deferred arcs of 3+ lines sit between literal lines of the same lean partitions, so a warp's
    stores skip their gaps; then the same frame with `lines` limited to its exact need."""
    case = Case("emit-round", round_scene, EPS_FILL, w=256, h=256)
    packed, st = gpu_flatten(renderer, oracle, case)
    ctr, jobs = st["counters"], st["jobs"]
    assert int(ctr[0]) == 0 and int(ctr[2]) == 0, ctr[:3]
    assert len(jobs) > 0 and ((jobs["meta"] & FJ_ARC) != 0).all() and n_of(jobs).min() >= 3
    assert len(np.unique(jobs["tag_ix"] >> 5)) >= 20  # many lean partitions with gaps
    guarded(renderer, packed, case, int(st["bump"]["lines"]))


def test_gpu_emit_headline_scene(renderer, oracle):  # noqa: F811
    """The headline scene (paris-like, 30,000 paths, 4096 x 4096): lines and path boxes equal the oracle's. Only the
    partitions holding a curve leave literal records for k_flatten_place."""
    from vello_b200 import scenes
    from vello_b200.encoding import resolve
    packed = resolve(scenes.paris_like(30000, 4096).encoding)
    case = Case("paris-like-30k", lambda s: None, EPS_FILL, w=4096, h=4096)
    _, st = gpu_flatten(renderer, oracle, case, packed)
    n_lines, ctr = int(st["bump"]["lines"]), st["counters"]
    assert int(ctr[1]) > 0 and int(ctr[2]) > 0
    assert int(ctr[0]) < 0.05 * n_lines, (int(ctr[0]), n_lines)
