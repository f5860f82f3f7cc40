"""flatten on the oracle, against the exact geometry of what it approximates (tests/flatten_ref.py).

The GPU parity tests compare k_flatten with the oracle, a port of the same f32 algorithm, so a wrong constant, branch or
clamp the two share cannot show there. These tests hold the oracle's `lines` to the curves and strokes themselves, on
crafted scenes: cusps, loops, inflections, degenerate control points, transforms from 1e-3 to 1e3, mirrors and skews,
strokes from 1e-3 to 1e4 px wide with every join and cap, curves far from the frame and circles of radius up to 1e6.
Each case also shows, through flatten_ref.classify_path, that it reaches the branch it is named for.
tests/test_gpu_flatten_geometry.py applies the same checks to the GPU's own lines.
"""
import math

import numpy as np
import pytest

from vello_b200.config import AA_AREA
from vello_b200.encoding import (BLACK, FILL_NON_ZERO, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE,
                                 STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, Color, Scene, Stroke, f16_to_f32,
                                 f32_to_f16, resolve)
from vello_b200.shapes import Affine, BezPath, Circle

from . import flatten_ref as ref

WHITE = Color.from_rgba8(255, 255, 255)
JOINS = {"bevel": STYLE_JOIN_BEVEL, "miter": STYLE_JOIN_MITER, "round": STYLE_JOIN_ROUND}
CAPS = {"butt": STYLE_CAP_BUTT, "square": STYLE_CAP_SQUARE, "round": STYLE_CAP_ROUND}

# Tolerances, device px, from the largest distances flatten_ref measured on the oracle (DESIGN.md, "tolerance envelope of
# flatten"), with a little room; a case must stay within its class's figure both ways (lines to geometry, geometry to lines):
EPS_FILL = 0.4      # fills: the Euler-spiral fit plus the chords (measured 0.363, a skewed cubic)
EPS_STROKE = 0.45   # strokes with curved segments: two offset curves, joins and caps (measured 0.408)
EPS_STRAIGHT = 0.3  # strokes of straight segments: exact outline pieces and the chords of round joins and caps (measured 0.253)
EPS_FAR_ULPS = 8    # a curve far from the frame: its f32 coordinates are only this many ulps precise
# Past the envelope (the reference's own behaviour, kept bit for bit):
EPS_CLAMP = 2.5     # a circle of radius 10^6 px: 100 lines per Euler segment are too few (measured 2.34 px)
EPS_LONG_ARC = 3.0  # a round cap of radius 10^6 px: 2,275 f32 rotations drift (measured 2.69 px)
RUNAWAY = 65536     # a curve 10^8 px away: its f32 points are 8 px apart and the subdivision runs towards SUBDIV_LIMIT


def ulp(x):
    return float(np.spacing(np.float32(abs(x))))


class Case:
    """A scene of one or more paths; `eps` the device tolerance of each path's contract, `expect` tags the classifier
    must report for the case (see `tags`), `outline` whether to check strokes against their exact outline."""

    def __init__(self, name, build, eps, expect=(), w=128, h=128, outline=None, runaway=False):
        self.name, self.build, self.eps, self.expect, self.w, self.h, self.outline = name, build, eps, set(expect), w, h, outline
        self.runaway = runaway  # past the count bound: at most RUNAWAY lines per segment side

    def __repr__(self):
        return self.name

    def scene(self):
        s = Scene()
        self.build(s)
        return s


def tags(paths):
    """What the paths reach in flatten, as a set: branch:<k1|dist|espc>, piece:<sin|pow|quad1|quad2>, clamped,
    subdiv_limit, deriv_thresh, tiny_chord, n:<lines> of every Euler segment, arc:<lines> of every arc, fast, and the
    classifier's flags (segment kinds, joins, caps, closed, tangent_fallback, mirror, non_uniform)."""
    out = set()
    for p in paths:
        c = ref.classify_path(p)
        out |= c["flags"]
        for e in c["euler"]:
            out |= {k for k in ("deriv_thresh", "tiny_chord") if e[k]}
            out.add("branch:" + e["branch"])
            out |= {"piece:" + x for x in e.get("pieces", ())}
            out.add(f"n:{e['n']}")
            if e["clamped"]:
                out.add("clamped")
            if e["subdiv_limit"]:
                out.add("subdiv_limit")
        out |= {f"arc:{n}" for n in c["arcs"]}
        if c["fast"]:
            out.add("fast")
    return out


def fill(path, xf=Affine.IDENTITY, rule=FILL_NON_ZERO):
    return lambda s: s.fill(rule, xf, WHITE, None, path)


def stroke(path, xf=Affine.IDENTITY, **kw):
    return lambda s: s.stroke(Stroke(**kw), xf, WHITE, None, path)


def cubic_path(p0, p1, p2, p3, close=True):
    els = [("M",) + p0, ("C",) + p1 + p2 + p3]
    return BezPath(els + ([("Z",)] if close else []))


def scaled(pts, k, o=(0.0, 0.0)):
    return [(o[0] + k * x, o[1] + k * y) for x, y in pts]


CUSP = [(0.0, 0.0), (1.0, 1.0), (0.0, 1.0), (1.0, 0.0)]
LOOP = [(0.0, 0.0), (1.5, 1.0), (-0.5, 1.0), (1.0, 0.0)]
S_CURVE = [(0.0, 0.5), (0.45, -0.5), (0.55, 1.5), (1.0, 0.5)]
BLOB = [(0.1, 0.5), (0.2, -0.2), (1.1, 0.3), (0.9, 0.9)]


def curve_cases():
    c = lambda pts, **kw: cubic_path(*pts, **kw)
    out = [
        Case("cusp", fill(c(scaled(CUSP, 100, (14, 14)))), EPS_FILL, {"branch:dist", "n:2"}),
        Case("loop", fill(c(scaled(LOOP, 60, (34, 20)))), EPS_FILL, {"branch:dist"}),
        Case("inflection", fill(c(scaled(S_CURVE, 100, (14, 14)))), EPS_FILL, {"branch:dist", "n:3"}),
        Case("collinear-double-back", fill(BezPath([("M", 10.0, 50.0), ("C", 110.0, 50.0, 0.0, 50.0, 60.0, 50.0),
                                                    ("L", 60.0, 90.0), ("Z",)])), EPS_FILL, {"branch:k1"}),
        Case("p0-eq-p1", fill(c([(20.0, 20.0), (20.0, 20.0), (100.0, 30.0), (100.0, 100.0)])), EPS_FILL, {"deriv_thresh"}),
        Case("p2-eq-p3", fill(c([(20.0, 20.0), (30.0, 100.0), (100.0, 100.0), (100.0, 100.0)])), EPS_FILL, {"deriv_thresh"}),
        Case("p0-eq-p1-p2-eq-p3", fill(c([(20.0, 20.0), (20.0, 20.0), (100.0, 90.0), (100.0, 90.0)])), EPS_FILL,
             {"deriv_thresh"}),
        # all four control points within 1e-6 px: a chord below DERIV_THRESH
        Case("within-1e-6", fill(BezPath([("M", 0.5, 0.5), ("C", 0.5 + 1e-6, 0.5, 0.5, 0.5 + 1e-6, 0.5 + 5e-7, 0.5 + 5e-7),
                                          ("L", 60.0, 60.0), ("L", 0.5, 60.0), ("Z",)])), EPS_FILL, {"tiny_chord"}),
        Case("quads", fill(BezPath([("M", 10.0, 100.0), ("Q", 64.0, -60.0, 118.0, 100.0), ("Q", 64.0, 20.0, 10.0, 100.0),
                                    ("Z",)])), EPS_FILL, {"seg:quad", "branch:dist"}),
    ]
    for k in (1e-3, 1e-1, 1e1, 1e3):
        out.append(Case(f"scale-{k:g}", fill(c(scaled(BLOB, 100 / k)), Affine.scale(k) * Affine.translate(10 / k, 10 / k)),
                        EPS_FILL, {"branch:dist", "n:8"}))
    out += [
        Case("mirror", fill(c(scaled(LOOP, 60)), Affine((-1.0, 0.0, 0.0, 1.0, 100.0, 20.0))), EPS_FILL, {"mirror"}),
        Case("mirror-y-rot", fill(c(scaled(S_CURVE, 80)), Affine.translate(20, 110) * Affine((0.6, 0.8, 0.8, -0.6, 0, 0)) *
                                  Affine.scale(1.0)), EPS_FILL, {"mirror"}),
        Case("skew", fill(c(scaled(BLOB, 80)), Affine((1.0, 0.3, 0.9, 1.0, 5.0, 5.0))), EPS_FILL, {"non_uniform"}),
    ]
    return out


def polyline(pts, close=False):
    return BezPath([("M",) + pts[0]] + [("L",) + p for p in pts[1:]] + ([("Z",)] if close else []))


def turn(deg, l1=50.0, l2=45.0, o=(30.0, 64.0)):
    """Two segments turning by `deg` at the vertex."""
    th = math.radians(deg)
    v = (o[0] + l1, o[1])
    return [o, v, (v[0] + l2 * math.cos(th), v[1] - l2 * math.sin(th))]


def miter_threshold_limits(pts):
    """The f16 miter limits one ulp either side of the exact threshold of the turn at pts[1]."""
    a, v, b = (np.array([np.float32(x) for x in p], np.float64) for p in pts)
    t0, t1 = ref._unit(v - a), ref._unit(b - v)
    d = float(t0 @ t1)
    lim = math.sqrt(2.0 / (1.0 + d))  # 2 |t0||t1| == (|t0||t1| + d) lim^2
    bits = f32_to_f16(lim)
    lo, hi = bits - 1, bits + 1
    while f16_to_f32(lo + 1) < lim:
        lo += 1
    while f16_to_f32(hi - 1) > lim:
        hi -= 1
    return f16_to_f32(lo), f16_to_f32(hi)


def stroke_cases():
    out = []
    arc = cubic_path((20.0, 100.0), (20.0, 30.0), (108.0, 30.0), (108.0, 100.0), close=False)
    reach = {1e-3: {"branch:dist"}, 0.5: {"piece:pow"}, 8.0: {"piece:pow"}, 40.0: {"piece:sin", "piece:quad1"},
             1e4: {"piece:quad2"}}
    for w in (1e-3, 0.5, 8.0, 40.0, 1e4):
        out.append(Case(f"width-{w:g}", stroke(arc, width=w, join=STYLE_JOIN_ROUND), EPS_STROKE, reach[w]))
    # radius of curvature 10 px at the top of the bend, half width 20: the inner offset curve forms an evolute
    out.append(Case("evolute", stroke(cubic_path((30.0, 100.0), (60.0, 10.0), (68.0, 10.0), (98.0, 100.0), close=False),
                                      width=40.0), EPS_STROKE, {"piece:quad2"}))
    out.append(Case("cusp-stroke", stroke(cubic_path(*scaled(CUSP, 80, (24, 24)), close=False), width=6.0,
                                          join=STYLE_JOIN_BEVEL, start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), EPS_STROKE,
                    {"branch:espc", "cap:butt"}))
    for jn, j in JOINS.items():
        for deg in (1e-3, 90.0, 179.9, 180.0):
            out.append(Case(f"join-{jn}-{deg:g}", stroke(polyline(turn(deg)), width=12.0, join=j, miter_limit=10.0,
                                                          start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), EPS_STRAIGHT,
                            {"fast", "join:miter-bevel" if jn == "miter" and deg > 170 else f"join:{jn}"}))
        out.append(Case(f"closed-{jn}", stroke(polyline([(20.0, 20.0), (100.0, 30.0), (60.0, 105.0)], close=True), width=10.0,
                                               join=j, miter_limit=4.0), EPS_STRAIGHT, {"closed", f"join:{jn}"}))
        out.append(Case(f"curve-join-{jn}", stroke(BezPath([("M", 20.0, 100.0), ("Q", 40.0, 10.0, 64.0, 60.0),
                                                            ("C", 80.0, 100.0, 100.0, 20.0, 110.0, 110.0)]),
                                                   width=9.0, join=j, miter_limit=4.0), EPS_STROKE,
                        {"branch:espc", f"join:{jn}", "seg:quad", "seg:cubic"}))
    pts = turn(120.0)
    lo, hi = miter_threshold_limits(pts)
    for name, lim, got in (("below", lo, "join:miter-bevel"), ("above", hi, "join:miter")):
        out.append(Case(f"miter-limit-{name}", stroke(polyline(pts), width=12.0, join=STYLE_JOIN_MITER, miter_limit=lim,
                                                      start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT), EPS_STRAIGHT, {got}))
    for cn, cap in CAPS.items():
        arcs = {"arc:7"} if cn == "round" else set()
        out.append(Case(f"cap-{cn}", stroke(polyline([(30.0, 40.0), (90.0, 80.0)]), width=16.0, start_cap=cap, end_cap=cap),
                        EPS_STRAIGHT, {f"cap:{cn}"} | arcs))
        out.append(Case(f"cap-{cn}-curve", stroke(arc, width=10.0, start_cap=cap, end_cap=cap, join=STYLE_JOIN_BEVEL),
                        EPS_STROKE, {f"cap:{cn}", "branch:espc"}))
    # zero-length segments (the encoder drops them) and one 3e-7 long (kept, shorter than TANGENT_THRESH: flatten falls
    # back to a fixed tangent), under a scale so that f32 resolves it
    out.append(Case("zero-length-segments", stroke(polyline([(-1.0, -0.5), (-1.0, -0.5), (0.5, -0.5), (0.5 + 3e-7, -0.5),
                                                             (0.5, 0.8), (0.5, 0.8)]), Affine.translate(64.0, 64.0) *
                                                   Affine.scale(40.0), width=0.2, join=STYLE_JOIN_MITER), EPS_STRAIGHT,
                    {"tangent_fallback", "join:miter"}))
    out.append(Case("dashes-on-curves", stroke(Circle(64.0, 64.0, 40.0), width=5.0, dash_pattern=(14.0, 6.0, 3.0, 6.0)),
                    EPS_STROKE, {"branch:espc", "cap:round", "seg:cubic"}))
    out.append(Case("non-uniform-scale", stroke(arc, Affine.translate(0, -40) * Affine.scale(0.25, 1.5), width=12.0,
                                                join=STYLE_JOIN_ROUND), EPS_STROKE, {"non_uniform", "branch:espc"}))
    out.append(Case("non-uniform-polyline", stroke(polyline([(20.0, 20.0), (100.0, 30.0), (60.0, 105.0)], close=True),
                                                   Affine((2.0, 0.3, -0.4, 0.5, -10.0, 20.0)), width=10.0,
                                                   join=STYLE_JOIN_MITER), EPS_STRAIGHT, {"non_uniform", "closed", "join:miter"}))
    out.append(Case("mirror-stroke", stroke(arc, Affine((-1.0, 0.0, 0.0, 1.0, 128.0, 0.0)), width=7.0,
                                            join=STYLE_JOIN_ROUND), EPS_STROKE, {"mirror", "branch:espc"}))
    return out


def far_cases():
    out = []
    for far in (1e3, 1e5, 1e6, 1e8):
        eps = max(EPS_FILL, EPS_FAR_ULPS * ulp(far))
        run = far >= 1e8
        out.append(Case(f"far-fill-{far:g}", fill(cubic_path(*scaled(BLOB, 60, (far, far)))), eps, runaway=run))
        out.append(Case(f"far-stroke-{far:g}", stroke(cubic_path(*scaled(BLOB, 60, (far, -far)), close=False), width=6.0), eps,
                        runaway=run))
    for r, n, arcs in ((1e2, "n:12", "arc:23"), (1e4, "n:64", "arc:223"), (1e6, "n:100", "arc:2275")):
        big = r >= 1e6
        out.append(Case(f"circle-{r:g}", fill(Circle(64.0 - r + 40.0, 64.0, r)), EPS_CLAMP if big else EPS_FILL,
                        {"branch:k1", n} | ({"clamped"} if big else set())))
        out.append(Case(f"round-cap-{r:g}", stroke(polyline([(64.0 - r, 64.0), (64.0, 64.0)]), width=2 * r),
                        EPS_LONG_ARC if big else EPS_STRAIGHT, {arcs, "cap:round"}))
    return out


CASES = curve_cases() + stroke_cases()
FAR_CASES = far_cases()


def run_oracle(oracle, case):
    packed = resolve(case.scene().encoding)
    oracle.bind(packed, case.w, case.h, BLACK.premul_rgba8_u32(), AA_AREA)
    oracle.run("pathtag", "flatten")
    return packed, oracle.buffer("lines")[: int(oracle.buffer("bump")["lines"][0])]


def check_case(case, lines):
    """The flatten contract for every path of the case; returns the decoded paths and what was measured."""
    paths = ref.decode(case.scene().encoding)
    reps = []
    for p in paths:
        n = int((lines["path_ix"] == p.index).sum())
        if case.runaway:
            sides = sum(len(sp.segs) for sp in p.subpaths) * (2 if p.is_stroke else 1)
            assert ref.count_bound(p) < n <= RUNAWAY * sides, (case.name, n)
        else:
            bound = ref.count_bound(p)
            assert n <= bound, f"{case.name} path {p.index}: {n} lines, the curve needs about {bound:.0f} at most"
        if p.is_stroke:
            reps.append(ref.check_stroke(p, lines, case.eps, exact_outline=case.outline))
        else:
            reps.append(ref.check_fill(p, lines, case.eps))
    return paths, reps


@pytest.mark.parametrize("case", CASES + FAR_CASES, ids=repr)
def test_flatten_geometry(oracle, case):
    _, lines = run_oracle(oracle, case)
    paths, _ = check_case(case, lines)
    got = tags(paths)
    assert case.expect <= got, (case.name, sorted(case.expect - got))
