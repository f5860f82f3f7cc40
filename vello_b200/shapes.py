"""Geometry helpers standing in for the parts of `kurbo 0.13.1` the scene builder touches.

kurbo is a third-party dependency that is *not* in the reference repository (Cargo.lock pins
kurbo 0.13.1); what is restated here is its published algorithm for turning shapes into path
elements (`Shape::path_elements(tolerance)`), which `PathEncoder::shape` calls with
tolerance 0.1 (vello_encoding/src/path.rs:655-657):

* Rect            -> M, L, L, L, Z
* Circle          -> cubic arcs, n = 4 with arm 0.551915024494 below the tolerance knee
* RoundedRect     -> quarter-circle arcs joined by lines
* BezPath.from_svg-> SVG path data incl. elliptical arcs -> cubics (tolerance 0.1)

All maths is f64 like kurbo; the encoder rounds to f32.
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass
from typing import Iterable, Iterator, List, Sequence, Tuple


@dataclass(frozen=True)
class Affine:
    """Column-major 2x3 affine [a, b, c, d, e, f]: x' = a x + c y + e, y' = b x + d y + f."""

    coeffs: Tuple[float, float, float, float, float, float] = (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)

    IDENTITY = None  # filled below

    @staticmethod
    def translate(x: float, y: float) -> "Affine":
        return Affine((1.0, 0.0, 0.0, 1.0, float(x), float(y)))

    @staticmethod
    def scale(s: float, sy: float | None = None) -> "Affine":
        return Affine((float(s), 0.0, 0.0, float(s if sy is None else sy), 0.0, 0.0))

    @staticmethod
    def rotate(th: float) -> "Affine":
        s, c = math.sin(th), math.cos(th)
        return Affine((c, s, -s, c, 0.0, 0.0))

    def __mul__(self, o: "Affine") -> "Affine":
        a = self.coeffs
        b = o.coeffs
        return Affine(
            (
                a[0] * b[0] + a[2] * b[1],
                a[1] * b[0] + a[3] * b[1],
                a[0] * b[2] + a[2] * b[3],
                a[1] * b[2] + a[3] * b[3],
                a[0] * b[4] + a[2] * b[5] + a[4],
                a[1] * b[4] + a[3] * b[5] + a[5],
            )
        )

    def apply(self, x: float, y: float) -> Tuple[float, float]:
        a = self.coeffs
        return (a[0] * x + a[2] * y + a[4], a[1] * x + a[3] * y + a[5])


Affine.IDENTITY = Affine()


@dataclass(frozen=True)
class Rect:
    x0: float
    y0: float
    x1: float
    y1: float

    @staticmethod
    def from_center_size(c, s) -> "Rect":
        return Rect(c[0] - 0.5 * s[0], c[1] - 0.5 * s[1], c[0] + 0.5 * s[0], c[1] + 0.5 * s[1])

    @staticmethod
    def from_origin_size(o, s) -> "Rect":
        return Rect(o[0], o[1], o[0] + s[0], o[1] + s[1])


@dataclass(frozen=True)
class Circle:
    cx: float
    cy: float
    r: float


@dataclass(frozen=True)
class Ellipse:
    """kurbo `Ellipse::new(center, radii, x_rotation)` (ellipse.rs): path = MoveTo(start) + `Arc` over 2 pi + ClosePath."""
    cx: float
    cy: float
    rx: float
    ry: float
    x_rotation: float = 0.0


@dataclass(frozen=True)
class Arc:
    """kurbo `Arc { center, radii, start_angle, sweep_angle, x_rotation }` (arc.rs): an open elliptical arc."""
    cx: float
    cy: float
    rx: float
    ry: float
    start_angle: float
    sweep_angle: float
    x_rotation: float = 0.0


@dataclass(frozen=True)
class RoundedRect:
    x0: float
    y0: float
    x1: float
    y1: float
    radius: float


@dataclass(frozen=True)
class Line:
    x0: float
    y0: float
    x1: float
    y1: float


class BezPath:
    """A list of path elements: ("M",x,y) ("L",x,y) ("Q",x1,y1,x,y) ("C",x1,y1,x2,y2,x,y) ("Z",)."""

    def __init__(self, els: Iterable[tuple] = ()):
        self.els: List[tuple] = list(els)

    def move_to(self, x, y):
        self.els.append(("M", float(x), float(y)))

    def line_to(self, x, y):
        self.els.append(("L", float(x), float(y)))

    def quad_to(self, x1, y1, x, y):
        self.els.append(("Q", float(x1), float(y1), float(x), float(y)))

    def curve_to(self, x1, y1, x2, y2, x, y):
        self.els.append(("C", float(x1), float(y1), float(x2), float(y2), float(x), float(y)))

    def close_path(self):
        self.els.append(("Z",))

    @staticmethod
    def from_svg(d: str) -> "BezPath":
        return BezPath(parse_svg_path(d))


def _arc_elements(cx, cy, rx, ry, start, sweep, x_rot, tolerance) -> Iterator[tuple]:
    """kurbo `Arc::append_iter`: n cubic pieces, n from the tolerance; arm = 4/3 tan(sweep/4n)."""
    sign = 1.0 if sweep >= 0 else -1.0
    scaled_err = max(rx, ry) / tolerance
    n_err = max((1.1163 * scaled_err) ** (1.0 / 6.0), 3.999_999)
    n = int(math.ceil(n_err * abs(sweep) * (1.0 / (2.0 * math.pi))))
    n = max(n, 1)
    angle_step = sweep / n
    arm_len = (4.0 / 3.0) * abs(math.tan(0.25 * angle_step)) * sign
    cr, sr = math.cos(x_rot), math.sin(x_rot)

    def sample(a):
        x, y = rx * math.cos(a), ry * math.sin(a)
        return (cr * x - sr * y, sr * x + cr * y)

    angle0 = start
    p0 = sample(angle0)
    for _ in range(n):
        angle1 = angle0 + angle_step
        p1 = (p0[0] - arm_len * _rot_d(rx, ry, angle0, cr, sr)[0], p0[1] - arm_len * _rot_d(rx, ry, angle0, cr, sr)[1])
        p3 = sample(angle1)
        d1 = _rot_d(rx, ry, angle1, cr, sr)
        p2 = (p3[0] + arm_len * d1[0], p3[1] + arm_len * d1[1])
        yield ("C", cx + p1[0], cy + p1[1], cx + p2[0], cy + p2[1], cx + p3[0], cy + p3[1])
        angle0, p0 = angle1, p3


def _rot_d(rx, ry, a, cr, sr):
    # rotated (rx sin a, -ry cos a): minus the derivative of the ellipse sample
    x, y = rx * math.sin(a), -ry * math.cos(a)
    return (cr * x - sr * y, sr * x + cr * y)


def path_elements(shape, tolerance: float = 0.1) -> Iterator[tuple]:
    if isinstance(shape, BezPath):
        yield from shape.els
    elif isinstance(shape, (list, tuple)):
        yield from shape
    elif isinstance(shape, Rect):
        yield ("M", shape.x0, shape.y0)
        yield ("L", shape.x1, shape.y0)
        yield ("L", shape.x1, shape.y1)
        yield ("L", shape.x0, shape.y1)
        yield ("Z",)
    elif isinstance(shape, Line):
        yield ("M", shape.x0, shape.y0)
        yield ("L", shape.x1, shape.y1)
    elif isinstance(shape, Circle):
        r = abs(shape.r)
        scaled_err = r / tolerance
        if scaled_err < 1.0 / 1.9608e-4:
            n, arm = 4, 0.551915024494
        else:
            n = int(math.ceil((1.1163 * scaled_err) ** (1.0 / 6.0)))
            arm = (4.0 / 3.0) * math.tan(math.pi / (2.0 * n))
        x, y = shape.cx, shape.cy
        yield ("M", x + r, y)
        dth = 2.0 * math.pi / n
        for ix in range(1, n + 1):
            th1 = dth * ix
            th0 = th1 - dth
            s0, c0 = math.sin(th0), math.cos(th0)
            if ix == n:
                s1, c1 = 0.0, 1.0
            else:
                s1, c1 = math.sin(th1), math.cos(th1)
            a = arm * r
            yield (
                "C",
                x + r * c0 - a * s0, y + r * s0 + a * c0,
                x + r * c1 + a * s1, y + r * s1 - a * c1,
                x + r * c1, y + r * s1,
            )
        yield ("Z",)
    elif isinstance(shape, Ellipse):
        # Ellipse::path_elements: radii / rotation come back out of the affine through `svd` (kurbo affine.rs), then
        # Arc { start 0, sweep 2 pi }.path_elements(tolerance) chained with ClosePath
        a, b = shape.rx * math.cos(shape.x_rotation), shape.rx * math.sin(shape.x_rotation)
        c, d = -shape.ry * math.sin(shape.x_rotation), shape.ry * math.cos(shape.x_rotation)
        a2, b2, c2, d2 = a * a, b * b, c * c, d * d
        # kurbo Affine::svd on coefficients [a, b, c, d] (x' = a x + c y, y' = b x + d y): the off-diagonal of M M^T is ab + cd
        rot = 0.5 * math.atan2(2.0 * (a * b + c * d), a2 - b2 + c2 - d2)
        s1 = a2 + b2 + c2 + d2
        s2 = math.sqrt((a2 - b2 + c2 - d2) ** 2 + 4.0 * (a * b + c * d) ** 2)
        rx, ry = math.sqrt(0.5 * (s1 + s2)), math.sqrt(max(0.5 * (s1 - s2), 0.0))
        cr, sr = math.cos(rot), math.sin(rot)
        yield ("M", shape.cx + cr * rx, shape.cy + sr * rx)
        yield from _arc_elements(shape.cx, shape.cy, rx, ry, 0.0, 2.0 * math.pi, rot, tolerance)
        yield ("Z",)
    elif isinstance(shape, Arc):
        # Arc::path_elements: MoveTo(start point) + append_iter
        cr, sr = math.cos(shape.x_rotation), math.sin(shape.x_rotation)
        x, y = shape.rx * math.cos(shape.start_angle), shape.ry * math.sin(shape.start_angle)
        yield ("M", shape.cx + cr * x - sr * y, shape.cy + sr * x + cr * y)
        yield from _arc_elements(shape.cx, shape.cy, shape.rx, shape.ry, shape.start_angle, shape.sweep_angle, shape.x_rotation, tolerance)
    elif isinstance(shape, RoundedRect):
        x0, y0, x1, y1 = shape.x0, shape.y0, shape.x1, shape.y1
        rad = min(abs(shape.radius), 0.5 * abs(x1 - x0), 0.5 * abs(y1 - y0))
        if rad <= 0.0:
            yield from path_elements(Rect(x0, y0, x1, y1), tolerance)
            return
        hp = 0.5 * math.pi
        # start at the top edge after the top-left corner, go clockwise (y down)
        yield ("M", x0 + rad, y0)
        corners = [
            (x1 - rad, y0 + rad, -hp),  # top-right: from angle -90 to 0
            (x1 - rad, y1 - rad, 0.0),  # bottom-right
            (x0 + rad, y1 - rad, hp),  # bottom-left
            (x0 + rad, y0 + rad, 2 * hp),  # top-left
        ]
        for (cx, cy, a0) in corners:
            yield ("L", cx + rad * math.cos(a0), cy + rad * math.sin(a0))
            yield from _arc_elements(cx, cy, rad, rad, a0, hp, 0.0, tolerance)
        yield ("Z",)
    else:
        raise TypeError(f"unsupported shape {type(shape)}")


# ---------------------------------------------------------------------------------------------
# SVG path data (the subset kurbo's `BezPath::from_svg` accepts: MmLlHhVvCcSsQqTtAaZz)
# ---------------------------------------------------------------------------------------------
_NUM = re.compile(r"[+-]?(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?")


class _Lexer:
    def __init__(self, s: str):
        self.s = s
        self.i = 0

    def skip(self):
        while self.i < len(self.s) and self.s[self.i] in " \t\r\n,":
            self.i += 1

    def peek_cmd(self):
        self.skip()
        if self.i < len(self.s) and self.s[self.i].isalpha():
            return self.s[self.i]
        return None

    def more_numbers(self) -> bool:
        self.skip()
        return self.i < len(self.s) and (self.s[self.i] in "+-." or self.s[self.i].isdigit())

    def num(self) -> float:
        self.skip()
        m = _NUM.match(self.s, self.i)
        if not m:
            raise ValueError(f"bad number at {self.i}: {self.s[self.i:self.i+16]!r}")
        self.i = m.end()
        return float(m.group(0))

    def flag(self) -> bool:
        self.skip()
        c = self.s[self.i]
        if c not in "01":
            raise ValueError("bad arc flag")
        self.i += 1
        return c == "1"


def _svg_arc_to_cubics(x0, y0, rx, ry, x_rot_deg, large, sweep, x, y, tolerance=0.1):
    """SVG implementation notes F.6.5 (endpoint -> centre) then `_arc_elements`."""
    if rx == 0.0 or ry == 0.0 or (x0 == x and y0 == y):
        if not (x0 == x and y0 == y):
            yield ("L", x, y)
        return
    rx, ry = abs(rx), abs(ry)
    phi = math.radians(x_rot_deg)
    cp, sp = math.cos(phi), math.sin(phi)
    dx2, dy2 = 0.5 * (x0 - x), 0.5 * (y0 - y)
    x1p = cp * dx2 + sp * dy2
    y1p = -sp * dx2 + cp * dy2
    lam = (x1p * x1p) / (rx * rx) + (y1p * y1p) / (ry * ry)
    if lam > 1.0:
        s = math.sqrt(lam)
        rx *= s
        ry *= s
    num = rx * rx * ry * ry - rx * rx * y1p * y1p - ry * ry * x1p * x1p
    den = rx * rx * y1p * y1p + ry * ry * x1p * x1p
    coef = math.sqrt(max(num / den, 0.0)) if den != 0.0 else 0.0
    if large == sweep:
        coef = -coef
    cxp = coef * rx * y1p / ry
    cyp = -coef * ry * x1p / rx
    cx = cp * cxp - sp * cyp + 0.5 * (x0 + x)
    cy = sp * cxp + cp * cyp + 0.5 * (y0 + y)
    a0 = math.atan2((y1p - cyp) / ry, (x1p - cxp) / rx)
    a1 = math.atan2((-y1p - cyp) / ry, (-x1p - cxp) / rx)
    d = a1 - a0
    if sweep and d < 0:
        d += 2 * math.pi
    elif not sweep and d > 0:
        d -= 2 * math.pi
    els = list(_arc_elements(cx, cy, rx, ry, a0, d, phi, tolerance))
    if els:
        last = els[-1]
        els[-1] = ("C", last[1], last[2], last[3], last[4], x, y)  # land exactly on the endpoint
    yield from els


def parse_svg_path(d: str) -> List[tuple]:
    lx = _Lexer(d)
    els: List[tuple] = []
    cx = cy = 0.0  # current point
    sx = sy = 0.0  # subpath start
    last_ctrl = None  # for S/T reflection
    last_cmd = ""
    cmd = None
    while True:
        c = lx.peek_cmd()
        if c is not None:
            cmd = c
            lx.i += 1
        elif not lx.more_numbers():
            break
        elif cmd is None:
            raise ValueError("path data must start with a command")
        elif cmd in "Mm":
            cmd = "L" if cmd == "M" else "l"  # implicit line-to after move-to
        rel = cmd.islower()
        u = cmd.upper()
        if u == "Z":
            els.append(("Z",))
            cx, cy = sx, sy
            last_ctrl = None
            last_cmd = u
            if lx.more_numbers():
                raise ValueError("numbers after close-path")
            continue
        if u == "M":
            x, y = lx.num(), lx.num()
            if rel:
                x, y = cx + x, cy + y
            els.append(("M", x, y))
            cx, cy = sx, sy = x, y
            last_ctrl = None
        elif u == "L":
            x, y = lx.num(), lx.num()
            if rel:
                x, y = cx + x, cy + y
            els.append(("L", x, y))
            cx, cy = x, y
            last_ctrl = None
        elif u == "H":
            x = lx.num()
            if rel:
                x += cx
            els.append(("L", x, cy))
            cx = x
            last_ctrl = None
        elif u == "V":
            y = lx.num()
            if rel:
                y += cy
            els.append(("L", cx, y))
            cy = y
            last_ctrl = None
        elif u == "C":
            v = [lx.num() for _ in range(6)]
            if rel:
                v = [v[0] + cx, v[1] + cy, v[2] + cx, v[3] + cy, v[4] + cx, v[5] + cy]
            els.append(("C", *v))
            last_ctrl = (v[2], v[3])
            cx, cy = v[4], v[5]
        elif u == "S":
            v = [lx.num() for _ in range(4)]
            if rel:
                v = [v[0] + cx, v[1] + cy, v[2] + cx, v[3] + cy]
            if last_cmd in ("C", "S") and last_ctrl is not None:
                x1, y1 = 2 * cx - last_ctrl[0], 2 * cy - last_ctrl[1]
            else:
                x1, y1 = cx, cy
            els.append(("C", x1, y1, v[0], v[1], v[2], v[3]))
            last_ctrl = (v[0], v[1])
            cx, cy = v[2], v[3]
        elif u == "Q":
            v = [lx.num() for _ in range(4)]
            if rel:
                v = [v[0] + cx, v[1] + cy, v[2] + cx, v[3] + cy]
            els.append(("Q", *v))
            last_ctrl = (v[0], v[1])
            cx, cy = v[2], v[3]
        elif u == "T":
            v = [lx.num() for _ in range(2)]
            if rel:
                v = [v[0] + cx, v[1] + cy]
            if last_cmd in ("Q", "T") and last_ctrl is not None:
                x1, y1 = 2 * cx - last_ctrl[0], 2 * cy - last_ctrl[1]
            else:
                x1, y1 = cx, cy
            els.append(("Q", x1, y1, v[0], v[1]))
            last_ctrl = (x1, y1)
            cx, cy = v[0], v[1]
        elif u == "A":
            rx, ry, rot = lx.num(), lx.num(), lx.num()
            large, sweep = lx.flag(), lx.flag()
            x, y = lx.num(), lx.num()
            if rel:
                x, y = cx + x, cy + y
            els.extend(_svg_arc_to_cubics(cx, cy, rx, ry, rot, large, sweep, x, y))
            cx, cy = x, y
            last_ctrl = None
        else:
            raise ValueError(f"unsupported path command {cmd!r}")
        last_cmd = u
    return els


# ---------------------------------------------------------------------------------------------
# kurbo::dash (kurbo 0.13.1 stroke.rs `DashIterator`), which vello applies on the CPU before encoding a dashed stroke
# (vello/src/scene.rs:404-438). kurbo is a Cargo dependency that is not in the reference repository: the state machine below
# restates its published algorithm (stash the first dash of a closed subpath so that it can be joined to the last one,
# walk arc length with `dash_remaining` / `seg_remaining`, split segments with subsegment / inv_arclen). Lines -- the
# reference's `longpathdash` scene -- use closed forms and are exact; for curves kurbo's arclen / inv_arclen (adaptive
# Gauss-Legendre, ITP root finding, accuracy 1e-6) are replaced by a fixed-order composite Gauss-Legendre rule and
# bisection of the same accuracy class, so dash end points on curves agree with kurbo's to ~1e-6, not bit for bit
# ("parity unpinned" for dashed curves; the C++ front end uses the identical arithmetic, vb_scene.cpp).
# ---------------------------------------------------------------------------------------------
_GL8_X = (0.1834346424956498, 0.5255324099163290, 0.7966664774136267, 0.9602898564975363)
_GL8_W = (0.3626837833783620, 0.3137066458778873, 0.2223810344533745, 0.1012285362903763)


def _lerp(a, b, t):
    return (a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1]))


def _seg_eval(seg, t):
    k = seg[0]
    if k == "L":
        return _lerp(seg[1], seg[2], t)
    mt = 1.0 - t
    if k == "Q":
        p0, p1, p2 = seg[1:]
        return (mt * mt * p0[0] + 2.0 * mt * t * p1[0] + t * t * p2[0], mt * mt * p0[1] + 2.0 * mt * t * p1[1] + t * t * p2[1])
    p0, p1, p2, p3 = seg[1:]
    a, b, c, d = mt * mt * mt, 3.0 * mt * mt * t, 3.0 * mt * t * t, t * t * t
    return (a * p0[0] + b * p1[0] + c * p2[0] + d * p3[0], a * p0[1] + b * p1[1] + c * p2[1] + d * p3[1])


def _seg_deriv(seg, t):
    k = seg[0]
    mt = 1.0 - t
    if k == "Q":
        p0, p1, p2 = seg[1:]
        return (2.0 * (mt * (p1[0] - p0[0]) + t * (p2[0] - p1[0])), 2.0 * (mt * (p1[1] - p0[1]) + t * (p2[1] - p1[1])))
    p0, p1, p2, p3 = seg[1:]
    a, b, c = 3.0 * mt * mt, 6.0 * mt * t, 3.0 * t * t
    return (a * (p1[0] - p0[0]) + b * (p2[0] - p1[0]) + c * (p3[0] - p2[0]), a * (p1[1] - p0[1]) + b * (p2[1] - p1[1]) + c * (p3[1] - p2[1]))


def _curve_arclen_range(seg, t0, t1, pieces=16):
    """Arc length of a quad / cubic over [t0, t1]: composite 8-point Gauss-Legendre on `pieces` equal sub-ranges."""
    total = 0.0
    h = (t1 - t0) / pieces
    for i in range(pieces):
        a = t0 + h * i
        mid, half = a + 0.5 * h, 0.5 * h
        acc = 0.0
        for x, w in zip(_GL8_X, _GL8_W):
            d0 = _seg_deriv(seg, mid - half * x)
            d1 = _seg_deriv(seg, mid + half * x)
            acc += w * (math.sqrt(d0[0] * d0[0] + d0[1] * d0[1]) + math.sqrt(d1[0] * d1[0] + d1[1] * d1[1]))
        total += acc * half
    return total


def _seg_arclen(seg):
    if seg[0] == "L":
        dx, dy = seg[2][0] - seg[1][0], seg[2][1] - seg[1][1]
        return math.sqrt(dx * dx + dy * dy)
    return _curve_arclen_range(seg, 0.0, 1.0)


def _seg_inv_arclen(seg, s):
    """t with arclen(seg[0..t]) == s."""
    if seg[0] == "L":
        return s / _seg_arclen(seg)
    lo, hi = 0.0, 1.0
    for _ in range(48):  # bisection: 2^-48 in t
        mid = 0.5 * (lo + hi)
        if _curve_arclen_range(seg, 0.0, mid) < s:
            lo = mid
        else:
            hi = mid
    return 0.5 * (lo + hi)


def _seg_subsegment(seg, t0, t1):
    k = seg[0]
    if k == "L":
        return ("L", _seg_eval(seg, t0), _seg_eval(seg, t1))
    if k == "Q":  # kurbo QuadBez::subsegment
        p0, p2 = _seg_eval(seg, t0), _seg_eval(seg, t1)
        a = (seg[2][0] - seg[1][0], seg[2][1] - seg[1][1])
        b = (seg[3][0] - seg[2][0], seg[3][1] - seg[2][1])
        d = _lerp(a, b, t0)
        return ("Q", p0, (p0[0] + d[0] * (t1 - t0), p0[1] + d[1] * (t1 - t0)), p2)
    p0, p3 = _seg_eval(seg, t0), _seg_eval(seg, t1)  # kurbo CubicBez::subsegment
    scale = (t1 - t0) * (1.0 / 3.0)
    d0, d1 = _seg_deriv(seg, t0), _seg_deriv(seg, t1)
    return ("C", p0, (p0[0] + scale * d0[0], p0[1] + scale * d0[1]), (p3[0] - scale * d1[0], p3[1] - scale * d1[1]), p3)


def _seg_to_el(seg):
    k = seg[0]
    if k == "L":
        return ("L", seg[2][0], seg[2][1])
    if k == "Q":
        return ("Q", seg[2][0], seg[2][1], seg[3][0], seg[3][1])
    return ("C", seg[2][0], seg[2][1], seg[3][0], seg[3][1], seg[4][0], seg[4][1])


def dash(elements: Iterable[tuple], dash_offset: float, dashes) -> List[tuple]:
    """`kurbo::dash(inner, dash_offset, dashes)` collected into a list (as vello does, scene.rs:428-433)."""
    dashes = [float(d) for d in dashes]
    if not dashes:
        return list(elements)
    NEED_INPUT, TO_STASH, WORKING, FROM_STASH = range(4)
    inner = iter(list(elements))
    # place in the dash array for the initial offset
    dash_ix = 0
    dash_remaining = dashes[0] - dash_offset
    is_active = True
    while dash_remaining < 0.0:
        dash_ix = (dash_ix + 1) % len(dashes)
        dash_remaining += dashes[dash_ix]
        is_active = not is_active
    S = dict(input_done=False, closepath_pending=False, dash_ix=dash_ix, init_dash_ix=dash_ix, init_dash_remaining=dash_remaining,
             init_is_active=is_active, is_active=is_active, state=NEED_INPUT, seg=("L", (0.0, 0.0), (0.0, 0.0)), t=0.0,
             dash_remaining=dash_remaining, seg_remaining=0.0, start_pt=(0.0, 0.0), last_pt=(0.0, 0.0), stash=[], stash_ix=0)
    out: List[tuple] = []

    def reset_phase():
        S["dash_ix"], S["dash_remaining"], S["is_active"] = S["init_dash_ix"], S["init_dash_remaining"], S["init_is_active"]

    def handle_closepath():
        if S["state"] == TO_STASH:
            S["stash"].append(("Z",))  # looped back without breaking a dash: play it back closed
        elif S["is_active"]:
            S["stash_ix"] = 1          # connect with the path in the stash, skip its MoveTo
        S["state"] = FROM_STASH
        reset_phase()

    def get_input():
        while True:
            if S["closepath_pending"]:
                handle_closepath()
                break
            el = next(inner, None)
            if el is None:
                S["input_done"] = True
                S["state"] = FROM_STASH
                return
            p0 = S["last_pt"]
            k = el[0]
            if k == "M":
                if S["stash"]:
                    S["state"] = FROM_STASH
                S["start_pt"] = S["last_pt"] = (el[1], el[2])
                reset_phase()
                continue
            if k == "L":
                S["seg"] = ("L", p0, (el[1], el[2]))
                S["last_pt"] = (el[1], el[2])
            elif k == "Q":
                S["seg"] = ("Q", p0, (el[1], el[2]), (el[3], el[4]))
                S["last_pt"] = (el[3], el[4])
            elif k == "C":
                S["seg"] = ("C", p0, (el[1], el[2]), (el[3], el[4]), (el[5], el[6]))
                S["last_pt"] = (el[5], el[6])
            else:  # ClosePath
                S["closepath_pending"] = True
                if p0 != S["start_pt"]:
                    S["seg"] = ("L", p0, S["start_pt"])
                    S["last_pt"] = S["start_pt"]
                else:
                    continue
            S["seg_remaining"] = _seg_arclen(S["seg"])
            break
        S["t"] = 0.0

    def step():
        result = None
        if S["state"] == TO_STASH and not S["stash"]:
            if S["is_active"]:
                p = S["seg"][1]
                result = ("M", p[0], p[1])
            else:
                S["state"] = WORKING
        elif S["dash_remaining"] < S["seg_remaining"]:
            seg = _seg_subsegment(S["seg"], S["t"], 1.0)  # next transition is a dash transition
            t1 = _seg_inv_arclen(seg, S["dash_remaining"])
            if S["is_active"]:
                result = _seg_to_el(_seg_subsegment(seg, 0.0, t1))
                S["state"] = WORKING
            else:
                p = _seg_eval(seg, t1)
                result = ("M", p[0], p[1])
            S["is_active"] = not S["is_active"]
            S["t"] += t1 * (1.0 - S["t"])
            S["seg_remaining"] -= S["dash_remaining"]
            S["dash_ix"] += 1
            if S["dash_ix"] == len(dashes):
                S["dash_ix"] = 0
            S["dash_remaining"] = dashes[S["dash_ix"]]
        else:
            if S["is_active"]:
                result = _seg_to_el(_seg_subsegment(S["seg"], S["t"], 1.0))
            S["dash_remaining"] -= S["seg_remaining"]
            get_input()
        return result

    guard = 0
    while True:
        guard += 1
        assert guard < 100_000_000
        st = S["state"]
        if st == NEED_INPUT:
            if S["input_done"]:
                break
            get_input()
            if S["input_done"]:
                # FROM_STASH drains whatever was stashed (kurbo returns None here only when the stash is empty)
                if not S["stash"]:
                    break
                continue
            S["state"] = TO_STASH
        elif st == TO_STASH:
            el = step()
            if el is not None:
                S["stash"].append(el)
        elif st == WORKING:
            el = step()
            if el is not None:
                out.append(el)
        else:  # FROM_STASH
            if S["stash_ix"] < len(S["stash"]):
                out.append(S["stash"][S["stash_ix"]])
                S["stash_ix"] += 1
            else:
                S["stash"].clear()
                S["stash_ix"] = 0
                if S["input_done"]:
                    break
                if S["closepath_pending"]:
                    S["closepath_pending"] = False
                    S["state"] = NEED_INPUT
                else:
                    S["state"] = TO_STASH
    return out
