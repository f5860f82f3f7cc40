"""A float64 statement of vello's paints -- what colour a covered pixel gets -- independent of the CUDA kernels and of the
oracle's float32 restatement of them. No CUDA, no oracle.

- `ramp`: the 512 texels of a gradient ramp (ramp_cache.rs `make_ramp`).
- `gradient_t` / `texel_index`: the ramp parameter of a linear, radial or sweep gradient at a pixel, and its texel.
- `image_sample`: nearest, bilinear and bicubic image sampling (fine.wgsl, CMD_IMAGE).
- `blur_rect`: the blurred rounded rectangle's alpha (fine.wgsl, CMD_BLUR_RECT).

Where fine evaluates a paint (k_fine.cu): gradients and blurred rectangles at the pixel's top-left CORNER (PXX(i), xyy: the
integer pixel coordinates), images at the pixel's CENTRE (PXX(i) + 0.5, xyy + 0.5). `corner_grid` / `centre_grid` give those
points for a frame.

Transforms are kurbo affines (a, b, c, d, e, f): (x, y) -> (a x + c y + e, b x + d y + f)."""
from __future__ import annotations

import math
from typing import Sequence, Tuple

import numpy as np

GRADIENT_WIDTH = 512
EXTEND_PAD, EXTEND_REPEAT, EXTEND_REFLECT = 0, 1, 2
QUALITY_LOW, QUALITY_MEDIUM, QUALITY_HIGH = 0, 1, 2
GRADIENT_EPSILON = 2.0 ** -12  # draw_leaf.wgsl: the strip and focal-on-circle tests


def corner_grid(w: int, h: int):
    """The points where fine evaluates gradients and blurred rectangles: pixel (x, y) at (x, y)."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    return x, y


def centre_grid(w: int, h: int):
    """The points where fine samples images: pixel (x, y) at (x + 0.5, y + 0.5)."""
    x, y = corner_grid(w, h)
    return x + 0.5, y + 0.5


def apply(m, x, y):
    a, b, c, d, e, f = (float(v) for v in m)
    return a * x + c * y + e, b * x + d * y + f


def inverse(m):
    a, b, c, d, e, f = (float(v) for v in m)
    det = a * d - b * c
    ia, ib, ic, id_ = d / det, -b / det, -c / det, a / det
    return (ia, ib, ic, id_, -(ia * e + ic * f), -(ib * e + id_ * f))


# ---- ramps ----------------------------------------------------------------------------------------------------------------
def _premul_rgba8(c: np.ndarray) -> np.ndarray:
    """Straight RGBA (..., 4) in 0..1 -> premultiplied RGBA8 with the encoder's rounding (floor(255 v + 0.5), clamped)."""
    p = np.concatenate([c[..., :3] * c[..., 3:4], c[..., 3:4]], axis=-1)
    return np.clip(np.floor(p * 255.0 + 0.5), 0, 255).astype(np.uint8)


def ramp(stops: Sequence[Tuple[float, Tuple[float, float, float, float]]], premul_interp: bool) -> np.ndarray:
    """(512, 4) uint8 premultiplied RGBA8: ramp_cache.rs `make_ramp` in float64. Stops are (offset, (r, g, b, a)) with straight
    colours. Texel i samples u = i / 511 and walks the stops the way make_ramp does:
    - the walk starts at u = 0 with the FIRST stop's colour, whatever its offset (an offset below 0, or above 0, of the first
      stop only moves where the first segment ends);
    - past the last stop every texel takes the last stop's colour (padding with the end colour);
    - a hard stop (two stops at one offset) resolves to the first of them at u equal to that offset and to the later one above
      it; a segment shorter than 1e-9 takes the colour of its end;
    - straight interpolation lerps the straight components; premultiplied interpolation lerps the premultiplied components
      and un-premultiplies, except where the lerped alpha is exactly 0 or 1 (there the premultiplied value is kept);
    then premultiply and round to RGBA8."""
    offs = [float(np.float32(o)) for o, _ in stops]  # offsets travel in f32
    cols = [np.array(c, dtype=np.float64) for _, c in stops]
    out = np.zeros((GRADIENT_WIDTH, 4), dtype=np.float64)
    last_u, last_c = 0.0, cols[0]
    this_u, this_c = last_u, last_c
    j = 0
    for i in range(GRADIENT_WIDTH):
        u = i / (GRADIENT_WIDTH - 1)
        while u > this_u:
            last_u, last_c = this_u, this_c
            if j + 1 < len(stops):
                this_u, this_c = offs[j + 1], cols[j + 1]
                j += 1
            else:
                break
        du = this_u - last_u
        if du < 1e-9:
            c = this_c
        else:
            t = (u - last_u) / du
            if premul_interp:
                pa = np.concatenate([last_c[:3] * last_c[3], last_c[3:]])
                pb = np.concatenate([this_c[:3] * this_c[3], this_c[3:]])
                pc = pa + (pb - pa) * t
                c = pc if pc[3] == 0.0 or pc[3] == 1.0 else np.concatenate([pc[:3] / pc[3], pc[3:]])
            else:
                c = last_c + (this_c - last_c) * t
        out[i] = c
    return _premul_rgba8(out)


def ramp_u32(r: np.ndarray) -> np.ndarray:
    """(512, 4) uint8 -> (512,) uint32 with r in the low byte (the renderer's ramp rows)."""
    return np.ascontiguousarray(r).view(np.uint32).reshape(-1)


# ---- gradients -------------------------------------------------------------------------------------------------------------
def extend(t, mode: int):
    """pad: clamp to [0, 1]; repeat: t - floor(t); reflect: |t - 2 round(t / 2)| (fine.wgsl extend_mode_normalized)."""
    t = np.asarray(t, dtype=np.float64)
    if mode == EXTEND_PAD:
        return np.clip(t, 0.0, 1.0)
    if mode == EXTEND_REPEAT:
        return t - np.floor(t)
    return np.abs(t - 2.0 * np.round(0.5 * t))


def texel_index(t_ext):
    """round(511 t) of an extended t, ties to even; a NaN t (see `gradient_t`) is texel 0."""
    t = np.asarray(t_ext, dtype=np.float64)
    k = np.round(np.where(np.isnan(t), 0.0, t) * (GRADIENT_WIDTH - 1))
    return k.astype(np.int64)


def sweep_poly(s):
    """Skia's polynomial for atan(s) / (2 pi), 0 <= s <= 1, which vello's sweep gradient uses for the angle."""
    ss = s * s
    return s * (0.15912117063999176025390625 + ss * (-5.185396969318389892578125e-2 + ss * (
        2.476101927459239959716796875e-2 + ss * (-7.0547382347285747528076171875e-3))))


def _radial_limits(c0x, c0y, c1x, c1y, r0, r1):
    """The cone vello paints for a two-point conical gradient (draw_leaf.wgsl), as cone parameters. Two tolerances make it
    paint a limit instead of the cone it was given:
    - |r0 - r1| <= 2^-12 (with c0 != c1): the strip kind, a cylinder of radius r0: r1 becomes r0;
    - otherwise, with f = r0 / (r0 - r1) (the focal point c0 + f (c1 - c0); r0 and r1 swapped first, c0 with c1, when r1 is 0)
      and radius = r1 / |focal point - c1|: |radius - 1| <= 2^-12 is the focal-on-circle kind, the cone through the same focal
      point and circle centre whose radius ratio is exactly 1: r1 becomes |focal point - c1| and r0 becomes f r1 / (f - 1).
    Every other input is returned as it is. (c0 == c1 never meets the second rule: its radius is infinite.)"""
    if abs(r0 - r1) <= GRADIENT_EPSILON:
        return c0x, c0y, c1x, c1y, r0, r0
    if (c0x, c0y) == (c1x, c1y):
        return c0x, c0y, c1x, c1y, r0, r1
    swapped = r1 == 0.0
    if swapped:
        c0x, c0y, c1x, c1y, r0, r1 = c1x, c1y, c0x, c0y, r1, r0
    f = r0 / (r0 - r1)
    fx, fy = c0x + f * (c1x - c0x), c0y + f * (c1y - c0y)
    dist = math.hypot(fx - c1x, fy - c1y)
    if abs(r1 / dist - 1.0) <= GRADIENT_EPSILON:
        r1 = dist
        r0 = f * r1 / (f - 1.0)
    if swapped:
        c0x, c0y, c1x, c1y, r0, r1 = c1x, c1y, c0x, c0y, r1, r0
    return c0x, c0y, c1x, c1y, r0, r1


def gradient_t(kind: str, params, transform, x, y):
    """The ramp parameter t at device points (x, y) (before the extend mode) and a mask of the points the gradient paints.

    `params` are the encoder's: linear (p0x, p0y, p1x, p1y); radial (c0x, c0y, c1x, c1y, r0, r1); sweep (cx, cy, t0, t1) with
    t0 / t1 in turns (the encoder divides the angles by 2 pi). `transform` maps gradient space to device space (the fill's
    transform times its brush transform).

    - linear: vello transforms p0 and p1 to device space (draw_leaf) and projects there: t = (q - p0') . (p1' - p0') /
      |p1' - p0'|^2. p0 == p1 is a NaN t: texel 0 in every extend mode (vb_f2i_sat of NaN; the NaN survives clamp, fract and
      the reflection).
    - radial: the two-point conical gradient itself. The point q = transform^-1 (x, y) is painted with the greatest t for which
      |q - c(t)| = r(t) and r(t) >= 0, where c(t) = c0 + t (c1 - c0) and r(t) = r0 + t (r1 - r0); with no such t the pixel is not
      painted. The cone is the one vello paints: within 2^-12 of a strip or of a focal point on the end circle, its limit
      (`_radial_limits`). Degenerate inputs: c0 == c1 with |r0 - r1| below 2^-12 is transparent (the encoder); with |r0 - r1|
      exactly 2^-12 draw_leaf takes the strip branch and divides by |c0 - c1| = 0, so nothing is painted either. vello's
      circular kind moves c0 by 2^-12 (draw_leaf), which this statement does not: the cases bound that difference.
    - sweep: phi = the angle of q - centre in turns, in [0, 1) (atan2, y down, so clockwise on screen), plus the error of
      the atan polynomial vello evaluates it with (`sweep_poly`, at most 2.7e-5 turns), then t = (phi - t0) / (t1 - t0). At
      the centre itself the angle is 0 (the shader's NaN test)."""
    inv = inverse(transform)
    if kind == "linear":
        p0 = apply(transform, params[0], params[1])
        p1 = apply(transform, params[2], params[3])
        dx, dy = p1[0] - p0[0], p1[1] - p0[1]
        n = dx * dx + dy * dy
        if n == 0.0:
            return np.full(np.shape(x), np.nan), np.ones(np.shape(x), bool)
        return ((x - p0[0]) * dx + (y - p0[1]) * dy) / n, np.ones(np.shape(x), bool)
    qx, qy = apply(inv, x, y)
    if kind == "sweep":
        dx, dy = qx - params[0], qy - params[1]
        with np.errstate(divide="ignore", invalid="ignore"):
            phi = np.arctan2(dy, dx) / (2.0 * math.pi)
            phi = np.where(phi < 0.0, phi + 1.0, phi)
            phi = np.where(phi >= 1.0, 0.0, phi)
            # vello's angle is Skia's 7th-degree polynomial of atan (fine.wgsl), off the true angle by up to 2.7e-5 turns
            # (0.014 texels): add its error, signed by how the octant folds the polynomial's value into the turn
            ax, ay = np.abs(dx), np.abs(dy)
            s = np.minimum(ax, ay) / np.maximum(ax, ay)
            s = np.where(np.isnan(s), 0.0, s)
            err = sweep_poly(s) - np.arctan(s) / (2.0 * math.pi)
            flips = (ax < ay).astype(int) + (dx < 0.0).astype(int) + (dy < 0.0).astype(int)
            phi = phi + np.where(flips % 2 == 1, -err, err)
        return (phi - params[2]) / (params[3] - params[2]), np.ones(np.shape(x), bool)
    c0x, c0y, c1x, c1y, r0, r1 = _radial_limits(*(float(v) for v in params))
    dcx, dcy, dr = c1x - c0x, c1y - c0y, r1 - r0
    if dcx == 0.0 and dcy == 0.0 and abs(dr) <= GRADIENT_EPSILON:
        return np.zeros(np.shape(x)), np.zeros(np.shape(x), bool)
    px, py = qx - c0x, qy - c0y
    a = dcx * dcx + dcy * dcy - dr * dr
    b = px * dcx + py * dcy + r0 * dr
    c = px * px + py * py - r0 * r0
    with np.errstate(divide="ignore", invalid="ignore"):
        if a == 0.0:
            t = c / (2.0 * b)
            ok = (b != 0.0) & (r0 + t * dr >= 0.0)
            return np.where(ok, t, 0.0), ok
        disc = b * b - a * c
        s = np.sqrt(np.maximum(disc, 0.0))
        hi, lo = (b + s) / a, (b - s) / a
        if a < 0.0:
            hi, lo = lo, hi
        hi_ok = (disc >= 0.0) & (r0 + hi * dr >= 0.0)
        lo_ok = (disc >= 0.0) & (r0 + lo * dr >= 0.0)
        t = np.where(hi_ok, hi, lo)
        return np.where(hi_ok | lo_ok, t, 0.0), hi_ok | lo_ok


# ---- images ----------------------------------------------------------------------------------------------------------------
_MF = np.array([
    [(1 / 6) / 3, -(3 / 6) / 3 - 1 / 3, (3 / 6) / 3 + 2 / 3, -(1 / 6) / 3 - 1 / 3],
    [1 - (2 / 6) / 3, 0.0, -3 + (12 / 6) / 3 + 1 / 3, 2 - (9 / 6) / 3 - 1 / 3],
    [(1 / 6) / 3, (3 / 6) / 3 + 1 / 3, 3 - (15 / 6) / 3 - 2 / 3, -2 + (9 / 6) / 3 + 1 / 3],
    [0.0, 0.0, -1 / 3, (1 / 6) / 3 + 1 / 3],
])


def cubic_weights(fr):
    """The Mitchell-Netravali B = C = 1/3 weights of the taps at -1.5, -0.5, 0.5, 1.5 (fine.wgsl cubic_weights): (4, ...)."""
    fr = np.asarray(fr, dtype=np.float64)
    return np.stack([m[0] + fr * (m[1] + fr * (m[2] + fr * m[3])) for m in _MF])


def _extend_axis(u, mode: int, size: float):
    if mode == EXTEND_PAD:
        return np.clip(u, 0.0, size)
    return extend(u / size, mode) * size


def image_sample(pixels: np.ndarray, x, y, transform, quality: int = QUALITY_MEDIUM, x_extend: int = EXTEND_PAD,
                 y_extend: int = EXTEND_PAD, premultiplied: bool = False, bgra: bool = False, alpha8: int = 255) -> np.ndarray:
    """The premultiplied RGBA (..., 4) float64 colour fine paints at device points (x, y) -- pass `centre_grid` points -- for
    the image `pixels` ((h, w, 4) uint8, in its own format) drawn with `transform` (image space to device space).

    u, v = transform^-1 (x, y), extended per axis (pad: clamp to [0, size]; repeat / reflect of u / size, times size). Samples
    read only the image's own texels: every tap is clamped to [0, size - 1] per axis before it is truncated to a texel.
    - nearest: texel (trunc(clamp(u)), trunc(clamp(v))).
    - bilinear: u' = u - 1/2; the taps are floor and ceil of clamp(u'), weighted by u' - floor(u') of the UNclamped u'.
    - bicubic: taps at u + {-1.5, -0.5, 0.5, 1.5}, weights `cubic_weights(fract(u + 1/2))`; the sum's alpha is clamped to
      [0, 1] and its colour to [0, alpha].
    Each tap is premultiplied first unless the image is premultiplied. The result is scaled by alpha8 / 255 (the brush's alpha
    byte) and, for a BGRA image, its first and third channels are swapped."""
    h, w = pixels.shape[:2]
    px = pixels.astype(np.float64) / 255.0
    if not premultiplied:
        px = np.concatenate([px[..., :3] * px[..., 3:4], px[..., 3:4]], axis=-1)
    u, v = apply(inverse(transform), np.asarray(x, np.float64), np.asarray(y, np.float64))
    u = _extend_axis(u, x_extend, float(w))
    v = _extend_axis(v, y_extend, float(h))

    def tap(uu, vv):
        iu = np.clip(uu, 0.0, w - 1.0).astype(np.int64)
        iv = np.clip(vv, 0.0, h - 1.0).astype(np.int64)
        return px[iv, iu]

    if quality == QUALITY_LOW:
        out = tap(u, v)
    elif quality == QUALITY_HIGH:
        # the taps u - 1.5 .. u + 1.5 truncate to floor(u + 1/2) - 2 .. floor(u + 1/2) + 1: taken from the same floor as the
        # weights, so that a u whose u + 1/2 rounds to an integer cannot pair the weights of one texel with the taps of the next
        bu, bv = np.floor(u + 0.5), np.floor(v + 0.5)
        wx, wy = cubic_weights((u + 0.5) - bu), cubic_weights((v + 0.5) - bv)
        out = np.zeros(np.shape(u) + (4,))
        for j in range(4):
            for i in range(4):
                out += (wx[i] * wy[j])[..., None] * tap(bu + (i - 2), bv + (j - 2))
        a = np.clip(out[..., 3], 0.0, 1.0)
        out = np.concatenate([np.clip(out[..., :3], 0.0, a[..., None]), a[..., None]], axis=-1)
    else:
        u, v = u - 0.5, v - 0.5
        uc, vc = np.clip(u, 0.0, w - 1.0), np.clip(v, 0.0, h - 1.0)
        fu, fv = (u - np.floor(u))[..., None], (v - np.floor(v))[..., None]
        x0, x1, y0, y1 = np.floor(uc), np.ceil(uc), np.floor(vc), np.ceil(vc)
        top = tap(x0, y0) * (1 - fv) + tap(x0, y1) * fv
        bot = tap(x1, y0) * (1 - fv) + tap(x1, y1) * fv
        out = top * (1 - fu) + bot * fu
    out = out * (alpha8 / 255.0)
    if bgra:
        out = out[..., [2, 1, 0, 3]]
    return out


def stored(c: np.ndarray) -> np.ndarray:
    """Premultiplied float RGBA (..., 4) -> the float RGBA a frame stores before rounding: fine un-premultiplies its result
    (rgb / max(a, 1e-6)), and the frame holds straight-alpha RGBA8 (round to nearest of 255 v)."""
    c = np.asarray(c, dtype=np.float64)
    a = c[..., 3:4]
    return np.clip(np.concatenate([c[..., :3] / np.maximum(a, 1e-6), a], axis=-1), 0.0, 1.0) * 255.0


def stored_texel(u32):
    """A premultiplied RGBA8 texel (uint32, r in the low byte) as a frame stores it: fine's output step in float32, exactly
    (unpack as byte / 255, multiply by 1 / max(a, 1e-6), floor(0.5 + 255 v)). A gradient pixel of full coverage over a
    transparent base is its ramp texel exactly, so its stored value is this."""
    f = np.float32
    b = np.stack([(np.asarray(u32, np.uint32) >> s) & 0xFF for s in (0, 8, 16, 24)], -1).astype(f) / f(255.0)
    a_inv = f(1.0) / np.maximum(b[..., 3:4], f(1e-6))
    v = np.concatenate([b[..., :3] * a_inv, b[..., 3:4]], axis=-1)
    q = np.floor(f(0.5) + f(255.0) * np.clip(v, f(0.0), f(1.0))).astype(np.uint32)
    return q[..., 0] | (q[..., 1] << 8) | (q[..., 2] << 16) | (q[..., 3] << 24)


# ---- blurred rounded rectangles ----------------------------------------------------------------------------------------------
def _erf7(x):
    """fine.wgsl erf7: vello's approximation of erf, which is part of the paint's definition."""
    y = np.clip(x * 1.1283791671, -100.0, 100.0)
    yy = y * y
    z = y + (0.24295 + (0.03395 + 0.0104 * yy) * yy) * (y * yy)
    return z / np.sqrt(1.0 + z * z)


def blur_rect(x, y, transform, width: float, height: float, radius: float, std_dev: float):
    """The alpha (0..1) of a blurred rounded rectangle at device points (x, y) -- pass `corner_grid` points. `transform` maps
    the rectangle's centred frame to device space (Scene.draw_blurred_rounded_rect: the fill's transform times a translation
    to the rectangle's centre); fine.wgsl CMD_BLUR_RECT, in float64, with sigma floored at 1e-5 as there."""
    bw, bh, rad = float(width), float(height), float(radius)
    sd = max(float(std_dev), 1e-5)
    lx, ly = apply(inverse(transform), np.asarray(x, np.float64), np.asarray(y, np.float64))
    inv = 1.0 / sd
    min_edge = min(bw, bh)
    rmax = 0.5 * min_edge
    r0 = min(math.hypot(rad, sd * 1.15), rmax)
    r1 = min(math.hypot(rad, sd * 2.0), rmax)
    exponent = 2.0 * r1 / r0 if r0 != 0.0 else math.nan  # a zero-width or zero-height rectangle: 0 / 0
    ew, eh = 0.5 * inv * bw, 0.5 * inv * bh
    delta = 1.25 * sd * (math.exp(-ew * ew) - math.exp(-eh * eh))
    w = bw + min(delta, 0.0)
    h = bh - max(delta, 0.0)
    scale = 0.5 * _erf7(inv * 0.5 * (max(w, h) - 0.5 * rad))
    y0 = np.abs(ly) - (h * 0.5 - r1)
    x0 = np.abs(lx) - (w * 0.5 - r1)
    x1, y1 = np.maximum(x0, 0.0), np.maximum(y0, 0.0)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d_pos = (x1 ** exponent + y1 ** exponent) ** (1.0 / exponent) if not math.isnan(exponent) else np.full(np.shape(x1), np.nan)
    d = d_pos + np.minimum(np.maximum(x0, y0), 0.0) - r1
    return scale * (_erf7(inv * (min_edge + d)) - _erf7(inv * d))
