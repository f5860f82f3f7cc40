"""Paint edge cases -- gradients, images and blurred rectangles at the inputs where their formulas branch -- checked against the
float64 statement of the paints in paint_ref.py, here on the CPU oracle's full pipeline (test_gpu_paint_edges.py runs the same
cases on the GPU). A case that fails here points at the reference or the oracle, so that a GPU failure points at the kernel.

Every case fills whole-pixel, axis-aligned rectangles (coverage exactly 1) with one paint over a transparent base, so every
covered pixel is the paint's own premultiplied colour (which the frame stores un-premultiplied, as fine does).

- Gradient pixels are exactly ramp[k], k from the reference. A neighbouring texel is accepted only where 511 t lies within
  the case's float32 error bound (`bound`, in texels) of a half-integer -- or, in repeat mode, of a whole turn, where the
  texel wraps between 0 and 511. Radial pixels within `edge` pixels of the painted region's edge are skipped. At most 1 % of
  a case's pixels may be exempt in either way, so no case passes by exempting everything. The cases just past a radial
  tolerance, where vello's own float32 formula cancels, say so and accept the texels within `spread` of the reference's.
- Image pixels are within 1 LSB of the reference and blurred rectangles within the case's stated bound, both compared in
  premultiplied RGBA8 (`_premul_diff`)."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np
import pytest

from vello_b200.config import AA_AREA
from vello_b200.encoding import (EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT, FILL_NON_ZERO, Color, Gradient, Image, Scene,
                                 resolve)
from vello_b200.shapes import Affine, Rect

from . import paint_ref as P

ALPHA_STRAIGHT, ALPHA_PREMUL = 0, 1
FORMAT_RGBA, FORMAT_BGRA = 0, 1
IDENT = (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)


def stop(o, r, g, b, a=1.0):
    return (o, Color(r, g, b, a))


# a ramp whose neighbouring texels always differ, so that a texel off by one shows
RAINBOW = [stop(0.0, 1, 0, 0), stop(0.33, 0, 1, 0), stop(0.66, 0, 0, 1), stop(1.0, 1, 1, 0.2, 0.6)]


def _affine(m):
    return Affine(tuple(float(v) for v in m))


@dataclass
class Case:
    """One paint over the whole w x h frame. kind: linear / radial / sweep / image / blur."""
    name: str
    kind: str
    w: int = 64
    h: int = 64
    params: tuple = ()
    stops: list = field(default_factory=lambda: list(RAINBOW))
    extend: int = EXTEND_PAD
    premul: bool = True
    brush: tuple = IDENT  # gradient / image brush transform (the fill's transform is the identity)
    bound: float = 2e-3  # texels of float32 error (gradients) or LSB (blur)
    edge: float = 0.0  # radial: pixels skipped at the painted region's edge
    image: Optional[Callable] = None  # image cases: () -> list of (Image, transform); the last is checked
    blur: tuple = ()  # (rect x0, y0, x1, y1, radius, std_dev)
    note: str = ""
    nan_info: bool = False  # draw_leaf writes NaNs into the paint's info words (degenerate geometry)
    spread: int = 0  # > 0: float32 cancellation in vello's own formula; any texel within `spread` of the reference's
    f32_t: bool = False  # t is exact in float32 at every pixel: the texel index takes fine's float32 product 511 t

    def scene(self):
        s = Scene()
        if self.kind in ("linear", "radial", "sweep"):
            g = Gradient(self.kind, tuple(self.params), list(self.stops), self.extend, self.premul)
            s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), g, _affine(self.brush), Rect(0, 0, self.w, self.h))
        elif self.kind == "image":
            ims = self.image()
            for i, (im, m) in enumerate(ims):  # the images before the last only take their atlas slots, outside the frame
                r = Rect(0, 0, self.w, self.h) if i == len(ims) - 1 else Rect(-8, -8, -4, -4)
                s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), im, _affine(m), r)
        else:
            x0, y0, x1, y1, rad, sd = self.blur
            s.draw_blurred_rounded_rect_in(Rect(0, 0, self.w, self.h), Affine.translate(0.0, 0.0), Rect(x0, y0, x1, y1),
                                           Color(0.2, 0.6, 1.0, 0.8), rad, sd)
        return s


def _grad_params(kind, p):
    """The encoder's gradient parameters -> gradient_t's (sweep angles in turns as the encoder stores them, in f32)."""
    f = np.float32
    if kind == "sweep":
        tau = f(2.0 * math.pi)
        return (float(f(p[0])), float(f(p[1])), float(f(f(p[2]) / tau)), float(f(f(p[3]) / tau)))
    return tuple(float(f(v)) for v in p)


def _premul_diff(img: np.ndarray, ref: np.ndarray) -> np.ndarray:
    """|frame - reference| in LSB of premultiplied RGBA8, less the frame's own rounding. A frame holds straight alpha (fine
    un-premultiplies), which amplifies float32 noise wherever alpha is near 0; so the frame is premultiplied again
    (colour * alpha / 255), and the half LSB each that rounding the colour and the alpha put into that product is allowed on top
    of the comparison's own 1 LSB."""
    g = img.astype(np.float64)
    got = np.concatenate([g[..., :3] * g[..., 3:4] / 255.0, g[..., 3:4]], axis=-1)
    d = np.abs(got - np.clip(ref, 0.0, 1.0) * 255.0)
    slack = np.concatenate([np.full(g.shape[:-1] + (3,), 1.0), np.full(g.shape[:-1] + (1,), 0.0)], axis=-1)
    return np.maximum(d - slack, 0.0)


def check_pixels(case: Case, img: np.ndarray, ramps: np.ndarray):
    """Assert that the frame `img` ((h, w, 4) uint8) is the case's paint; `ramps` are the ramp rows the frame read."""
    w, h = case.w, case.h
    got = np.ascontiguousarray(img).view(np.uint32).reshape(h, w)
    if case.kind in ("linear", "radial", "sweep"):
        params = _grad_params(case.kind, case.params)
        x, y = P.corner_grid(w, h)
        t, valid = P.gradient_t(case.kind, params, case.brush, x, y)
        te = P.extend(t, case.extend)
        k = P.texel_index(te)
        u = np.nan_to_num(te) * (P.GRADIENT_WIDTH - 1)  # a NaN t is texel 0
        if case.f32_t:
            # the geometry makes t exact in float32, so fine's t is the reference's; its product t * 511 is a float32
            # product, which can round to a tie that the exact product is not
            assert np.array_equal(te.astype(np.float32).astype(np.float64), te)
            u = (te.astype(np.float32) * np.float32(P.GRADIENT_WIDTH - 1)).astype(np.float64)
            k = np.round(u).astype(np.int64)
        row = P.stored_texel(ramps[0] if len(ramps) else np.zeros(P.GRADIENT_WIDTH, np.uint32))
        want = np.where(valid, row[np.clip(k, 0, 511)], 0)
        near = np.abs(u - np.floor(u) - 0.5) < case.bound
        lo, hi = np.clip(np.floor(u), 0, 511).astype(np.int64), np.clip(np.floor(u) + 1, 0, 511).astype(np.int64)
        wrap = np.zeros_like(near)
        if case.extend == EXTEND_REPEAT:
            wrap = np.abs(t - np.round(t)) * (P.GRADIENT_WIDTH - 1) < case.bound
        ok = (got == want) | (valid & near & ((got == row[lo]) | (got == row[hi]))) | \
             (valid & wrap & ((got == row[0]) | (got == row[511])))
        skip = np.zeros_like(ok)
        if case.edge > 0:
            for ddx, ddy in ((-1, -1), (-1, 1), (1, -1), (1, 1)):
                _, v2 = P.gradient_t(case.kind, params, case.brush, x + ddx * case.edge, y + ddy * case.edge)
                skip |= v2 != valid
        if case.spread:
            for dk in range(-case.spread, case.spread + 1):
                ok |= valid & (got == row[np.clip(k + dk, 0, 511)])
        exempt = (valid & (near | wrap)) | skip
        bad = ~ok & ~skip
        assert not bad.any(), f"{case.name}: {int(bad.sum())} pixels differ from ramp[k], first at {tuple(np.argwhere(bad)[0])}: " \
                              f"got {got[bad][0]:#010x} want {want[bad][0]:#010x} (t = {t[bad][0]!r})"
        if not case.spread:
            assert exempt.mean() <= 0.01, f"{case.name}: {exempt.mean():.2%} of the pixels exempt"
    elif case.kind == "image":
        im, m = case.image()[-1]
        x, y = P.centre_grid(w, h)
        a8 = int(np.float32(im.alpha) * np.float32(255.0) + np.float32(0.5)) & 0xFF
        ref = P.image_sample(im.data, x, y, m, im.quality, im.x_extend, im.y_extend, im.alpha_type == ALPHA_PREMUL,
                             im.format == FORMAT_BGRA, a8)
        d = _premul_diff(img, ref)
        assert d.max() <= 1.0, f"{case.name}: max |diff| {d.max():.3f} LSB at {tuple(np.argwhere(d > 1.0)[0])}"
    else:
        x0, y0, x1, y1, rad, sd = case.blur
        x, y = P.corner_grid(w, h)
        m = (1.0, 0.0, 0.0, 1.0, 0.5 * (x0 + x1), 0.5 * (y0 + y1))
        a = P.blur_rect(x, y, m, x1 - x0, y1 - y0, rad, sd)
        col = np.array([0.2 * 0.8, 0.6 * 0.8, 1.0 * 0.8, 0.8])
        c8 = np.floor(col * 255.0 + 0.5) / 255.0  # the colour travels as premultiplied RGBA8
        ref = c8[None, None, :] * a[..., None]
        if np.isnan(a).any():
            assert np.isnan(a).all() and not img.any(), f"{case.name}: a NaN alpha must store as 0"
            return
        d = _premul_diff(img, ref)
        assert d.max() <= case.bound, f"{case.name}: max |diff| {d.max():.3f} LSB (bound {case.bound})"


# ---- the cases ----------------------------------------------------------------------------------------------------------------
ROT = (math.cos(0.4), math.sin(0.4), -math.sin(0.4), math.cos(0.4), 30.0, -7.0)
SHEAR = (1.0, 0.35, -0.6, 1.2, 5.0, 3.0)
MIRROR = (-1.0, 0.0, 0.0, 1.0, 64.0, 0.0)
NONUNIFORM = (1.7, 0.3, -0.2, 0.6, 4.0, 9.0)

LINEAR = [
    Case("lin_short_pad", "linear", params=(20.3, 5.0, 20.301, 5.0)),
    Case("lin_long_pad", "linear", params=(-4e5, 3.0, 6e5, 3.0)),
    Case("lin_p0_eq_p1", "linear", params=(10.0, 10.0, 10.0, 10.0), nan_info=True),
    Case("lin_p0_eq_p1_repeat", "linear", params=(10.0, 10.0, 10.0, 10.0), extend=EXTEND_REPEAT, nan_info=True),
    # t = x / 1024 exactly in f32, so 511 t = 255.5 at x = 512: a tie, which rounds to the even texel 256
    Case("lin_texel_tie", "linear", w=600, h=4, params=(0.0, 0.0, 1024.0, 0.0), bound=0.0, f32_t=True),
    # t = (x - p0x) / 1024 exactly in f32; at x = 520, t = 131585 / 2^18 and the float32 product 511 t rounds to the tie
    # 256.5, whose floor is even: rint gives 256, round-half-away 257
    Case("lin_texel_tie_even_floor", "linear", w=600, h=4, params=(520.0 - 514.00390625, 0.0, 520.0 - 514.00390625 + 1024.0, 0.0),
         bound=0.0, f32_t=True),
    # t = 512 (x + y) + c exactly in f32, |t| up to 10^4: the extend modes' arithmetic far from [0, 1]
    Case("lin_big_t_repeat", "linear", w=16, h=16, params=(-9.765625 + 2 ** -12, 0.0, -9.765625 + 2 ** -12 + 2 ** -10, 2 ** -10),
         extend=EXTEND_REPEAT, bound=0.0, f32_t=True),
    Case("lin_big_t_reflect", "linear", w=16, h=16, params=(-9.765625 + 2 ** -12, 0.0, -9.765625 + 2 ** -12 + 2 ** -10, 2 ** -10),
         extend=EXTEND_REFLECT, bound=0.0, f32_t=True),
    Case("lin_big_neg_t_reflect", "linear", w=16, h=16, params=(19.53125 + 3 * 2 ** -12, 0.0, 19.53125 + 3 * 2 ** -12 + 2 ** -10,
                                                                 2 ** -10), extend=EXTEND_REFLECT, bound=0.0, f32_t=True),
    Case("lin_rotated_reflect", "linear", params=(0.0, 0.0, 23.0, 9.0), brush=ROT, extend=EXTEND_REFLECT),
    Case("lin_sheared_repeat", "linear", params=(3.0, 1.0, 40.0, 17.0), brush=SHEAR, extend=EXTEND_REPEAT),
    Case("lin_mirrored_pad", "linear", params=(2.0, 0.0, 50.0, 30.0), brush=MIRROR),
]

RADIAL = [
    # draw_leaf moves the centre of a circular gradient by 2^-12 (the reference does not): up to 511 * 2^-12 / (r1 - r0)
    # = 0.0012 texels on top of float32's 0.002
    Case(f"rad_circular_{n}", "radial", params=(32.3, 31.6, 32.3, 31.6, 4.0, 104.0), extend=e, bound=4e-3)
    for n, e in (("pad", EXTEND_PAD), ("repeat", EXTEND_REPEAT), ("reflect", EXTEND_REFLECT))
] + [
    Case("rad_r0_zero", "radial", params=(30.0, 28.0, 30.0, 28.0, 0.0, 21.0), extend=EXTEND_REPEAT, bound=4e-3),
    Case("rad_swapped", "radial", params=(20.0, 30.0, 40.0, 34.0, 25.0, 0.0), bound=4e-3, edge=0.05),
    Case("rad_swapped_reflect", "radial", params=(20.0, 30.0, 40.0, 34.0, 25.0, 0.0), extend=EXTEND_REFLECT, bound=4e-3, edge=0.05),
    Case("rad_r0_gt_r1_focal_gt_1", "radial", params=(30.0, 30.0, 35.0, 32.0, 30.0, 10.0), bound=4e-3, edge=0.05),
    Case("rad_cone_radius_gt_1", "radial", params=(30.0, 32.0, 34.0, 32.0, 5.0, 30.0), extend=EXTEND_REFLECT, bound=4e-3),
    Case("rad_cone_radius_lt_1", "radial", params=(10.0, 32.0, 50.0, 32.0, 5.0, 30.0), bound=4e-3, edge=0.05),
    Case("rad_cone_outside", "radial", params=(5.0, 5.0, 20.0, 12.0, 2.0, 6.0), extend=EXTEND_REPEAT, bound=3e-3, edge=0.05),
] + [
    # the strip kind: r0 == r1 with c0 != c1, and |r0 - r1| = 2^-12 (still the strip: vello paints radius r0) and 2^-11 (a
    # cone whose focal point lies 20480 radii away)
    Case(f"rad_strip_{n}", "radial", params=(10.0, 20.0, 50.0, 40.0, 10.0, 10.0), extend=e, bound=4e-3, edge=0.05)
    for n, e in (("pad", EXTEND_PAD), ("repeat", EXTEND_REPEAT), ("reflect", EXTEND_REFLECT))
] + [
    Case("rad_strip_dr_eps", "radial", params=(10.0, 20.0, 50.0, 40.0, 10.0, 10.0 + 2 ** -12), extend=EXTEND_REPEAT, bound=4e-3,
         edge=0.05),
    # Just past the strip's tolerance vello's own float32 arithmetic is the limit: fine forms t as focal_x + (a term of the
    # same size), with focal_x = -20480, so its t carries an error of a few ulp(20480) = 2^-9: up to 3 texels. The
    # reference cannot state which way that float32 cancellation rounds, so any texel within 3 of its own is accepted.
    Case("rad_strip_dr_2eps", "radial", params=(10.0, 20.0, 50.0, 40.0, 10.0, 10.0 + 2 ** -11), bound=4e-3, edge=0.05, spread=3),
] + [
    # the focal-on-circle kind: r0 = 0 and r1 = |c1 - c0| exactly (radius 1), c0 off the pixel grid so that the boundary
    # line through the focal point crosses no pixel corner; then radius 1 +- 2^-12 (still this kind: vello paints radius 1)
    # and 1 +- 2^-11 (the general cone on either side of radius 1)
    Case(f"rad_focal_{n}", "radial", params=(20.375, 32.5, 40.375, 32.5, 0.0, 20.0), extend=e, bound=4e-3, edge=0.05)
    for n, e in (("pad", EXTEND_PAD), ("repeat", EXTEND_REPEAT), ("reflect", EXTEND_REFLECT))
] + [
    Case(f"rad_focal_radius_{n}", "radial", params=(20.375, 32.5, 40.375, 32.5, 0.0, 20.0 * r), extend=EXTEND_REFLECT, bound=4e-3,
         edge=0.05)
    for n, r in (("1_plus_eps", 1 + 2 ** -12), ("1_minus_eps", 1 - 2 ** -12))
] + [
    # Just past the focal-on-circle tolerance draw_leaf scales by 1 / (radius^2 - 1) ~ 2^10, so the kernel's t carries
    # about 2^10 times float32's relative error, and far from the focus (t in the hundreds) that is up to 2 texels after
    # the reflection. The reference cannot state how that float32 error rounds, so any texel within 2 of its own is accepted.
    Case(f"rad_focal_radius_{n}", "radial", params=(20.375, 32.5, 40.375, 32.5, 0.0, 20.0 * r), extend=EXTEND_REFLECT, bound=4e-3,
         edge=0.05, spread=2)
    for n, r in (("1_plus_2eps", 1 + 2 ** -11), ("1_minus_2eps", 1 - 2 ** -11))
] + [
    Case("rad_same_centre_eps", "radial", params=(30.0, 30.0, 30.0, 30.0, 10.0, 10.0 + 2 ** -12), nan_info=True,
         note="c0 == c1, |r0 - r1| == 2^-12: nothing painted"),
    Case("rad_nonuniform", "radial", params=(10.0, 12.0, 18.0, 15.0, 3.0, 25.0), brush=NONUNIFORM, extend=EXTEND_REFLECT, bound=4e-3,
         edge=0.05),
]

TAU = 2.0 * math.pi
SWEEP = [
    Case("sweep_centre_on_corner", "sweep", params=(32.0, 32.0, 0.0, TAU), bound=1e-3),
    Case("sweep_t0_gt_t1", "sweep", params=(31.0, 30.0, 0.75 * TAU, 0.25 * TAU), bound=1e-3),
    Case("sweep_over_one_turn", "sweep", params=(32.0, 32.0, -0.5 * TAU, 1.5 * TAU), extend=EXTEND_REFLECT, bound=1e-3),
    Case("sweep_negative_repeat", "sweep", params=(20.0, 40.0, -0.7 * TAU, -0.2 * TAU), extend=EXTEND_REPEAT, bound=1e-3),
    Case("sweep_narrow_span", "sweep", params=(32.0, 32.0, 0.1 * TAU, 0.1 * TAU + 1.1 * 2 ** -15 * TAU), bound=1e-3),
]

RAMPS = [
    ("two_stops", [stop(0.0, 1, 0, 0), stop(1.0, 0, 0, 1)], True),
    ("hard_stops", [stop(0.0, 1, 0, 0), stop(0.5, 1, 0, 0), stop(0.5, 0, 1, 0), stop(0.5, 0, 0, 1), stop(1.0, 1, 1, 1)], True),
    ("inside", [stop(0.2, 1, 0.5, 0), stop(0.45, 0, 1, 0.5), stop(0.8, 0.3, 0, 1)], False),
    ("outside", [stop(-0.5, 1, 0, 0), stop(0.3, 0, 1, 0), stop(1.7, 0, 0, 1)], True),
    ("many", [stop(i / 599.0, (i * 37 % 256) / 255.0, (i * 91 % 256) / 255.0, (i * 13 % 256) / 255.0, 0.5 + (i % 2) * 0.5)
              for i in range(600)], True),
    ("alpha0_premul", [stop(0.0, 1, 0, 0, 0.0), stop(0.5, 0, 1, 0, 1.0), stop(1.0, 0, 0, 1, 0.0)], True),
    ("alpha0_straight", [stop(0.0, 1, 0, 0, 0.0), stop(0.5, 0, 1, 0, 1.0), stop(1.0, 0, 0, 1, 0.0)], False),
]
RAMP_CASES = [Case(f"ramp_{n}", "linear", w=520, h=2, params=(0.0, 0.0, 511.0, 0.0), stops=s, premul=pm, bound=1e-3)
              for n, s, pm in RAMPS]


def _img(w, h, seed, alpha_floor=0):
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    d[..., 3] = np.maximum(d[..., 3], alpha_floor)
    return d


def _premul(d):
    out = d.copy()
    out[..., :3] = np.minimum(d[..., :3], d[..., 3:4])  # a valid premultiplied image: colour <= alpha
    return out


IMG_5x3 = _img(5, 3, 1)
IMG_1x1 = _img(1, 1, 2, 40)
IMG_1xN = _img(1, 7, 3)
IMG_Nx1 = _img(9, 1, 4)
IMG_BIG = _img(64, 64, 5)
NEIGH = _img(6, 2, 6)  # shorter than IMG_5x3, so that the atlas ends at IMG_5x3's last row


def _one(data, m, **kw):
    return lambda: [(Image(data, **kw), m)]


MAG4 = (4.0, 0.0, 0.0, 4.0, 3.0, 5.0)
IMAGE = [
    Case(f"img_q{q}_x{xe}_y{ye}", "image", image=_one(IMG_5x3, MAG4, quality=q, x_extend=xe, y_extend=ye))
    for q in (0, 1, 2) for xe, ye in ((EXTEND_PAD, EXTEND_REPEAT), (EXTEND_REPEAT, EXTEND_REFLECT), (EXTEND_REFLECT, EXTEND_PAD))
] + [
    Case("img_1x1_bicubic", "image", image=_one(IMG_1x1, (7.0, 0.0, 0.0, 7.0, 10.0, 10.0), quality=2)),
    Case("img_1x1_bilinear_repeat", "image", image=_one(IMG_1x1, (3.0, 0.0, 0.0, 3.0, 1.0, 2.0), quality=1, x_extend=EXTEND_REPEAT,
                                                      y_extend=EXTEND_REFLECT)),
    Case("img_1xN_bilinear_reflect", "image", image=_one(IMG_1xN, (5.0, 0.0, 0.0, 3.0, 2.0, 1.0), quality=1, x_extend=EXTEND_REFLECT,
                                                       y_extend=EXTEND_REPEAT)),
    Case("img_Nx1_bicubic_repeat", "image", image=_one(IMG_Nx1, (3.0, 0.0, 0.0, 5.0, 1.0, 4.0), quality=2, x_extend=EXTEND_REPEAT)),
    Case("img_premul_bgra", "image", image=_one(_premul(IMG_5x3), MAG4, quality=1, alpha_type=ALPHA_PREMUL, format=FORMAT_BGRA)),
    Case("img_straight_bgra_alpha", "image", image=_one(IMG_5x3, MAG4, quality=2, format=FORMAT_BGRA, alpha=0.55)),
    Case("img_premul_alpha_nearest", "image", image=_one(_premul(IMG_5x3), MAG4, quality=0, alpha_type=ALPHA_PREMUL, alpha=0.3)),
    Case("img_magnify_1000", "image", image=_one(IMG_5x3, (1000.0, 0.0, 0.0, 1000.0, -2480.0, -1470.0), quality=1)),
    Case("img_minify", "image", image=_one(IMG_BIG, (1 / 7.3, 0.0, 0.0, 1 / 5.1, 1.0, 2.0), quality=2, x_extend=EXTEND_REPEAT,
                                         y_extend=EXTEND_REFLECT)),
    Case("img_rotated_bilinear", "image", image=_one(IMG_5x3, (3.0, 2.0, -2.0, 3.0, 30.0, 5.0), quality=1, x_extend=EXTEND_REFLECT,
                                                   y_extend=EXTEND_REPEAT)),
    # the checked image sits right of its neighbour in the atlas, on the atlas's right and bottom edges: no tap may read the
    # neighbour's texels or past the atlas
    Case("img_slots_touch_bicubic", "image", image=lambda: [(Image(NEIGH), (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)),
                                                          (Image(IMG_5x3, quality=2), (6.0, 0.0, 0.0, 6.0, 4.0, 3.0))]),
    Case("img_slots_touch_bilinear", "image", image=lambda: [(Image(NEIGH), (1.0, 0.0, 0.0, 1.0, 0.0, 0.0)),
                                                           (Image(IMG_5x3, quality=1, x_extend=EXTEND_REPEAT),
                                                            (6.0, 0.0, 0.0, 6.0, 4.0, 3.0))]),
]

BLUR = [
    # edges at half-integers: every pixel corner is 1/2 away from the edge, where sigma = 10^-3 makes the alpha 0 or 1
    Case("blur_sharp", "blur", blur=(10.5, 12.5, 50.5, 40.5, 0.0, 1e-3), bound=1.0),
    Case("blur_sharp_round", "blur", blur=(10.5, 12.5, 50.5, 40.5, 6.0, 1e-3), bound=1.0),
    # sigma = 10^3 over a 4000 x 3000 rectangle centred near the frame: an alpha of about 0.4, varying slowly
    Case("blur_wide", "blur", blur=(-1967.5, -1467.5, 2032.5, 1532.5, 0.0, 1e3), bound=1.0),
    # zero width: min_edge = 0 makes both corner radii 0 and the exponent 0 / 0, so the alpha is NaN, which fine's store
    # clamps to 0 (fmaxf(0, NaN) = 0): nothing is painted
    Case("blur_zero_width", "blur", blur=(20.5, 10.5, 20.5, 50.5, 0.0, 2.0), bound=0.0),
    Case("blur_radius_over_half", "blur", blur=(8.0, 9.0, 40.0, 30.0, 25.0, 3.0), bound=1.0),
    Case("blur_radius_zero", "blur", blur=(8.0, 9.0, 40.0, 30.0, 0.0, 4.0), bound=1.0),
]

CASES = LINEAR + RADIAL + SWEEP + RAMP_CASES + IMAGE + BLUR


def _ids(cases):
    return [c.name for c in cases]


@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_reference_matches_oracle(oracle, case):
    """The reference and the oracle's full pipeline (area AA) agree on every case."""
    packed = resolve(case.scene().encoding)
    img = oracle.render(packed, case.w, case.h, 0, AA_AREA)
    check_pixels(case, img, packed.ramps)


@pytest.mark.parametrize("name,stops,premul", RAMPS, ids=[r[0] for r in RAMPS])
def test_ramp_reference_matches_host_ramp(name, stops, premul):
    """encoding.make_ramp (float32) is within 1 LSB of the float64 ramp."""
    from vello_b200.encoding import make_ramp
    want = P.ramp([(o, (c.r, c.g, c.b, c.a)) for o, c in stops], premul).astype(np.int32)
    got = np.ascontiguousarray(make_ramp(stops, premul)).view(np.uint8).reshape(-1, 4).astype(np.int32)
    assert np.abs(got - want).max() <= 1, (name, int(np.abs(got - want).max()))


# ---- the atlas's 16-bit places ------------------------------------------------------------------------------------------------
def _past_row_65535():
    """A 1 x 65535 image, then two 2048 x 1 images: the first starts a shelf at y = 65535 (the last row a place holds), the
    second one at y = 65536."""
    s = Scene()
    tall = Image(np.broadcast_to(np.array([9, 8, 7, 255], np.uint8), (65535, 1, 4)))
    for im in (tall, Image(np.zeros((1, 2048, 4), np.uint8)), Image(np.zeros((1, 2048, 4), np.uint8))):
        s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), im, None, Rect(0, 0, 8, 8))
    return s


def test_resolve_refuses_atlas_places_past_16_bits():
    """A place past row 65535 would spill y into x in the draw data's (x << 16) | y, and a side of 65536 packs a size of 0:
    the Python resolve refuses both, before it allocates the atlas."""
    with pytest.raises(ValueError, match="65535"):
        resolve(_past_row_65535().encoding)
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), Image(np.broadcast_to(np.zeros(4, np.uint8), (1, 65536, 4))), None,
           Rect(0, 0, 8, 8))
    with pytest.raises(ValueError, match="65535"):
        resolve(s.encoding)


def test_native_resolve_refuses_atlas_places_past_16_bits():
    """vb_scene_resolve refuses the same scenes (VB_E_INVALID)."""
    from vello_b200.scene_native import NativeScene
    ns = NativeScene()
    tall = Image(np.broadcast_to(np.array([9, 8, 7, 255], np.uint8), (65535, 1, 4)))
    for im in (tall, Image(np.zeros((1, 2048, 4), np.uint8)), Image(np.zeros((1, 2048, 4), np.uint8))):
        ns.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), im, None, Rect(0, 0, 8, 8))
    with pytest.raises(ValueError):
        ns.resolve()
    wide = NativeScene()
    wide.fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), Image(np.zeros((1, 65536, 4), np.uint8)), None, Rect(0, 0, 8, 8))
    with pytest.raises(ValueError):
        wide.resolve()
