"""vello's blend path -- the 16 mix modes, the 14 compose operators, layer alpha, the luminance mask and the 8-bit blend
stack -- restated in float64 from the W3C *Compositing and Blending Level 1* text, as vello applies it (shared/blend.wgsl,
fine.wgsl END_CLIP), vectorised over numpy arrays.

Every quantity is an `F`: its float64 value `v` (the exact result of the spec's formula on the stated inputs) and `e`, a
running bound on the error of fine's float32 evaluation of the same formula: unit roundoff 2^-24 per +, -, *, /, sqrt,
propagated to first order with the exact cross terms; min, max and clamp are exact on the interval [v - e, v + e]. The
spec's decimal constants (0.3 / 0.59 / 0.11, 0.2125 / 0.7154 / 0.0721) carry their float32 rounding in `e`. A value whose
float32 result may overflow, or be a 0/0, is `wild`: fine's byte there is not stated, and any byte is accepted.

Where fine quantises, stated exactly:
- colour and texel bytes are byte / 255 in float32; premultiplied image texels are used as they are, rgb > a included;
- the layer's source is fg = rgba * area * layer_alpha in float32, layer_alpha being the float32 the encoding stores;
- unpremultiply is c * (1 / max(a, 1e-15)) in float32. `leaf()` evaluates it exactly as float32 (three correctly rounded
  operations on stated float32 inputs), because the spec's tests `cb == 0`, `cs == 1`, `cb == 1`, `cs == 0`, `cs <= 0.5`
  and `cb <= 0.25` and set_sat's ordering are decided on that value. For 25 alphas a (7, 14, 28, ...) the float32 product
  (a/255) * (1 / (a/255)) is 1 - 2^-24, so p == a does not unpremultiply to 1 and the dodge / burn early-outs are not taken
  there: the reference follows vello (`if cb == 1.0`, blend.wgsl:39), which tests the value fine computed;
- every BEGIN_CLIP stores the backdrop through pack4x8unorm, floor(0.5 + 255 clamp(x)): `pack8`;
- the frame stores separated alpha, c / max(a, 1e-6), through the same rounding: `store8`.

Degenerate rules:
- clip_color on a grey colour (x == l and n == l in the spec's arithmetic): both branches' quotients are 0/0 in exact
  arithmetic; float32 evaluates l = lum(c) with constants that sum to 1 - 1.5e-8, so the quotient is +-1 (the channel goes to
  0 when n < 0, to 1 when x > 1) unless l rounds to exactly x, where it is NaN. Neither outcome is stated: wild.
- a texel with rgb > a unpremultiplies to a channel over 1; with a = 0, to p / 255 * 1e15. Those are inputs like any other;
  products of three of them overflow float32 (soft-light of two such texels): wild.
- compose CLEAR: Fa = Fb = 0, so the colour and alpha are exactly 0, which the frame stores as 0.

Branches: where a comparison's operand lies within its bound of the threshold, both outcomes are evaluated and the result is
their hull. `tally` counts, per formula, which branches the decided pixels took, so a case can assert what it reached.
"""
from __future__ import annotations

import collections

import numpy as np

U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
f32 = np.float32


class F:
    """A float64 value with a bound on float32's error, elementwise over numpy arrays."""
    __slots__ = ("v", "e", "wild")

    def __init__(self, v, e=0.0, wild=False):
        self.v = np.asarray(v, np.float64)
        self.e = np.asarray(e, np.float64)
        self.wild = np.asarray(wild, bool)

    @staticmethod
    def of(x) -> "F":
        return x if isinstance(x, F) else F(x)

    @staticmethod
    def rounded(v, e, wild) -> "F":
        """The float32 rounding of a result whose exact operands are within e of v."""
        e = e + U * (np.abs(v) + e)
        bad = ~(np.abs(v) + e <= FLT_MAX)  # overflow, inf or NaN
        return F(np.where(bad, 0.0, v), np.where(bad, 0.0, e), wild | bad)

    def __add__(a, b):
        b = F.of(b)
        return F.rounded(a.v + b.v, a.e + b.e, a.wild | b.wild)

    __radd__ = __add__

    def __sub__(a, b):
        b = F.of(b)
        return F.rounded(a.v - b.v, a.e + b.e, a.wild | b.wild)

    def __rsub__(a, b):
        return F.of(b) - a

    def __mul__(a, b):
        b = F.of(b)
        return F.rounded(a.v * b.v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e, a.wild | b.wild)

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = F.of(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            den = np.abs(b.v) - b.e
            e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf)
        return F.rounded(v, e, a.wild | b.wild)

    def __rtruediv__(a, b):
        return F.of(b) / a

    def __neg__(a):
        return F(-a.v, a.e, a.wild)

    def sqrt(a) -> "F":
        v = np.sqrt(np.maximum(a.v, 0.0))
        lo = np.sqrt(np.maximum(a.v - a.e, 0.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.minimum(np.where(v + lo > 0, a.e / np.where(v + lo > 0, v + lo, 1.0), np.inf), np.sqrt(a.e))
        return F.rounded(v, e, a.wild | (a.v + a.e < 0))

    @property
    def lo(self):
        return self.v - self.e

    @property
    def hi(self):
        return self.v + self.e

    @staticmethod
    def interval(lo, hi, wild) -> "F":
        return F(0.5 * (lo + hi), 0.5 * (hi - lo), wild)

    def __abs__(a):
        lo, hi = np.abs(a.lo), np.abs(a.hi)
        cross = (a.lo < 0) & (a.hi > 0)
        return F.interval(np.where(cross, 0.0, np.minimum(lo, hi)), np.maximum(lo, hi), a.wild)


def fmin(a, b) -> F:
    a, b = F.of(a), F.of(b)
    return F.interval(np.minimum(a.lo, b.lo), np.minimum(a.hi, b.hi), a.wild | b.wild)


def fmax(a, b) -> F:
    a, b = F.of(a), F.of(b)
    return F.interval(np.maximum(a.lo, b.lo), np.maximum(a.hi, b.hi), a.wild | b.wild)


def clamp01(a: F) -> F:
    return fmin(fmax(a, 0.0), 1.0)


def const(x: float) -> F:
    """A decimal constant of the spec, with its float32 rounding in the bound."""
    return F(x, abs(float(f32(x)) - x))


def hull(a: F, b: F) -> F:
    return F.interval(np.minimum(a.lo, b.lo), np.maximum(a.hi, b.hi), a.wild | b.wild)


def where(c, a: F, b: F) -> F:
    a, b = F.of(a), F.of(b)
    return F(np.where(c, a.v, b.v), np.where(c, a.e, b.e), np.where(c, a.wild, b.wild))


class Tally(collections.Counter):
    def add(self, name, mask):
        self[name] += int(np.count_nonzero(mask))


def branch(a: F, op: str, t, yes: F, no: F, tally: Tally | None = None, name: str = "") -> F:
    """`yes if a <op> t else no`. Decided on a.v where the bound keeps a off the threshold; the hull of both otherwise."""
    t = F.of(t)
    d = a.v - t.v
    pred = {"<=": d <= 0, "<": d < 0, ">": d > 0, "==": d == 0}[op]
    amb = (np.abs(d) <= a.e + t.e) & (a.e + t.e > 0)
    if tally is not None:
        tally.add(name + ".yes", pred & ~amb)
        tally.add(name + ".no", ~pred & ~amb)
    out = where(pred, yes, no)
    if amb.any():
        out = where(amb, hull(F.of(yes), F.of(no)), out)
    return out


# ---- the W3C separable blend functions B(cb, cs) -----------------------------------------------------------------------
def multiply(cb, cs, T=None):
    return cb * cs


def screen(cb, cs, T=None):
    return cb + cs - cb * cs


def hard_light(cb, cs, T=None, name="hard_light"):
    return branch(cs, "<=", 0.5, cb * 2.0 * cs, screen(cb, 2.0 * cs - 1.0), T, name + ".cs_le_half")


def overlay(cb, cs, T=None):
    return hard_light(cs, cb, T, "overlay")


def darken(cb, cs, T=None):
    return fmin(cb, cs)


def lighten(cb, cs, T=None):
    return fmax(cb, cs)


def _early_outs(T, name, first, second):
    """Tally which of two ordered early-outs (exact tests) a pixel takes, and the corner where both tests hold."""
    if T is not None:
        T.add(name + ".first", first)
        T.add(name + ".second", ~first & second)
        T.add(name + ".general", ~first & ~second)
        T.add(name + ".corner", first & second)


def color_dodge(cb, cs, T=None):
    """0 if cb == 0, else 1 if cs == 1, else min(1, cb / (1 - cs)): the cb test comes first, so the corner is 0."""
    one, zero = F(np.ones_like(cb.v)), F(np.zeros_like(cb.v))
    with np.errstate(all="ignore"):
        general = fmin(1.0, cb / (1.0 - cs))
    _early_outs(T, "color_dodge", (cb.v == 0) & (cb.e == 0), (cs.v == 1) & (cs.e == 0))
    return branch(cb, "==", 0.0, zero, branch(cs, "==", 1.0, one, general))


def color_burn(cb, cs, T=None):
    """1 if cb == 1, else 0 if cs == 0, else 1 - min(1, (1 - cb) / cs): the cb test comes first, so the corner is 1."""
    one, zero = F(np.ones_like(cb.v)), F(np.zeros_like(cb.v))
    with np.errstate(all="ignore"):
        general = 1.0 - fmin(1.0, (1.0 - cb) / cs)
    _early_outs(T, "color_burn", (cb.v == 1) & (cb.e == 0), (cs.v == 0) & (cs.e == 0))
    return branch(cb, "==", 1.0, one, branch(cs, "==", 0.0, zero, general))


def soft_light(cb, cs, T=None):
    low = cb - (1.0 - 2.0 * cs) * cb * (1.0 - cb)
    # D(cb) only matters where cs > 1/2: tally it there
    sub = None if T is None else Tally()
    d = branch(cb, "<=", 0.25, ((16.0 * cb - 12.0) * cb + 4.0) * cb, cb.sqrt(), sub, "soft_light.d_poly")
    if T is not None:
        gt = cs.v > 0.5 + cs.e
        T.add("soft_light.d_poly.yes", gt & (cb.v <= 0.25 - cb.e))
        T.add("soft_light.d_poly.no", gt & (cb.v > 0.25 + cb.e))
    return branch(cs, "<=", 0.5, low, cb + (2.0 * cs - 1.0) * (d - cb), T, "soft_light.cs_le_half")


def difference(cb, cs, T=None):
    return abs(cb - cs)


def exclusion(cb, cs, T=None):
    return cb + cs - 2.0 * cb * cs


# ---- the non-separable ones: Lum, ClipColor, SetLum, Sat, SetSat on colours (r, g, b) of F --------------------------------
LUM = (0.3, 0.59, 0.11)
SVG_LUM = (0.2125, 0.7154, 0.0721)  # the luminance mask's (sRGB) coefficients, fine.wgsl END_CLIP


def lum(c, k=LUM):
    return c[0] * const(k[0]) + c[1] * const(k[1]) + c[2] * const(k[2])


def _grey(c):
    return (c[0].v == c[1].v) & (c[1].v == c[2].v) & (c[0].e == c[1].e) & (c[1].e == c[2].e)


def clip_color(c, T=None):
    l = lum(c)
    n = fmin(c[0], fmin(c[1], c[2]))
    x = fmax(c[0], fmax(c[1], c[2]))
    grey = _grey(c)
    with np.errstate(all="ignore"):
        lo = [l + (ch - l) * l / (l - n) for ch in c]
    neg = [branch(n, "<", 0.0, lo[i], c[i], T if i == 0 else None, "clip_color.n_lt_0") for i in range(3)]
    with np.errstate(all="ignore"):
        hi = [l + (ch - l) * (1.0 - l) / (x - l) for ch in neg]
    out = [branch(x, ">", 1.0, hi[i], neg[i], T if i == 0 else None, "clip_color.x_gt_1") for i in range(3)]
    # the 0/0 of a grey colour that either branch touches (see the module's degenerate rules)
    touched = grey & ((n.lo < 0) | (x.hi > 1))
    return [F(o.v, o.e, o.wild | touched) for o in out]


def set_lum(c, l, T=None):
    d = l - lum(c)
    return clip_color([ch + d for ch in c], T)


def sat(c):
    return fmax(c[0], fmax(c[1], c[2])) - fmin(c[0], fmin(c[1], c[2]))


PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]  # (min, mid, max) channel indices


def set_sat(c, s, T=None):
    """SetSat: Cmid scaled into [0, s] by (Cmid - Cmin) / (Cmax - Cmin), Cmax = s, Cmin = 0; all 0 when Cmax == Cmin. Every
    ordering consistent with the bounds is evaluated (the spec's result is the same for tied channels, so the hull is tight
    there), and float32 keeps the scaled Cmid in [0, s] because it is ordered like its inputs."""
    v = np.stack([ch.v for ch in c])
    primary = np.argsort(v, axis=0, kind="stable")
    zero = F(np.zeros_like(v[0]))
    results = []
    for p in PERMS:
        lo, mid, hi = (c[i] for i in p)
        is_primary = (primary[0] == p[0]) & (primary[1] == p[1])
        ok = (mid.v - lo.v >= -(mid.e + lo.e)) & (hi.v - mid.v >= -(hi.e + mid.e))
        with np.errstate(all="ignore"):
            scaled = (mid - lo) * s / (hi - lo)
        scaled = F.interval(np.clip(scaled.lo, 0.0, None), np.minimum(scaled.hi, s.hi * (1 + 2 * U)), scaled.wild)
        spread = hi - lo
        res = [None] * 3
        res[p[0]] = zero
        res[p[1]] = branch(spread, ">", 0.0, scaled, zero)
        res[p[2]] = branch(spread, ">", 0.0, s, zero)
        if T is not None:
            strict = (mid.v - lo.v > mid.e + lo.e) & (hi.v - mid.v > hi.e + mid.e)
            T.add("set_sat.order_" + "".join("rgb"[i] for i in p), is_primary & strict)
            T.add("set_sat.equal", is_primary & (spread.hi <= 0))
        results.append((is_primary, ok, res))
    out = list(results[0][2])
    for is_primary, _, res in results[1:]:
        out = [where(is_primary, r, o) for r, o in zip(res, out)]
    for is_primary, ok, res in results:
        alt = ok & ~is_primary
        if alt.any():
            out = [where(alt, hull(o, r), o) for o, r in zip(out, res)]
    return out


SEPARABLE = {1: multiply, 2: screen, 3: overlay, 4: darken, 5: lighten, 6: color_dodge, 7: color_burn, 8: hard_light,
             9: soft_light, 10: difference, 11: exclusion}
MIXES = ["normal", "multiply", "screen", "overlay", "darken", "lighten", "color_dodge", "color_burn", "hard_light", "soft_light",
         "difference", "exclusion", "hue", "saturation", "color", "luminosity"]  # peniko::Mix values 0..15
COMPOSES = ["clear", "copy", "dest", "src_over", "dest_over", "src_in", "dest_in", "src_out", "dest_out", "src_atop",
            "dest_atop", "xor", "plus", "plus_lighter"]  # peniko::Compose values 0..13


def blend_mix(cb, cs, mix, T=None):
    """B(Cb, Cs) of the mix mode, on unpremultiplied colours (lists of three F)."""
    if mix == 0:
        return list(cs)
    if mix in SEPARABLE:
        return [SEPARABLE[mix](cb[i], cs[i], T) for i in range(3)]
    if mix == 12:  # hue
        return set_lum(set_sat(cs, sat(cb), T), lum(cb), T)
    if mix == 13:  # saturation
        return set_lum(set_sat(cb, sat(cs), T), lum(cb), T)
    if mix == 14:  # color
        return set_lum(cs, lum(cb), T)
    if mix == 15:  # luminosity
        return set_lum(cb, lum(cs), T)
    raise ValueError(mix)


def porter_duff(compose, as_, ab):
    """(Fa, Fb) of the compose operator (the spec's table; plus-lighter is `plus`, clamped)."""
    one, zero = F(np.ones_like(as_.v)), F(np.zeros_like(as_.v))
    return {0: (zero, zero), 1: (one, zero), 2: (zero, one), 3: (one, 1.0 - as_), 4: (1.0 - ab, one), 5: (ab, zero),
            6: (zero, as_), 7: (1.0 - ab, zero), 8: (zero, 1.0 - as_), 9: (ab, 1.0 - as_), 10: (1.0 - ab, as_),
            11: (1.0 - ab, 1.0 - as_), 12: (one, one), 13: (one, one)}[compose]


def unpremultiply(c):
    """Premultiplied (r, g, b, a) of F -> unpremultiplied (r, g, b): c * (1 / max(a, 1e-15))."""
    inv = 1.0 / fmax(c[3], float(f32(1e-15)))
    return [c[i] * inv for i in range(3)]


def leaf(rgba32: np.ndarray):
    """Stated float32 inputs, shape (..., 4) -> (premultiplied rgba as F, unpremultiplied rgb as exact F). See the module
    docstring: fine's unpremultiply of a stated input is evaluated in float32."""
    c = np.asarray(rgba32, f32)
    inv = f32(1.0) / np.maximum(c[..., 3], f32(1e-15))
    un = c[..., :3] * inv[..., None]
    return [F(c[..., i].astype(np.float64)) for i in range(4)], [F(un[..., i].astype(np.float64)) for i in range(3)]


def blend(bg, fg, mix: int, compose: int, T=None, un_bg=None, un_fg=None):
    """vello's blend_mix_compose (fine.wgsl END_CLIP) of premultiplied (r, g, b, a) F lists -> premultiplied result. un_bg /
    un_fg: their unpremultiplied colours when stated exactly (`leaf`)."""
    ab, as_ = bg[3], fg[3]
    if T is not None:
        for nm, a in (("ab", ab), ("as", as_)):
            T.add(nm + "_0", a.hi <= 0)
            T.add(nm + "_partial", (a.lo > 0) & (a.hi < 1))
            T.add(nm + "_1", a.lo >= 1)
    if (mix == 0 or mix == 128) and compose == 3:
        # normal / src-over (and Mix::Clip, 0x8003): backdrop * (1 - src.a) + src, blend.wgsl:302-304
        k = 1.0 - as_
        return [F.rounded(bg[i].v * k.v + fg[i].v, np.abs(bg[i].v) * k.e + np.abs(k.v) * bg[i].e + bg[i].e * k.e + fg[i].e,
                          bg[i].wild | k.wild | fg[i].wild) for i in range(4)]
    cs = un_fg if un_fg is not None else unpremultiply(fg)
    cb = un_bg if un_bg is not None else unpremultiply(bg)
    mixed = blend_mix(cb, cs, mix, T)
    # the source colour mixed with B(Cb, Cs) by the backdrop's alpha (spec: Cs = (1 - ab) Cs + ab B(Cb, Cs))
    cs = [cs[i] * (1.0 - ab) + mixed[i] * ab for i in range(3)]
    if compose == 3:
        # src-over: co = mix(backdrop.rgb, cs, src.a), blend.wgsl:312-314
        return [bg[i] * (1.0 - as_) + cs[i] * as_ for i in range(3)] + [as_ + ab * (1.0 - as_)]
    if compose == 13:
        sums = [as_ * cs[i] + ab * cb[i] for i in range(3)] + [as_ + ab]
        if T is not None:
            T.add("plus_lighter.clamped", sums[3].lo > 1)
            T.add("plus_lighter.unclamped", sums[3].hi < 1)
        return [fmin(1.0, s) for s in sums]
    fa, fb = porter_duff(compose, as_, ab)
    as_fa, ab_fb = as_ * fa, ab * fb
    return [as_fa * cs[i] + ab_fb * cb[i] for i in range(3)] + [fmin(as_fa + ab_fb, 1.0)]


def luminance_mask(bg, fg, area, T=None, un_fg=None):
    """END_CLIP of a luminance mask layer: bg * clamp(svg_lum(unpremultiply(fg)) * fg.a); at area == 0 the backdrop."""
    un = un_fg if un_fg is not None else unpremultiply(fg)
    l = clamp01(lum(un, SVG_LUM) * fg[3])
    out = [bg[i] * l for i in range(4)]
    zero = np.asarray(area) == 0
    if T is not None:
        T.add("luminance_mask.area_0", zero)
        T.add("luminance_mask.area_1", ~zero)
    return [where(zero, bg[i], out[i]) for i in range(4)]


def over(bg, fg):
    """rgba * (1 - fg.a) + fg, one rounding for the fused multiply-add (fine.wgsl:1117)."""
    return blend(bg, fg, 0, 3)


def _bytes(x: F):
    """floor(0.5 + 255 clamp(x)) for the value and both ends of its bound, with float32's rounding of 255 x + 0.5."""
    y = clamp01(x) * 255.0 + 0.5
    # a tie of the byte inputs: the spec's value on the bytes rounds half-way (e.g. the mean of an odd sum of bytes at layer
    # alpha 1/2), displaced only by the float32 rounding of byte / 255 (under 4 * 255 * 2^-24 LSB); its byte is float32's
    # rounding error, not the formula
    tie = np.abs(y.v - np.round(y.v)) <= 4 * 255 * U
    return (np.floor(y.v).astype(np.int64), np.floor(y.lo).astype(np.int64), np.floor(y.hi).astype(np.int64), y.e, y.wild,
            tie & ~y.wild)


def pack8(c):
    """pack4x8unorm of premultiplied (r, g, b, a) F: per channel (byte, lowest byte, highest byte); a byte is ambiguous
    where its bound straddles a rounding tie. A wild value is never stored by these cases (asserted)."""
    out = []
    for ch in c:
        b, lo, hi, _, w, _ = _bytes(ch)
        assert not w.any(), "a blend-stack store of an unstated value"
        out.append((b, lo, hi))
    return out


def store8(c):
    """The frame's store: separated alpha, c / max(a, 1e-6), then floor(0.5 + 255 clamp(x)). Per channel:
    (byte, lowest byte, highest byte, bound in LSB, wild, exact tie)."""
    inv = 1.0 / fmax(c[3], float(f32(1e-6)))
    return [_bytes(c[i] * inv) for i in range(3)] + [_bytes(c[3])]


# ---- scalar helpers for first-principles spot checks (test_oracle_analytic.py) --------------------------------------------
def w3c_mix(mode, cb, cs):
    """B(Cb, Cs) of the named mix mode on float unpremultiplied colours -> list of float (the bound dropped)."""
    m = MIXES.index(mode)
    return [float(x.v) for x in blend_mix([F(float(v)) for v in cb], [F(float(v)) for v in cs], m)]


def w3c_composite(mix, compose, cb, ab, cs, as_):
    """Unpremultiplied backdrop / source colours and alphas -> premultiplied result (r, g, b, a), per the spec: Cs mixed
    with B(Cb, Cs) by ab, then Porter-Duff (plus-lighter clamped)."""
    cbf, csf = [F(float(v)) for v in cb], [F(float(v)) for v in cs]
    abf, asf = F(float(ab)), F(float(as_))
    bm = blend_mix(cbf, csf, mix)
    cm = [csf[i] * (1.0 - abf) + bm[i] * abf for i in range(3)]
    if compose == 13:
        return [float(fmin(1.0, asf * cm[i] + abf * cbf[i]).v) for i in range(3)] + [float(fmin(1.0, asf + abf).v)]
    fa, fb = porter_duff(compose, asf, abf)
    return [float((asf * fa * cm[i] + abf * fb * cbf[i]).v) for i in range(3)] + [float(fmin(asf * fa + abf * fb, 1.0).v)]
