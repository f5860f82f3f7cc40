"""Blend edge cases -- the 16 mix modes, the 14 compose operators, layer alpha, clip layers, luminance masks and a nested
chain across the blend stack's register / spill split -- checked against the float64 statement of vello's blends in
blend_ref.py, here on the CPU oracle's full pipeline (test_gpu_blend_edges.py runs the same cases on the GPU).

Every case is one 256 x 256 frame over a transparent base. A premultiplied, nearest-sampled image drawn at identity makes
each pixel's backdrop exactly one texel: colour x of COLOURS in column x. Each layer draws its own source image, colour y
of COLOURS (permuted per level) in row y, so the frame holds all 65536 (backdrop, source) pairs of the colour set.

The check (`check`): each channel byte must be the reference's; an adjacent byte is accepted only where the reference's
float32 error bound straddles a rounding tie (or where a blend-stack store's bound straddles one: the reference then
evaluates both stored bytes). At most 1 % of a case's channel values may be accepted that way, and the median bound must
stay under 0.01 LSB. Two kinds of channel value are not counted in that 1 %: exact ties of the byte inputs (the spec's value
rounds half-way, e.g. the mean of an odd sum of bytes at layer alpha 1/2), where either neighbour is accepted, and values
blend_ref marks wild (its degenerate rules), where any byte is; these are reported, and wild ones capped at 8 %. Before
comparing, each case asserts from the reference's branch tallies that its frame reached every
branch of the formulas it uses (`reach`)."""
from __future__ import annotations

import functools
import itertools
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pytest

from vello_b200.config import AA_AREA
from vello_b200.encoding import (ALPHA_PREMULTIPLIED, FILL_NON_ZERO, QUALITY_LOW, Color, Image, Scene, resolve)
from vello_b200.shapes import Affine, Rect

from . import blend_ref as B

W = H = 256
LUM, CLIP = "luminance", "clip"


# ---- the colour set -----------------------------------------------------------------------------------------------------------
def _colours() -> np.ndarray:
    """256 premultiplied RGBA8 texels, the edges first (asserted to fit), then seeded random valid texels."""
    out = []
    strict = list(itertools.permutations((0, 1, 2)))
    one_tie = [(0, 0, 1), (0, 1, 0), (1, 0, 0), (1, 1, 0), (1, 0, 1), (0, 1, 1)]
    for a in (0, 1, 2, 64, 127, 128, 254, 255, 7, 28, 252):
        # all 13 weak orderings of (r, g, b) on the ladder 0, a/4, a (unpremultiplied 0, 1/4, 1 when 4 divides a); the ties
        # on a/4, a; grey at each rung. A channel of exactly 1/2 stores as 127.5, a rounding tie: a few colours only
        lad = (0, a // 4, a)
        out += [tuple(lad[r] for r in rk) + (a,) for rk in strict]
        out += [tuple((a // 4, a)[r] for r in rk) + (a,) for rk in one_tie]
        out += [(g, g, g, a) for g in sorted(set(lad))]
    out += [(16, 32, 64, 64), (64, 32, 128, 128), (127, 254, 0, 254)]  # 1/4, 1/2, 1 and 1/2, 1/4, 1
    for v in (0, 1, 2, 63, 64, 127, 128, 191, 192, 253, 254, 255):  # every channel value, opaque, alone and mixed
        out += [(v, v, v, 255), (v, 255 - v, 128, 255), (255, v, 0, 255)]
    # dodge / burn corners: cb = 0 beside cs = 1 comes from the ladders; channels near 0 and 1 unpremultiplied
    out += [(1, 254, 128, 255), (254, 1, 0, 255), (63, 0, 64, 64)]
    # set_lum leaves the gamut: saturated colours against light and dark targets
    out += [(255, 0, 0, 255), (0, 0, 255, 255), (0, 255, 0, 255), (255, 255, 0, 255), (0, 255, 255, 255), (20, 0, 0, 255)]
    # rgb > a, including a = 0
    out += [(200, 10, 100, 128), (255, 200, 40, 64), (64, 0, 32, 0), (3, 2, 1, 1), (90, 90, 90, 2)]
    seen, uniq = set(), []
    for c in out:
        if c not in seen:
            seen.add(c)
            uniq.append(c)
    assert len(uniq) <= 256, len(uniq)
    rng = np.random.default_rng(20261017)
    while len(uniq) < 256:
        a = int(rng.integers(0, 256))
        c = tuple(int(v) for v in rng.integers(0, a + 1, size=3)) + (a,)
        if c not in seen:
            seen.add(c)
            uniq.append(c)
    return np.array(uniq, np.uint8)


COLOURS = _colours()
PERM_STEP = (1, 37, 101, 149, 199, 233, 251)  # level k's source row y is colour (y * step[k] + k) % 256


def _source(k: int) -> np.ndarray:
    """Level k's source texels (H, W, 4): colour of row y."""
    ix = (np.arange(H) * PERM_STEP[k] + k) % 256
    return np.broadcast_to(COLOURS[ix][:, None, :], (H, W, 4))


BACKDROP = np.broadcast_to(COLOURS[None, :, :], (H, W, 4))


@dataclass(frozen=True)
class Level:
    mix: object  # 0..15, LUM (a luminance mask layer) or CLIP (push_clip_layer)
    compose: int = 3
    alpha: float = 1.0


@dataclass(frozen=True)
class Case:
    name: str
    levels: tuple  # Level, outermost first; level k draws _source(k)
    under: Optional[Color] = None  # a colour filled over the backdrop image before the first push
    clip: tuple = (0, 0, W, H)  # every layer's clip rectangle (pixel aligned)
    content: tuple = (0, 0, W, H)  # the innermost source's rectangle

    def scene(self) -> Scene:
        s = Scene()
        s.draw_image(Image(np.ascontiguousarray(BACKDROP), alpha_type=ALPHA_PREMULTIPLIED, quality=QUALITY_LOW), Affine.IDENTITY)
        if self.under is not None:
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, self.under, None, Rect(0, 0, W, H))
        clip = Rect(*self.clip)
        for k, lv in enumerate(self.levels):
            if lv.mix == LUM:
                s.push_luminance_mask_layer(FILL_NON_ZERO, lv.alpha, Affine.IDENTITY, clip)
            elif lv.mix == CLIP:
                s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, clip)
            else:
                s.push_layer(FILL_NON_ZERO, lv.mix, lv.compose, lv.alpha, Affine.IDENTITY, clip)
            im = Image(np.ascontiguousarray(_source(k)), alpha_type=ALPHA_PREMULTIPLIED, quality=QUALITY_LOW)
            rect = self.content if k == len(self.levels) - 1 else (0, 0, W, H)
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, im, None, Rect(*rect))
        for _ in self.levels:
            s.pop_layer()
        return s

    def reach(self) -> list:
        """The tallies this case's frame must reach: every branch of every formula it uses."""
        need = []
        for lv in self.levels:
            if lv.mix == LUM:
                need += ["luminance_mask.area_0", "luminance_mask.area_1"]
                continue
            if lv.mix == CLIP or (lv.mix == 0 and lv.compose == 3):
                continue
            need += ["ab_0", "ab_partial", "ab_1", "as_0"]
            if lv.alpha == 0.0:  # every source is transparent: only the compose operator's backdrop terms are reached
                continue
            need += ["as_partial"] + (["as_1"] if lv.alpha == 1.0 else [])
            m = lv.mix
            if m in (3, 8):
                nm = "overlay" if m == 3 else "hard_light"
                need += [nm + ".cs_le_half.yes", nm + ".cs_le_half.no"]
            if m in (6, 7):
                nm = B.MIXES[m]
                need += [nm + s for s in (".first", ".second", ".general", ".corner")]
            if m == 9:
                need += ["soft_light.cs_le_half.yes", "soft_light.cs_le_half.no", "soft_light.d_poly.yes", "soft_light.d_poly.no"]
            if m in (12, 13):
                need += ["set_sat.order_" + "".join("rgb"[i] for i in p) for p in B.PERMS] + ["set_sat.equal"]
            if m >= 12:
                need += ["clip_color.n_lt_0.yes", "clip_color.x_gt_1.yes", "clip_color.n_lt_0.no", "clip_color.x_gt_1.no"]
            if lv.compose == 13:
                need += ["plus_lighter.clamped", "plus_lighter.unclamped"]
        return need


# ---- the reference frame ------------------------------------------------------------------------------------------------------
def _rect_mask(r) -> np.ndarray:
    y, x = np.mgrid[0:H, 0:W]
    return (x >= r[0]) & (x < r[2]) & (y >= r[1]) & (y < r[3])


def _expect(case: Case, alt=None, T=None):
    """The reference's frame: store8's per channel (byte, lo, hi, bound, wild), and each blend-stack store's ambiguity
    (level, channel) -> mask. `alt` = (level, channel): that store takes its other byte where its bound straddles a tie."""
    f = np.float32
    bd = [B.F(v) for v in np.moveaxis(BACKDROP.astype(f) / f(255), -1, 0)]
    rgba = bd
    if case.under is not None:
        u = np.array([(case.under.premul_rgba8_u32() >> (8 * i)) & 0xFF for i in range(4)], f) / f(255)
        rgba = B.over(rgba, [B.F(np.full((H, W), float(v))) for v in u])
    stack, amb = [], {}
    area = _rect_mask(case.clip).astype(np.float64)
    srcs = []
    inside = _rect_mask(case.clip)
    tiles = inside.reshape(H // 16, 16, W // 16, 16)
    partial = np.repeat(np.repeat(tiles.any(axis=(1, 3)) & ~tiles.all(axis=(1, 3)), 16, 0), 16, 1)
    backdrop = rgba
    for k, lv in enumerate(case.levels):
        packed = B.pack8(rgba)
        stored = []
        for ch, (b, lo, hi) in enumerate(packed):
            straddle = (lo != hi) & (partial if lv.mix == CLIP else True)
            if straddle.any():
                amb[(k, ch)] = straddle
            if alt == (k, ch):
                b = np.where(straddle, np.where(b == lo, hi, lo), b)
            stored.append(b)
        stack.append(np.stack(stored, -1))
        src = _source(k).copy()
        if k == len(case.levels) - 1:
            src[~_rect_mask(case.content)] = 0
        srcs.append(src)
        # the layer starts cleared; its source is drawn over transparent, exactly the texel
        rgba = B.leaf(src.astype(f) / f(255))[0]
    for k in reversed(range(len(case.levels))):
        lv = case.levels[k]
        bg, un_bg = B.leaf(stack[k].astype(f) / f(255))
        alpha = f(lv.alpha)
        if k == len(case.levels) - 1:  # the innermost layer: fg = texel * area * alpha, stated exactly in float32
            fg, un_fg = B.leaf((srcs[k].astype(f) / f(255)) * area.astype(f)[..., None] * alpha)
        else:
            fg = [c * area * float(alpha) if (lv.alpha != 1.0 or (area != 1).any()) else c for c in rgba]
            un_fg = None
        if lv.mix == LUM:
            rgba = B.luminance_mask(bg, fg, area, T, un_fg)
        elif lv.mix == CLIP:
            # coarse elides a clip layer (Mix::Clip) in the tiles its clip covers whole: there the source is drawn straight
            # over the unstored backdrop. Only the tiles the clip cuts store the backdrop and blend (coarse.wgsl BEGIN_CLIP /
            # END_CLIP, the `is_blend` test)
            assert len(case.levels) == 1
            elided = B.over(backdrop, fg)
            rgba = B.blend(bg, fg, 128, 3, T, un_bg, un_fg)
            rgba = [B.where(partial, q, B.where(inside, e, b)) for q, e, b in zip(rgba, elided, backdrop)]
        else:
            rgba = B.blend(bg, fg, lv.mix, lv.compose, T, un_bg, un_fg)
    return B.store8(rgba), amb


@functools.lru_cache(maxsize=8)
def expectation(case: Case):
    """Per channel: accepted byte range per alternative, plus the case's tallies."""
    T = B.Tally()
    out, amb = _expect(case, None, T)
    alts = []
    for key, mask in amb.items():
        alt_out, _ = _expect(case, key)
        alts.append((mask, alt_out))
    if amb:
        n = sum(m.astype(np.int32) for m in amb.values())
        assert n.max() <= 1, f"{case.name}: a pixel with two ambiguous blend-stack stores"
    return out, alts, T


def check(case: Case, img: np.ndarray) -> dict:
    """Assert that the frame img ((H, W, 4) uint8) is the reference's, under the rule in the module docstring."""
    out, alts, T = expectation(case)
    missing = [n for n in case.reach() if T[n] == 0]
    assert not missing, f"{case.name}: the frame does not reach {missing}"
    got = img.astype(np.int64)
    ok = np.zeros(got.shape, bool)
    exempt = np.zeros(got.shape, bool)
    unstated = np.zeros(got.shape, bool)
    bounds = []
    ties = np.zeros(got.shape, bool)
    for ch in range(4):
        b, lo, hi, e, wild, tie = out[ch]
        g = got[..., ch]
        ok[..., ch] = ((g >= lo) & (g <= hi)) | wild
        exempt[..., ch] = (lo != hi) & ~wild & ~tie
        ties[..., ch] = tie
        unstated[..., ch] = wild
        bounds.append(e[~wild])
        for mask, alt_out in alts:
            _, alo, ahi, _, awild, _ = alt_out[ch]
            ok[..., ch] |= mask & (((g >= alo) & (g <= ahi)) | awild)
            exempt[..., ch] |= mask & ((alo != lo) | (ahi != hi))
            unstated[..., ch] |= mask & awild
    bad = ~ok
    if bad.any():
        y, x, ch = (int(v) for v in np.argwhere(bad)[0])
        b, lo, hi, e, _, _ = out[ch]
        raise AssertionError(f"{case.name}: {int(bad.sum())} channel values differ from the reference, first at (y={y}, x={x}, "
                             f"channel {ch}): got {got[y, x, ch]}, want {b[y, x]} (accepted {lo[y, x]}..{hi[y, x]}, bound "
                             f"{e[y, x]:.3g} LSB); backdrop {tuple(BACKDROP[y, x])}, source {tuple(_source(0)[y, x])}")
    frac = float(exempt.mean())
    med = float(np.median(np.concatenate(bounds)))
    assert frac <= 0.01, f"{case.name}: {frac:.2%} of the channel values exempt"
    assert med < 0.01, f"{case.name}: median bound {med:.3g} LSB"
    # the channels whose float32 value the reference cannot state (blend_ref's degenerate rules: mostly a grey on the gamut's
    # edge in clip_color, where float32's lum of the grey equals it and the quotient is 0/0) stay a small, known minority
    assert unstated.mean() <= 0.08, f"{case.name}: {unstated.mean():.2%} of the channel values unstated"
    return dict(exempt=frac, median_bound=med, exact_ties=float(ties.mean()), unstated=float(unstated.mean()))


# ---- the cases ----------------------------------------------------------------------------------------------------------------
def _grid(mix, compose):
    return Case(f"mix_{B.MIXES[mix]}_{B.COMPOSES[compose]}", (Level(mix, compose),))


GRID_ALL = [_grid(m, c) for m in range(16) for c in range(14)]
# the CPU runs every mix under src-over, and every compose under normal, multiply (separable) and hue (non-separable)
GRID_CPU = [c for c in GRID_ALL if c.levels[0].compose == 3 or c.levels[0].mix in (0, 1, 12)]

ALPHA = [Case(f"alpha_{n}_{B.MIXES[m]}_{B.COMPOSES[c]}", (Level(m, c, a),))
         for n, a in (("0", 0.0), ("1_255", 1 / 255), ("0.3", 0.3), ("0.5", 0.5), ("254_255", 254 / 255), ("1", 1.0))
         for m, c in ((0, 3), (1, 9), (12, 11))]

# clip layers (Mix::Clip, the src-over fast path) over translucent backdrops: a colour over the backdrop image, so the
# stored backdrop is a computed value, rounded by BEGIN_CLIP's pack4x8unorm
CLIPS = [Case("clip_under_translucent", (Level(CLIP),), under=Color(0.3, 0.7, 0.2, 0.45), clip=(0, 0, W, 200)),
         Case("clip_under_opaque_ish", (Level(CLIP),), under=Color(0.9, 0.1, 0.55, 0.8), clip=(0, 0, 200, 200))]

# luminance masks: the clip covers x < 200 (tile column 12 is cut, so its pixels x >= 200 are area 0 inside a clipped
# tile); the mask content covers y < 176 only, so part of the clip region has no content
MASKS = [Case(f"luminance_mask_alpha_{n}", (Level(LUM, 3, a),), clip=(0, 0, 200, H), content=(0, 0, W, 176))
         for n, a in (("1", 1.0), ("0.6", 0.6))]

# six nested layers: levels 0-3 keep their backdrops in registers, 4 and 5 in blend_spill (VB_BLEND_STACK_SPLIT = 4)
CHAINS = [Case("chain_six_levels", (Level(1, 9), Level(12, 3), Level(9, 11, 0.75), Level(2, 4), Level(15, 12), Level(6, 5))),
          Case("chain_six_levels_b", (Level(14, 10), Level(3, 13), Level(11, 3), Level(13, 9, 0.5), Level(8, 1), Level(7, 3)))]

CASES_CPU = GRID_CPU + ALPHA + CLIPS + MASKS + CHAINS
CASES_GPU = GRID_ALL + ALPHA + CLIPS + MASKS + CHAINS


@functools.lru_cache(maxsize=1)
def _scene_cache():
    return {}


def packed_scene(case: Case):
    cache = _scene_cache()
    if case.name not in cache:
        cache.clear()
        cache[case.name] = resolve(case.scene().encoding)
    return cache[case.name]


@pytest.mark.parametrize("case", CASES_CPU, ids=[c.name for c in CASES_CPU])
def test_reference_matches_oracle(oracle, case):
    """The reference and the oracle's full pipeline (area AA) agree on every case."""
    img = oracle.render(packed_scene(case), W, H, 0, AA_AREA)
    check(case, img)


# ---- spot values from the spec, computed by hand ------------------------------------------------------------------------------
def _mix1(mode, cb, cs):
    return B.w3c_mix(mode, cb, cs)


def test_spot_values():
    # colour-dodge: cb = 0 is tested first, so (cb, cs) = (0, 1) is 0; colour-burn: cb = 1 first, so (1, 0) is 1
    assert _mix1("color_dodge", [0, 0.5, 0.2], [1, 1, 0.6]) == [0.0, 1.0, 0.5]
    assert _mix1("color_burn", [1, 0.5, 0.6], [0, 0, 0.8]) == [1.0, 0.0, 0.5]
    # soft-light at cs = 1 is D(cb): the polynomial up to cb = 1/4, D(1/8) = ((16/8 - 12)/8 + 4)/8 = 0.34375 and D(1/4) =
    # 1/2, then sqrt; at cs = 1/4, cb - (1/2) cb (1 - cb)
    assert np.allclose(_mix1("soft_light", [0.125, 0.25, 0.5], [1, 1, 1]), [0.34375, 0.5, 0.5 ** 0.5], rtol=0, atol=1e-15)
    assert np.allclose(_mix1("soft_light", [0.5, 0.2, 1], [0.25, 0.25, 0.25]), [0.375, 0.12, 1], rtol=0, atol=1e-15)
    # hue of a grey source keeps the backdrop's luminance with zero saturation: grey at lum(cb)
    cb = [0.8, 0.4, 0.2]
    l = 0.3 * 0.8 + 0.59 * 0.4 + 0.11 * 0.2
    assert np.allclose(_mix1("hue", cb, [0.5, 0.5, 0.5]), [l, l, l])
    # luminosity of black onto a colour: every channel to 0 (ClipColor's n < 0 branch)
    assert np.allclose(_mix1("luminosity", [0.9, 0.1, 0.3], [0, 0, 0]), [0, 0, 0], atol=1e-12)
    # plus-lighter saturates colour and alpha at 1
    assert np.allclose(B.w3c_composite(0, 13, [0.8, 0.2, 0.6], 0.9, [0.7, 0.1, 0.9], 0.8), [1.0, 0.26, 1.0, 1.0])
    # Porter-Duff src-atop: Fa = ab, Fb = 1 - as
    assert np.allclose(B.w3c_composite(0, 9, [0.2, 0.4, 0.6], 0.5, [1.0, 0.0, 0.5], 0.25),
                       [0.25 * 0.5 * 1.0 + 0.5 * 0.75 * 0.2, 0.5 * 0.75 * 0.4, 0.25 * 0.5 * 0.5 + 0.5 * 0.75 * 0.6, 0.25 * 0.5 + 0.5 * 0.75])


def test_bound_covers_float32():
    """The error bound contains float32's result for a formula with every kind of operation, on random inputs."""
    rng = np.random.default_rng(3)
    a, b, c = (rng.random(10000) for _ in range(3))
    fa, fb, fc = (B.F(x.astype(np.float32).astype(np.float64)) for x in (a, b, c))
    r = ((fa * fb + fc) / (fb + 0.5)).sqrt() - B.fmin(fa, fc) * B.const(0.59)
    x, y, z = (v.astype(np.float32) for v in (a, b, c))
    g = np.sqrt((x * y + z) / (y + np.float32(0.5))) - np.minimum(x, z) * np.float32(0.59)
    assert (np.abs(g.astype(np.float64) - r.v) <= r.e).all()
    assert np.median(r.e) < 1e-6
