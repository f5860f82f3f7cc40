"""Scene encoding: the six `vello_encoding` streams, the packed scene buffer and `Layout`.

This is the host side *above* the drop-in boundary (SURVEY.md section 1): it exists so that tests and
benchmarks can produce byte-identical inputs to what `Resolver::resolve` hands to the GPU
pipeline. It restates, it does not copy:

* `PathEncoder` state machine        -- vello_encoding/src/path.rs:425-838
* `Style` bit layout                 -- vello_encoding/src/path.rs:11-120
* `Encoding::encode_*`               -- vello_encoding/src/encoding.rs:189-530
* `Scene::{fill,stroke,push_layer..}`-- vello/src/scene.rs:100-470
* `resolve_solid_paths_only/resolve` -- vello_encoding/src/resolve.rs:107-399
* draw tags / draw data structs      -- vello_encoding/src/draw.rs:17-236
* f32<->f16                          -- vello_encoding/src/math.rs:93-145
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass, field
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import shapes as _shapes
from .shapes import Affine

# ---------------------------------------------------------------------------------------------
# Path tags (vello_encoding/src/path.rs:244-316)
# ---------------------------------------------------------------------------------------------
TAG_LINE_TO_F32 = 0x9
TAG_QUAD_TO_F32 = 0xA
TAG_CUBIC_TO_F32 = 0xB
TAG_LINE_TO_I16 = 0x1
TAG_QUAD_TO_I16 = 0x2
TAG_CUBIC_TO_I16 = 0x3
TAG_TRANSFORM = 0x20
TAG_PATH = 0x10
TAG_STYLE = 0x40
TAG_SUBPATH_END_BIT = 0x4

# Draw tags (vello_encoding/src/draw.rs:17-44)
DRAWTAG_NOP = 0
DRAWTAG_COLOR = 0x44
DRAWTAG_LINEAR_GRADIENT = 0x114
DRAWTAG_RADIAL_GRADIENT = 0x29C
DRAWTAG_SWEEP_GRADIENT = 0x254
DRAWTAG_IMAGE = 0x28C
DRAWTAG_BLUR_RECT = 0x2D4
DRAWTAG_BEGIN_CLIP = 0x49
DRAWTAG_END_CLIP = 0x21


def drawtag_info_size(tag: int) -> int:
    """Words of `info` a draw tag occupies (draw.rs: `(tag >> 6) & 0xf`)."""
    return (tag >> 6) & 0xF


# Style flags (path.rs:30-66)
STYLE_FLAGS_STYLE_BIT = 0x8000_0000
STYLE_FLAGS_FILL_BIT = 0x4000_0000
STYLE_JOIN_BEVEL = 0
STYLE_JOIN_MITER = 0x1000_0000
STYLE_JOIN_ROUND = 0x2000_0000
STYLE_CAP_BUTT = 0
STYLE_CAP_SQUARE = 0x0100_0000
STYLE_CAP_ROUND = 0x0200_0000

FILL_NON_ZERO = 0
FILL_EVEN_ODD = 1

# Blend (peniko::Mix / Compose numeric values; shared/blend.wgsl:7-24,220-233)
MIX_NORMAL, MIX_MULTIPLY, MIX_SCREEN, MIX_OVERLAY, MIX_DARKEN, MIX_LIGHTEN = 0, 1, 2, 3, 4, 5
MIX_COLOR_DODGE, MIX_COLOR_BURN, MIX_HARD_LIGHT, MIX_SOFT_LIGHT = 6, 7, 8, 9
MIX_DIFFERENCE, MIX_EXCLUSION, MIX_HUE, MIX_SATURATION, MIX_COLOR, MIX_LUMINOSITY = 10, 11, 12, 13, 14, 15
MIX_CLIP = 128
COMPOSE_CLEAR, COMPOSE_COPY, COMPOSE_DEST, COMPOSE_SRC_OVER, COMPOSE_DEST_OVER = 0, 1, 2, 3, 4
COMPOSE_SRC_IN, COMPOSE_DEST_IN, COMPOSE_SRC_OUT, COMPOSE_DEST_OUT = 5, 6, 7, 8
COMPOSE_SRC_ATOP, COMPOSE_DEST_ATOP, COMPOSE_XOR, COMPOSE_PLUS, COMPOSE_PLUS_LIGHTER = 9, 10, 11, 12, 13

CLIP_BLEND_MODE = 0x8003  # draw.rs:216 (Mix::Clip << 8 | SrcOver)
LUMINANCE_MASK_BLEND_MODE = 0x10000  # draw.rs:215

EXTEND_PAD, EXTEND_REPEAT, EXTEND_REFLECT = 0, 1, 2
QUALITY_LOW, QUALITY_MEDIUM, QUALITY_HIGH = 0, 1, 2
FORMAT_RGBA8, FORMAT_BGRA8 = 0, 1
ALPHA_STRAIGHT, ALPHA_PREMULTIPLIED = 0, 1

PATH_REDUCE_WG = 256  # config.rs


def _f32(x: float) -> float:
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _f32_bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f32_to_f16(val: float) -> int:
    """math.rs:93-127 (Giesen float_to_half_fast3), bit-for-bit."""
    INF_32 = 255 << 23
    INF_16 = 31 << 23
    MAGIC = 15 << 23
    ROUND_MASK = (~0xFFF) & 0xFFFFFFFF
    u = _f32_bits(val)
    sign = u & 0x8000_0000
    u ^= sign
    if u >= INF_32:
        out = 0x7E00 if u > INF_32 else 0x7C00
    else:
        u &= ROUND_MASK
        f = np.float32(np.array([u], dtype=np.uint32).view(np.float32)[0]) * np.float32(
            np.array([MAGIC], dtype=np.uint32).view(np.float32)[0]
        )
        u = int(np.array([f], dtype=np.float32).view(np.uint32)[0])
        u = (u - ROUND_MASK) & 0xFFFFFFFF
        if u > INF_16:
            u = INF_16
        out = (u >> 13) & 0xFFFF
    return out | (sign >> 16)


def f16_to_f32(bits: int) -> float:
    """math.rs:133-154."""
    return float(np.array([bits], dtype=np.uint16).view(np.float16)[0])


# ---------------------------------------------------------------------------------------------
# Colours and brushes
# ---------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Color:
    """Straight-alpha sRGB colour, components in 0..1 (peniko `AlphaColor<Srgb>`)."""

    r: float
    g: float
    b: float
    a: float = 1.0

    @staticmethod
    def from_rgba8(r: int, g: int, b: int, a: int = 255) -> "Color":
        f = np.float32
        return Color(float(f(r) / f(255)), float(f(g) / f(255)), float(f(b) / f(255)), float(f(a) / f(255)))

    def with_alpha(self, a: float) -> "Color":
        return Color(self.r, self.g, self.b, a)

    def multiply_alpha(self, m: float) -> "Color":
        return Color(self.r, self.g, self.b, float(np.float32(self.a) * np.float32(m)))

    def premul_rgba8_u32(self) -> int:
        """`premultiply().to_rgba8().to_u32()` -- draw.rs:76-84; r is the low byte."""
        f = np.float32
        a = f(self.a)
        comps = [f(self.r) * a, f(self.g) * a, f(self.b) * a, a]
        out = 0
        for i, c in enumerate(comps):
            v = int(min(max(math.floor(float(c * f(255.0) + f(0.5))), 0), 255))
            out |= v << (8 * i)
        return out


BLACK = Color(0.0, 0.0, 0.0, 1.0)
WHITE = Color(1.0, 1.0, 1.0, 1.0)
RED = Color(1.0, 0.0, 0.0, 1.0)
LIME = Color(0.0, 1.0, 0.0, 1.0)
BLUE = Color(0.0, 0.0, 1.0, 1.0)
TRANSPARENT = Color(0.0, 0.0, 0.0, 0.0)


@dataclass
class Gradient:
    kind: str  # "linear" | "radial" | "sweep"
    params: Tuple[float, ...]
    stops: List[Tuple[float, Color]]
    extend: int = EXTEND_PAD
    premul_interp: bool = True  # peniko default InterpolationAlphaSpace::Premultiplied

    @staticmethod
    def linear(p0, p1, stops, extend=EXTEND_PAD, premul_interp=True) -> "Gradient":
        return Gradient("linear", (p0[0], p0[1], p1[0], p1[1]), list(stops), extend, premul_interp)

    @staticmethod
    def radial(c0, r0, c1, r1, stops, extend=EXTEND_PAD, premul_interp=True) -> "Gradient":
        return Gradient("radial", (c0[0], c0[1], c1[0], c1[1], r0, r1), list(stops), extend, premul_interp)

    @staticmethod
    def sweep(center, a0, a1, stops, extend=EXTEND_PAD, premul_interp=True) -> "Gradient":
        return Gradient("sweep", (center[0], center[1], a0, a1), list(stops), extend, premul_interp)


@dataclass
class Image:
    """RGBA8/BGRA8 image + sampler (peniko `ImageBrush`).

    `key` (optional) names the image in the atlas the way vello's blob id does: images with the same key share one atlas slot,
    and a renderer's override of the key (`Renderer.override_image`) supplies its pixels from device memory at the device
    resolve. A registered texture (`Renderer.register_texture`) has a key that points at no host memory and a zero-strided
    `data` of zeros, so the host resolve leaves its atlas region zero."""

    data: np.ndarray  # (h, w, 4) uint8
    format: int = FORMAT_RGBA8
    alpha_type: int = ALPHA_STRAIGHT
    quality: int = QUALITY_MEDIUM
    x_extend: int = EXTEND_PAD
    y_extend: int = EXTEND_PAD
    alpha: float = 1.0
    key: Optional[int] = None

    @property
    def width(self) -> int:
        return int(self.data.shape[1])

    @property
    def height(self) -> int:
        return int(self.data.shape[0])


@dataclass
class Stroke:
    """kurbo `Stroke` (defaults: round join, round caps, miter limit 4)."""

    width: float
    join: int = STYLE_JOIN_ROUND
    miter_limit: float = 4.0
    start_cap: int = STYLE_CAP_ROUND
    end_cap: int = STYLE_CAP_ROUND
    dash_pattern: Tuple[float, ...] = ()  # kurbo Stroke::dash_pattern / dash_offset: expanded on the CPU (scene.rs:411-438)
    dash_offset: float = 0.0


def style_from_fill(fill: int) -> Tuple[int, float]:
    return (STYLE_FLAGS_FILL_BIT if fill == FILL_EVEN_ODD else 0, 0.0)


def style_from_stroke(s: Stroke) -> Optional[Tuple[int, float]]:
    if s.width == 0.0:
        return None
    flags = STYLE_FLAGS_STYLE_BIT | s.join | (s.start_cap << 2) | s.end_cap | f32_to_f16(s.miter_limit)
    return (flags, _f32(s.width))


# ---------------------------------------------------------------------------------------------
# Path encoder
# ---------------------------------------------------------------------------------------------
_EPS = 1e-12  # path.rs:841

_START, _MOVETO, _NONEMPTY = 0, 1, 2


class PathEncoder:
    """State machine restated from path.rs:425-838. Coordinates are rounded to f32 on entry."""

    def __init__(self, enc: "Encoding", is_fill: bool):
        self.enc = enc
        self.tags = enc.path_tags
        self.data = enc.path_data  # list of python floats already rounded to f32
        self.first_point = (0.0, 0.0)
        self.first_start_tangent_end = (0.0, 0.0)
        self.state = _START
        self.n_encoded_segments = 0
        self.is_fill = is_fill

    def move_to(self, x, y):
        x, y = _f32(x), _f32(y)
        if self.is_fill:
            self.close()
        if self.state == _MOVETO:
            del self.data[-2:]
        elif self.state == _NONEMPTY:
            if not self.is_fill:
                self._insert_stroke_cap_marker(False)
            if self.tags:
                self.tags[-1] |= TAG_SUBPATH_END_BIT
        self.first_point = (x, y)
        self.data.extend((x, y))
        self.state = _MOVETO

    def _last_point(self):
        return (self.data[-2], self.data[-1])

    def _zero_len(self, p1, p2=None, p3=None):
        p0 = self._last_point()
        p2 = p2 or p1
        p3 = p3 or p1
        f = np.float32
        xs = [f(p0[0]), f(p1[0]), f(p2[0]), f(p3[0])]
        ys = [f(p0[1]), f(p1[1]), f(p2[1]), f(p3[1])]
        return not ((max(xs) - min(xs)) > _EPS or (max(ys) - min(ys)) > _EPS)

    @staticmethod
    def _neq(a, b):
        f = np.float32
        return abs(f(a[0]) - f(b[0])) > _EPS or abs(f(a[1]) - f(b[1])) > _EPS

    def line_to(self, x, y):
        x, y = _f32(x), _f32(y)
        if self.state == _START:
            if self.n_encoded_segments == 0:
                self.move_to(x, y)
                return
            self.move_to(*self.first_point)
        if self.state == _MOVETO:
            p0 = self.first_point
            if not self._neq((x, y), p0):
                return
            f = np.float32
            third = f(1.0) / f(3.0)
            self.first_start_tangent_end = (
                float(f(p0[0]) + third * (f(x) - f(p0[0]))),
                float(f(p0[1]) + third * (f(y) - f(p0[1]))),
            )
        if self._zero_len((x, y)):
            return
        self.data.extend((x, y))
        self.tags.append(TAG_LINE_TO_F32)
        self.state = _NONEMPTY
        self.n_encoded_segments += 1

    def quad_to(self, x1, y1, x2, y2):
        x1, y1, x2, y2 = _f32(x1), _f32(y1), _f32(x2), _f32(y2)
        if self.state == _START:
            if self.n_encoded_segments == 0:
                self.move_to(x2, y2)
                return
            self.move_to(*self.first_point)
        if self.state == _MOVETO:
            p0 = self.first_point
            f = np.float32
            third = f(1.0) / f(3.0)
            if self._neq((x1, y1), p0):
                t = (float(f(x1) + third * (f(p0[0]) - f(x1))), float(f(y1) + third * (f(p0[1]) - f(y1))))
            elif self._neq((x2, y2), p0):
                t = (float(f(x1) + third * (f(x2) - f(x1))), float(f(y1) + third * (f(y2) - f(y1))))
            else:
                return
            self.first_start_tangent_end = t
        if self._zero_len((x1, y1), (x2, y2)):
            return
        self.data.extend((x1, y1, x2, y2))
        self.tags.append(TAG_QUAD_TO_F32)
        self.state = _NONEMPTY
        self.n_encoded_segments += 1

    def cubic_to(self, x1, y1, x2, y2, x3, y3):
        x1, y1, x2, y2, x3, y3 = (_f32(v) for v in (x1, y1, x2, y2, x3, y3))
        if self.state == _START:
            if self.n_encoded_segments == 0:
                self.move_to(x3, y3)
                return
            self.move_to(*self.first_point)
        if self.state == _MOVETO:
            p0 = self.first_point
            if self._neq((x1, y1), p0):
                t = (x1, y1)
            elif self._neq((x2, y2), p0):
                t = (x2, y2)
            elif self._neq((x3, y3), p0):
                t = (x3, y3)
            else:
                return
            self.first_start_tangent_end = t
        if self._zero_len((x1, y1), (x2, y2), (x3, y3)):
            return
        self.data.extend((x1, y1, x2, y2, x3, y3))
        self.tags.append(TAG_CUBIC_TO_F32)
        self.state = _NONEMPTY
        self.n_encoded_segments += 1

    def empty_path(self):
        self.data.extend((0.0, 0.0, 0.0, 0.0))
        self.tags.append(TAG_LINE_TO_F32)
        self.n_encoded_segments += 1

    def close(self):
        if self.state == _START:
            return
        if self.state == _MOVETO:
            del self.data[-2:]
            self.state = _START
            return
        if len(self.data) < 2:
            return
        fp = self.first_point
        lp = self._last_point()
        # bitwise comparison of the f32 pairs (path.rs:661-662)
        if _f32_bits(lp[0]) != _f32_bits(fp[0]) or _f32_bits(lp[1]) != _f32_bits(fp[1]):
            self.data.extend(fp)
            self.tags.append(TAG_LINE_TO_F32)
            self.n_encoded_segments += 1
        if not self.is_fill:
            self._insert_stroke_cap_marker(True)
        if self.tags:
            self.tags[-1] |= TAG_SUBPATH_END_BIT
        self.state = _START

    def _insert_stroke_cap_marker(self, is_closed: bool):
        assert not self.is_fill and self.state == _NONEMPTY
        if is_closed:
            self.line_to(*self.first_start_tangent_end)
        else:
            self.quad_to(self.first_point[0], self.first_point[1], *self.first_start_tangent_end)

    def path_elements(self, els: Iterable[tuple]):
        for el in els:
            k = el[0]
            if k == "M":
                self.move_to(el[1], el[2])
            elif k == "L":
                self.line_to(el[1], el[2])
            elif k == "Q":
                self.quad_to(el[1], el[2], el[3], el[4])
            elif k == "C":
                self.cubic_to(el[1], el[2], el[3], el[4], el[5], el[6])
            elif k == "Z":
                self.close()
            else:
                raise ValueError(k)

    def finish(self, insert_path_marker: bool) -> int:
        if self.is_fill:
            self.close()
        if self.state == _MOVETO:
            del self.data[-2:]
        if self.n_encoded_segments != 0:
            if not self.is_fill and self.state == _NONEMPTY:
                self._insert_stroke_cap_marker(False)
            if self.tags:
                self.tags[-1] |= TAG_SUBPATH_END_BIT
            self.enc.n_path_segments += self.n_encoded_segments
            if insert_path_marker:
                self.tags.append(TAG_PATH)
                self.enc.n_paths += 1
        return self.n_encoded_segments


# ---------------------------------------------------------------------------------------------
# Encoding (the six streams) + late-bound resources
# ---------------------------------------------------------------------------------------------
@dataclass
class Layout:
    """`vello_encoding::Layout` (resolve.rs:16-39): 10 x u32, offsets in u32 words."""

    n_draw_objects: int = 0
    n_paths: int = 0
    n_clips: int = 0
    bin_data_start: int = 0
    path_tag_base: int = 0
    path_data_base: int = 0
    draw_tag_base: int = 0
    draw_data_base: int = 0
    transform_base: int = 0
    style_base: int = 0

    def as_array(self) -> np.ndarray:
        return np.array(
            [
                self.n_draw_objects, self.n_paths, self.n_clips, self.bin_data_start,
                self.path_tag_base, self.path_data_base, self.draw_tag_base, self.draw_data_base,
                self.transform_base, self.style_base,
            ],
            dtype=np.uint32,
        )

    def path_tags_size(self) -> int:
        """Bytes of the (padded) tag stream (resolve.rs `path_tags_size`)."""
        return (self.path_data_base - self.path_tag_base) * 4


class Encoding:
    """Restated `vello_encoding::Encoding` (encoding.rs:26-53)."""

    def __init__(self):
        self.path_tags: List[int] = []
        self.path_data: List[float] = []  # f32 values
        self.draw_tags: List[int] = []
        self.draw_data: List[int] = []  # u32 words
        self.transforms: List[Tuple[float, ...]] = []  # 6 x f32
        self.styles: List[Tuple[int, float]] = []
        self.n_paths = 0
        self.n_path_segments = 0
        self.n_clips = 0
        self.n_open_clips = 0
        # late bound
        self.ramp_patches: List[dict] = []
        self.image_patches: List[dict] = []
        self._force_next = False

    # -- styles / transforms ------------------------------------------------------------------
    def encode_style(self, style: Tuple[int, float]):
        if not self.styles or self.styles[-1] != style:
            self.path_tags.append(TAG_STYLE)
            self.styles.append(style)

    def encode_fill_style(self, fill: int):
        self.encode_style(style_from_fill(fill))

    def encode_stroke_style(self, stroke: Stroke) -> bool:
        st = style_from_stroke(stroke)
        if st is None:
            return False
        self.encode_style(st)
        return True

    def encode_transform(self, t: Affine) -> bool:
        tt = tuple(_f32(v) for v in t.coeffs)
        if not self.transforms or self.transforms[-1] != tt:
            self.path_tags.append(TAG_TRANSFORM)
            self.transforms.append(tt)
            return True
        return False

    def swap_last_path_tags(self):
        self.path_tags[-1], self.path_tags[-2] = self.path_tags[-2], self.path_tags[-1]

    # -- paths --------------------------------------------------------------------------------
    def encode_path_elements(self, els, is_fill: bool) -> bool:
        pe = PathEncoder(self, is_fill)
        pe.path_elements(els)
        return pe.finish(True) != 0

    def encode_shape(self, shape, is_fill: bool, tolerance: float = 0.1) -> bool:
        return self.encode_path_elements(_shapes.path_elements(shape, tolerance), is_fill)

    def encode_empty_shape(self):
        pe = PathEncoder(self, True)
        pe.empty_path()
        pe.finish(True)

    # -- brushes ------------------------------------------------------------------------------
    def encode_color(self, color: Color):
        self.draw_tags.append(DRAWTAG_COLOR)
        self.draw_data.append(color.premul_rgba8_u32())

    def _add_ramp(self, g: Gradient, alpha: float):
        stops = g.stops
        if alpha != 1.0:
            stops = [(o, c.multiply_alpha(alpha)) for (o, c) in stops]
        if len(stops) == 0:
            return "empty", None
        if len(stops) == 1:
            return "one", stops[0][1]
        self.ramp_patches.append(
            dict(draw_data_offset=len(self.draw_data), stops=stops, extend=g.extend, premul=g.premul_interp)
        )
        return "many", None

    def encode_brush(self, brush, alpha: float = 1.0):
        if isinstance(brush, Color):
            self.encode_color(brush if alpha == 1.0 else brush.multiply_alpha(alpha))
        elif isinstance(brush, Gradient):
            g = brush
            p = [_f32(v) for v in g.params]
            if g.kind == "radial":
                eps = 1.0 / (1 << 12)
                if (p[0], p[1]) == (p[2], p[3]) and abs(p[4] - p[5]) < eps:
                    self.encode_color(TRANSPARENT)
                    return
            if g.kind == "sweep":
                tau = 2.0 * math.pi
                t0, t1 = _f32(_f32(g.params[2]) / _f32(tau)), _f32(_f32(g.params[3]) / _f32(tau))
                if abs(t0 - t1) < 1.0 / (1 << 15):
                    self.encode_color(TRANSPARENT)
                    return
            kind, col = self._add_ramp(g, alpha)
            if kind == "empty":
                self.encode_color(TRANSPARENT)
            elif kind == "one":
                self.encode_color(col)
            elif g.kind == "linear":
                self.draw_tags.append(DRAWTAG_LINEAR_GRADIENT)
                self.draw_data.extend([0] + [_f32_bits(v) for v in p[:4]])
            elif g.kind == "radial":
                self.draw_tags.append(DRAWTAG_RADIAL_GRADIENT)
                self.draw_data.extend([0] + [_f32_bits(v) for v in p[:6]])
            else:
                self.draw_tags.append(DRAWTAG_SWEEP_GRADIENT)
                self.draw_data.extend([0, _f32_bits(p[0]), _f32_bits(p[1]), _f32_bits(t0), _f32_bits(t1)])
        elif isinstance(brush, Image):
            im = brush
            a8 = int(np.float32(im.alpha) * np.float32(alpha) * np.float32(255.0) + np.float32(0.5)) & 0xFF
            self.image_patches.append(dict(draw_data_offset=len(self.draw_data), image=im))
            self.draw_tags.append(DRAWTAG_IMAGE)
            self.draw_data.extend(
                [
                    0,
                    ((im.width << 16) | (im.height & 0xFFFF)) & 0xFFFFFFFF,
                    (im.format << 15) | (im.alpha_type << 14) | (im.quality << 12)
                    | (im.x_extend << 10) | (im.y_extend << 8) | a8,
                ]
            )
        else:
            raise TypeError(type(brush))

    def encode_blurred_rounded_rect(self, color: Color, width, height, radius, std_dev):
        self.draw_tags.append(DRAWTAG_BLUR_RECT)
        self.draw_data.extend([color.premul_rgba8_u32()] + [_f32_bits(v) for v in (width, height, radius, std_dev)])

    def encode_begin_clip(self, blend_mode: int, alpha: float):
        self.draw_tags.append(DRAWTAG_BEGIN_CLIP)
        self.draw_data.extend([blend_mode, _f32_bits(alpha)])
        self.n_clips += 1
        self.n_open_clips += 1

    def append(self, other: "Encoding", transform: Optional[Affine] = None):
        """`Encoding::append` (encoding.rs:94-174) without glyph runs: concatenate `other`'s streams; its transforms are
        pre-multiplied by `transform` in f32 (`Transform * Transform`, math.rs:51-73); late-bound patches move with the
        draw data."""
        dd = len(self.draw_data)
        self.ramp_patches.extend(dict(p, draw_data_offset=p["draw_data_offset"] + dd) for p in other.ramp_patches)
        self.image_patches.extend(dict(p, draw_data_offset=p["draw_data_offset"] + dd) for p in other.image_patches)
        self.path_tags.extend(other.path_tags)
        self.path_data.extend(other.path_data)
        self.draw_tags.extend(other.draw_tags)
        self.draw_data.extend(other.draw_data)
        self.n_paths += other.n_paths
        self.n_path_segments += other.n_path_segments
        self.n_clips += other.n_clips
        self.n_open_clips += other.n_open_clips
        if transform is not None:
            f = np.float32
            a = [f(v) for v in transform.coeffs]
            for x in other.transforms:
                b = [f(v) for v in x]
                self.transforms.append(tuple(float(v) for v in (
                    a[0] * b[0] + a[2] * b[1], a[1] * b[0] + a[3] * b[1], a[0] * b[2] + a[2] * b[3], a[1] * b[2] + a[3] * b[3],
                    a[0] * b[4] + a[2] * b[5] + a[4], a[1] * b[4] + a[3] * b[5] + a[5])))
        else:
            self.transforms.extend(other.transforms)
        self.styles.extend(other.styles)

    def encode_end_clip(self):
        if self.n_open_clips > 0:
            self.draw_tags.append(DRAWTAG_END_CLIP)
            self.path_tags.append(TAG_PATH)
            self.n_paths += 1
            self.n_clips += 1
            self.n_open_clips -= 1


# ---------------------------------------------------------------------------------------------
# Scene: the user-facing builder (vello/src/scene.rs)
# ---------------------------------------------------------------------------------------------
class Scene:
    def __init__(self):
        self.encoding = Encoding()

    @property
    def n_draw_objects(self) -> int:
        """The draw objects encoded so far: the draw-object index the next fill, stroke, draw_image, blurred rectangle or
        push_*_layer receives (read it before and after a call to note the index that call gave; a shape that encodes nothing
        adds no draw). `Renderer.hit_test` answers with these indices."""
        return len(self.encoding.draw_tags)

    @property
    def n_points(self) -> int:
        """The path points encoded so far (path-data words / 2): the row `Renderer.bind_path_points` reads for the next point
        a call encodes (read it before and after a call to learn the rows that call produced). A fill or stroke whose shape
        encodes nothing adds no point; a push_*_layer whose clip encodes nothing adds 2, the empty path (0, 0) -> (0, 0) that
        stands in for the clip. A move-to writes 1 point, a line-to, quad-to and cubic-to 1, 2 and 3; a closed fill subpath repeats its start
        point when its last point differs; a stroke subpath ends with a cap marker (closed: a line-to, 1 point; open: a quad-to,
        2 points); a dash's pieces are separate subpaths; arcs, circles and ellipses are cubics."""
        return len(self.encoding.path_data) // 2

    @property
    def n_stops(self) -> int:
        """The gradient stops encoded so far: the stops of the ramp patches, concatenated in draw-data order, and the row
        `Renderer.bind_gradient_stops` reads for the next stop a call encodes (read it before and after a call to learn the
        rows that call produced). Only a gradient that keeps a ramp adds stops, after the brush alpha; a gradient with no stop
        or one stop, and a degenerate radial or sweep gradient, is encoded as a colour and adds none."""
        return sum(len(p["stops"]) for p in self.encoding.ramp_patches)

    @property
    def n_transforms(self) -> int:
        """The transform-stream entries encoded so far: the row `Renderer.bind_transforms` reads for the next entry a call
        pushes (read it before and after a call to learn the rows that call produced). A call pushes its transform only when it
        differs from the last entry, so consecutive calls with equal transforms share one row. A brush transform is an entry of
        its own, after the shape's, holding `transform * brush_transform`; a blurred rectangle pushes `transform *
        translate(centre)` the same way, and `draw_image` pushes only its transform. A fill whose shape encodes nothing still
        pushes its transform; a stroke of width 0 pushes nothing."""
        return len(self.encoding.transforms)

    def fill(self, style: int, transform: Affine, brush, brush_transform: Optional[Affine], shape):
        e = self.encoding
        e.encode_transform(transform)
        e.encode_fill_style(style)
        if e.encode_shape(shape, True):
            if brush_transform is not None and e.encode_transform(transform * brush_transform):
                e.swap_last_path_tags()
            e.encode_brush(brush, 1.0)

    def _stroke_inner(self, stroke: Stroke, transform: Affine, shape) -> bool:
        e = self.encoding
        e.encode_transform(transform)
        ok = e.encode_stroke_style(stroke)
        assert ok
        # non-dashed strokes go through Encoding::encode_shape -> PathEncoder::shape -> path_elements(0.1)
        # (vello/src/scene.rs:417-421, vello_encoding/src/path.rs:655-657); only the dash expansion uses 0.01
        if not stroke.dash_pattern:
            return e.encode_shape(shape, False)
        # dashes are not supported by the GPU pipeline: the shape (flattened at SHAPE_TOLERANCE = 0.01) is cut into dashes
        # on the CPU by kurbo::dash and the dashes are encoded as the path (scene.rs:404,422-437)
        dashed = _shapes.dash(_shapes.path_elements(shape, 0.01), stroke.dash_offset, stroke.dash_pattern)
        return e.encode_path_elements(dashed, False)

    def stroke(self, stroke: Stroke, transform: Affine, brush, brush_transform: Optional[Affine], shape):
        if stroke.width == 0.0:
            return
        e = self.encoding
        if self._stroke_inner(stroke, transform, shape):
            if brush_transform is not None and e.encode_transform(transform * brush_transform):
                e.swap_last_path_tags()
            e.encode_brush(brush, 1.0)

    def _push_layer_inner(self, blend_mode: int, alpha: float, clip_style, transform: Affine, clip):
        e = self.encoding
        if isinstance(clip_style, Stroke):
            if clip_style.width == 0.0:
                e.encode_fill_style(FILL_NON_ZERO)
                ok = False
            else:
                ok = self._stroke_inner(clip_style, transform, clip)
        else:
            e.encode_transform(transform)
            e.encode_fill_style(clip_style)
            ok = e.encode_shape(clip, True)
        if not ok:
            e.encode_empty_shape()
        e.encode_begin_clip(blend_mode, alpha)

    def push_layer(self, clip_style, mix: int, compose: int, alpha: float, transform: Affine, clip):
        self._push_layer_inner(((mix << 8) | compose), _f32(min(max(alpha, 0.0), 1.0)), clip_style, transform, clip)

    def push_luminance_mask_layer(self, clip_style, alpha: float, transform: Affine, clip):
        self._push_layer_inner(LUMINANCE_MASK_BLEND_MODE, _f32(min(max(alpha, 0.0), 1.0)), clip_style, transform, clip)

    def push_clip_layer(self, clip_style, transform: Affine, clip):
        self._push_layer_inner(CLIP_BLEND_MODE, 1.0, clip_style, transform, clip)

    def pop_layer(self):
        self.encoding.encode_end_clip()

    def append(self, other: "Scene", transform: Optional[Affine] = None):
        """`Scene::append` (vello/src/scene.rs:464-469)."""
        self.encoding.append(other.encoding, transform)

    def draw_image(self, image: Image, transform: Affine):
        self.fill(FILL_NON_ZERO, transform, image, None, _shapes.Rect(0.0, 0.0, float(image.width), float(image.height)))

    def draw_blurred_rounded_rect(self, transform: Affine, rect: "_shapes.Rect", color: Color, radius: float, std_dev: float):
        """scene.rs:256-270: the blurred rectangle drawn in the rectangle inflated by 2.5 sigma."""
        k = 2.5 * std_dev
        shape = _shapes.Rect(rect.x0 - k, rect.y0 - k, rect.x1 + k, rect.y1 + k)
        self.draw_blurred_rounded_rect_in(shape, transform, rect, color, radius, std_dev)

    def draw_blurred_rounded_rect_in(self, shape, transform: Affine, rect: "_shapes.Rect", color: Color, radius: float, std_dev: float):
        """scene.rs:282-314: the blurred rounded rectangle clipped to `shape`."""
        e = self.encoding
        e.encode_transform(transform)
        e.encode_fill_style(FILL_NON_ZERO)
        if e.encode_shape(shape, True):
            cx, cy = 0.5 * (rect.x0 + rect.x1), 0.5 * (rect.y0 + rect.y1)
            if e.encode_transform(transform * Affine.translate(cx, cy)):
                e.swap_last_path_tags()
            e.encode_blurred_rounded_rect(color, rect.x1 - rect.x0, rect.y1 - rect.y0, radius, std_dev)


def batch(scenes: Sequence[Scene]) -> Tuple[Scene, List[int]]:
    """A batch for `Renderer.set_cells` / `render_batch` (the native `vb_scene_batch`): one scene holding every scene appended
    with the identity transform, each followed by the END_CLIP / PATH tags that close its open layers (what resolve would add
    at the end of that scene alone), and the draw-object offsets of the scenes (len(scenes) + 1 entries)."""
    out = Scene()
    e = out.encoding
    offsets = [0]
    for s in scenes:
        e.append(s.encoding)
        while e.n_open_clips > 0:
            e.encode_end_clip()
        offsets.append(e.n_paths)  # after resolve every draw object is a path
    return out, offsets


# ---------------------------------------------------------------------------------------------
# Ramps (ramp_cache.rs:119-155) and image atlas (shelf packer; atlas placement is ours, the
# reference uses guillotiere -- only the (x, y) written into draw data matters to the pipeline)
# ---------------------------------------------------------------------------------------------
N_RAMP_SAMPLES = 512
ATLAS_MAX_COORD = 65535  # the largest atlas x, y, width and height the draw data's 16-bit fields hold


def make_ramp(stops: Sequence[Tuple[float, Color]], premul_interp: bool) -> np.ndarray:
    f = np.float32
    out = np.zeros(N_RAMP_SAMPLES, dtype=np.uint32)
    last_u = f(0.0)
    last_c = stops[0][1]
    this_u = last_u
    this_c = last_c
    j = 0

    def comps(c: Color):
        return np.array([c.r, c.g, c.b, c.a], dtype=np.float32)

    for i in range(N_RAMP_SAMPLES):
        u = f(i) / f(N_RAMP_SAMPLES - 1)
        while u > this_u:
            last_u, last_c = this_u, this_c
            if j + 1 < len(stops):
                this_u = f(stops[j + 1][0])
                this_c = stops[j + 1][1]
                j += 1
            else:
                break
        du = this_u - last_u
        if du < f(1e-9):
            c = comps(this_c)
        else:
            t = (u - last_u) / du
            a, b = comps(last_c), comps(this_c)
            if premul_interp:
                # AlphaColor::lerp: premultiply, lerp_rect, un-premultiply (color crate)
                pa = np.array([a[0] * a[3], a[1] * a[3], a[2] * a[3], a[3]], dtype=np.float32)
                pb = np.array([b[0] * b[3], b[1] * b[3], b[2] * b[3], b[3]], dtype=np.float32)
                pc = pa + (pb - pa) * t
                if pc[3] == 0.0 or pc[3] == 1.0:
                    c = pc
                else:
                    inv = f(1.0) / pc[3]
                    c = np.array([pc[0] * inv, pc[1] * inv, pc[2] * inv, pc[3]], dtype=np.float32)
            else:
                c = a + (b - a) * t
        out[i] = Color(float(c[0]), float(c[1]), float(c[2]), float(c[3])).premul_rgba8_u32()
    return out


@dataclass
class Packed:
    """What crosses the drop-in boundary: packed scene bytes + Layout + ramps + atlas."""

    scene: np.ndarray  # uint32 words
    layout: Layout
    ramps: np.ndarray  # (n_ramps, 512) uint32, premultiplied RGBA8
    atlas: np.ndarray  # (h, w, 4) uint8

    def nbytes(self) -> int:
        return int(self.scene.nbytes)


def viewed(packed: Packed, view: Affine) -> Packed:
    """The packed scene of `Scene().append(scene, view)`, made by mapping `packed`'s transform words: every transform T
    becomes view * T in f32 with `Encoding.append`'s arithmetic (the product the renderer's `set_view` computes on the
    device). Nothing else of a packed scene depends on the transforms."""
    lay = packed.layout
    scene = np.array(packed.scene, dtype=np.uint32)
    t = scene[lay.transform_base:lay.style_base].view(np.float32).reshape(-1, 6)
    a = [np.float32(v) for v in view.coeffs]
    b = [t[:, k].copy() for k in range(6)]
    with np.errstate(over="ignore", invalid="ignore"):  # f32 overflow is part of the arithmetic, as on the device
        t[:, 0] = a[0] * b[0] + a[2] * b[1]
        t[:, 1] = a[1] * b[0] + a[3] * b[1]
        t[:, 2] = a[0] * b[2] + a[2] * b[3]
        t[:, 3] = a[1] * b[2] + a[3] * b[3]
        t[:, 4] = a[0] * b[4] + a[2] * b[5] + a[4]
        t[:, 5] = a[1] * b[4] + a[3] * b[5] + a[5]
    return Packed(scene, lay, packed.ramps, packed.atlas)


def _align_up(n: int, a: int) -> int:
    return (n + a - 1) // a * a


def resolve(enc: Encoding) -> Packed:
    """`Resolver::resolve` without glyph runs (resolve.rs:107-154,183-399)."""
    # late-bound: ramps
    draw_data = list(enc.draw_data)
    ramp_rows: List[np.ndarray] = []
    ramp_keys = {}
    for p in enc.ramp_patches:
        key = (tuple((o, c) for o, c in p["stops"]), p["premul"])
        if key not in ramp_keys:
            ramp_keys[key] = len(ramp_rows)
            ramp_rows.append(make_ramp(p["stops"], p["premul"]))
        rid = ramp_keys[key]
        draw_data[p["draw_data_offset"]] = ((rid << 2) | p["extend"]) & 0xFFFFFFFF
    # late-bound: images -> simple shelf atlas (VbShelfPacker, vb_resolve.h); the draw data holds a place and a size as
    # 16-bit fields, so an image with a side over ATLAS_MAX_COORD, or a place below row ATLAS_MAX_COORD, is refused
    atlas_w = 1
    shelves: List[Tuple[int, int, Image]] = []
    x = y = shelf_h = 0
    MAXW = 2048
    placed = {}
    for p in enc.image_patches:
        im = p["image"]
        # the image cache is keyed by the pixel blob's identity (image_cache.rs:113-114), not by the brush
        k = ("key", im.key) if im.key is not None else ("id", id(im.data))
        if k not in placed:
            if im.width > ATLAS_MAX_COORD or im.height > ATLAS_MAX_COORD:
                raise ValueError(f"resolve: a {im.width}x{im.height} image has a side over {ATLAS_MAX_COORD} texels")
            if x + im.width > MAXW:
                if y + shelf_h > ATLAS_MAX_COORD:
                    raise ValueError(f"resolve: the atlas would place an image at row {y + shelf_h}, past {ATLAS_MAX_COORD}")
                y += shelf_h
                x = 0
                shelf_h = 0
            placed[k] = (x, y)
            shelves.append((x, y, im))
            x += im.width
            shelf_h = max(shelf_h, im.height)
            atlas_w = max(atlas_w, x)
        px, py = placed[k]
        draw_data[p["draw_data_offset"]] = ((px << 16) | py) & 0xFFFFFFFF
    atlas_h = max(1, y + shelf_h)
    atlas = np.zeros((atlas_h, atlas_w, 4), dtype=np.uint8)
    for (px, py, im) in shelves:
        atlas[py : py + im.height, px : px + im.width] = im.data

    layout = Layout(n_paths=enc.n_paths, n_clips=enc.n_clips)
    n_tags = len(enc.path_tags) + enc.n_open_clips
    padded = _align_up(n_tags, 4 * PATH_REDUCE_WG)
    tags = np.zeros(padded, dtype=np.uint8)
    tags[: len(enc.path_tags)] = np.asarray(enc.path_tags, dtype=np.uint8) if enc.path_tags else []
    tags[len(enc.path_tags) : n_tags] = TAG_PATH
    chunks = [tags.view(np.uint32)]
    off = padded // 4
    layout.path_tag_base = 0
    layout.path_data_base = off
    pd = _path_data_array(enc.path_data)
    chunks.append(pd.view(np.uint32))
    off += pd.size
    layout.draw_tag_base = off
    dtags = list(enc.draw_tags) + [DRAWTAG_END_CLIP] * enc.n_open_clips
    layout.bin_data_start = sum(drawtag_info_size(t) for t in enc.draw_tags)
    chunks.append(np.asarray(dtags, dtype=np.uint32))
    off += len(dtags)
    layout.draw_data_base = off
    chunks.append(np.asarray(draw_data, dtype=np.uint32))
    off += len(draw_data)
    layout.transform_base = off
    tr = np.asarray(enc.transforms, dtype=np.float32).reshape(-1)
    chunks.append(tr.view(np.uint32))
    off += tr.size
    layout.style_base = off
    st = np.zeros(2 * len(enc.styles), dtype=np.uint32)
    for i, (fl, lw) in enumerate(enc.styles):
        st[2 * i] = fl
        st[2 * i + 1] = _f32_bits(lw)
    chunks.append(st)
    layout.n_draw_objects = layout.n_paths
    scene = np.concatenate([c.astype(np.uint32, copy=False).reshape(-1) for c in chunks]) if chunks else np.zeros(0, np.uint32)
    ramps = np.stack(ramp_rows) if ramp_rows else np.zeros((0, N_RAMP_SAMPLES), dtype=np.uint32)
    return Packed(scene=np.ascontiguousarray(scene), layout=layout, ramps=ramps, atlas=atlas)


def _path_data_array(path_data) -> np.ndarray:
    return np.asarray(path_data, dtype=np.float32).reshape(-1)
