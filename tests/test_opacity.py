"""Bound opacity without a GPU (Renderer.bind_draw_opacity): the Python row checks, with a stub `__cuda_array_interface__` and
a stub library; a float32 restatement of the words bound opacity writes into the frame's draw data (k_draw_data), tied to
both scene front ends at every rounding edge of the image alpha byte; and the re-encoded scene the GPU tests
(test_gpu_opacity.py) compare with. The compiled kernel is checked in test_compiled_kernels.py and test_draw_colors.py."""
import numpy as np
import pytest

from vello_b200.encoding import (ALPHA_PREMULTIPLIED, ALPHA_STRAIGHT, CLIP_BLEND_MODE, COMPOSE_COPY, COMPOSE_PLUS, COMPOSE_SRC_IN,
                                 COMPOSE_SRC_OVER, COMPOSE_XOR, DRAWTAG_BEGIN_CLIP, DRAWTAG_IMAGE, EXTEND_PAD, EXTEND_REFLECT,
                                 EXTEND_REPEAT, FILL_EVEN_ODD, FILL_NON_ZERO, FORMAT_BGRA8, FORMAT_RGBA8, MIX_COLOR_BURN,
                                 MIX_DIFFERENCE, MIX_HUE, MIX_MULTIPLY, MIX_NORMAL, MIX_SCREEN, QUALITY_HIGH, QUALITY_LOW,
                                 QUALITY_MEDIUM, Color, Gradient, Image, Packed, Scene, Stroke, resolve)
from vello_b200.shapes import Affine, Circle, Rect, RoundedRect

from .test_visibility import _Cai, _NoLib

f32 = np.float32
NORMAL_SRC_OVER = (MIX_NORMAL << 8) | COMPOSE_SRC_OVER


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def clamp01(a):
    """A finite row clamped to [0, 1] as both encoders' push_layer clamp it: -0.0 stays -0.0."""
    a = f32(a)
    return f32(0.0) if a < 0 else (f32(1.0) if a > 1 else a)


def image_byte(a):
    """The encoders' alpha byte of an image alpha a in [0, 1] (brush alpha 1): int(f32(a) * 255 + 0.5), each step rounded."""
    return int(f32(f32(a) * f32(255.0)) + f32(0.5))


def opacity_slots(packed):
    """Per draw object, where bound opacity writes (k_draw_data_slots): (word, kind) with the word relative to the draw data
    that its row replaces, kind "layer", "clip" or "image", or None for a draw object whose row is ignored."""
    L = packed.layout
    scene = np.asarray(packed.scene, dtype=np.uint32)
    tags = scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects]
    dd = scene[L.draw_data_base:L.transform_base]
    out, off = [], 0
    for t in tags.tolist():
        if t == DRAWTAG_BEGIN_CLIP:
            out.append((off + 1, "clip" if int(dd[off]) == CLIP_BLEND_MODE else "layer"))
        elif t == DRAWTAG_IMAGE:
            out.append((off + 2, "image"))
        else:
            out.append(None)
        off += (t >> 2) & 7
    return out


def patched_draw_data(packed, rows):
    """The draw data a frame with bound opacity rows reads: the scene's, with each bound word whose row is finite converted."""
    L = packed.layout
    dd = np.array(packed.scene[L.draw_data_base:L.transform_base], dtype=np.uint32)
    rows = np.asarray(rows, dtype=np.float32).reshape(-1)
    for k, slot in enumerate(opacity_slots(packed)[:len(rows)]):
        if slot is None or not np.isfinite(rows[k]):
            continue
        w, kind = slot
        a = clamp01(rows[k])
        if kind == "image":
            dd[w] = (int(dd[w]) & ~0xFF) | image_byte(a)
        elif kind == "layer" or a < 1:
            dd[w] = int(np.array([a], dtype=np.float32).view(np.uint32)[0])
            if kind == "clip":
                dd[w - 1] = NORMAL_SRC_OVER
    return dd


def patched(packed, rows):
    """The host route as packed words: the scene with its draw data patched as a bound frame patches it."""
    L = packed.layout
    scene = np.array(packed.scene, dtype=np.uint32)
    scene[L.draw_data_base:L.transform_base] = patched_draw_data(packed, rows)
    return Packed(scene, L, packed.ramps, packed.atlas)


# ---- scenes whose layers and images take their alpha from rows ---------------------------------------------------------------
def _img(seed, h, w, premul):
    px = np.random.default_rng(seed).integers(0, 256, (h, w, 4), dtype=np.uint8)
    if premul:
        px[..., :3] = (px[..., :3].astype(np.uint32) * px[..., 3:] // 255).astype(np.uint8)
    return px


IMAGES = [dict(data=_img(71, 14, 18, False), format=FORMAT_RGBA8, alpha_type=ALPHA_STRAIGHT, quality=QUALITY_MEDIUM),
          dict(data=_img(72, 12, 16, True), format=FORMAT_BGRA8, alpha_type=ALPHA_PREMULTIPLIED, quality=QUALITY_LOW,
               x_extend=EXTEND_REPEAT, y_extend=EXTEND_REFLECT),
          dict(data=_img(73, 10, 13, True), format=FORMAT_RGBA8, alpha_type=ALPHA_PREMULTIPLIED, quality=QUALITY_HIGH),
          dict(data=_img(74, 16, 11, False), format=FORMAT_BGRA8, alpha_type=ALPHA_STRAIGHT, quality=QUALITY_HIGH,
               x_extend=EXTEND_REFLECT, y_extend=EXTEND_PAD)]
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (0.6, Color(0.2, 0.9, 0.3, 0.8)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]


def opacity_ops(seed=0, dx=0.0, full_clip=False):
    """A scene as a list of (kind, encoded alpha, call): call(s, alpha) encodes exactly one draw object, a layer or an image
    with that alpha. kind is "layer", "clip" (push_clip_layer, encoded alpha 1), "image", "pop" or "draw" (a draw whose row
    is ignored: solid fills and strokes, gradients, blurred rectangles). Blend layers of several mix and compose modes, a
    luminance mask, clip layers, layers nested deeper than the blend stack's split (4), and images of both formats and alpha
    types, three qualities and every extend. With `full_clip` the scene opens with a clip layer covering the whole frame."""
    g = np.random.default_rng(seed)
    ops = []

    def col(a=None):
        c = g.uniform(0.05, 1.0, 4)
        c[3] = g.choice([1.0, 0.8, 0.5]) if a is None else a
        return Color(*map(float, c))

    def draw(f):
        ops.append(("draw", None, lambda s, a, f=f: f(s)))

    def layer(mix, compose, alpha, clip, style=FILL_NON_ZERO, xf=Affine.IDENTITY):
        ops.append(("layer", alpha, lambda s, a: s.push_layer(style, mix, compose, a, xf, clip)))

    def lum(alpha, clip):
        ops.append(("layer", alpha, lambda s, a: s.push_luminance_mask_layer(FILL_NON_ZERO, a, Affine.IDENTITY, clip)))

    def clip_layer(clip, style=FILL_NON_ZERO, xf=Affine.IDENTITY):
        ops.append(("clip", 1.0, lambda s, a: s.push_clip_layer(style, xf, clip) if a >= 1 else
                    s.push_layer(style, MIX_NORMAL, COMPOSE_SRC_OVER, a, xf, clip)))

    def image(i, alpha, xf):
        ops.append(("image", alpha, lambda s, a: s.draw_image(Image(**IMAGES[i], alpha=float(a)), xf)))

    def pop():
        ops.append(("pop", None, lambda s, a: s.pop_layer()))

    if full_clip:
        clip_layer(Rect(-50, -50, 1000, 1000))
    for i in range(5):
        c = col()
        draw(lambda s, i=i, c=c: s.fill(FILL_NON_ZERO, Affine.translate(dx + 10 + 70 * i, 10 + 11 * i), c, None, Rect(0, 0, 60, 45)))
    c = col()
    draw(lambda s: s.stroke(Stroke(6.0), Affine.IDENTITY, c, None, Circle(dx + 110, 110, 55)))
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((dx, 0), (dx + 150, 0), STOPS), None, Rect(dx + 5, 170, 160, 230)))
    c = col()
    draw(lambda s: s.draw_blurred_rounded_rect(Affine.translate(dx + 230, 40), Rect(0, 0, 80, 50), c, 9.0, 6.0))
    image(0, 1.0, Affine.translate(dx + 180, 150) * Affine.scale(3.0))
    image(1, 0.8, Affine.translate(dx + 20, 240) * Affine.rotate(0.2) * Affine.scale(2.5))
    # a multiply layer holding an image, a nested clip and a luminance mask
    layer(MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.9, Circle(dx + 200, 160, 95))
    c = col()
    draw(lambda s: s.fill(FILL_EVEN_ODD, Affine.IDENTITY, c, None, RoundedRect(dx + 110, 80, 300, 250, 16)))
    image(2, 0.6, Affine.translate(dx + 210, 90) * Affine.scale(4.0))
    clip_layer(Rect(dx + 130, 100, 270, 230), xf=Affine.rotate(0.08))
    c = col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Circle(dx + 200, 165, 62)))
    lum(1.0, Rect(dx + 140, 120, 260, 220))
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((dx + 140, 0), (dx + 260, 0), STOPS), None, Rect(dx + 140, 120, 260, 220)))
    pop()
    pop()
    pop()
    # nested deeper than the blend stack's split: screen > xor > clip > difference > clip > plus > hue, each with a draw
    nest = [("layer", MIX_SCREEN, COMPOSE_SRC_OVER, 1.0), ("layer", MIX_NORMAL, COMPOSE_XOR, 0.85), ("clip",),
            ("layer", MIX_DIFFERENCE, COMPOSE_SRC_OVER, 0.7), ("clip",), ("layer", MIX_NORMAL, COMPOSE_PLUS, 0.95),
            ("layer", MIX_HUE, COMPOSE_SRC_OVER, 1.0)]
    for d, spec in enumerate(nest):
        clip = RoundedRect(dx + 200 + 6 * d, 170 + 5 * d, dx + 380 - 5 * d, 315 - 4 * d, 10)
        if spec[0] == "clip":
            clip_layer(clip)
        else:
            layer(spec[1], spec[2], spec[3], clip)
        c = col(0.85)
        draw(lambda s, d=d, c=c: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Circle(dx + 260 + 12 * d, 220 + 8 * d, 45 - 3 * d)))
    image(3, 0.9, Affine.translate(dx + 300, 250) * Affine.scale(3.0))
    for _ in nest:
        pop()
    # a destructive compose and a colour-burn layer with a stroked clip
    layer(MIX_NORMAL, COMPOSE_COPY, 0.75, Circle(dx + 330, 80, 40))
    c = col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Rect(dx + 300, 50, 370, 110)))
    pop()
    ops.append(("layer", 0.65, lambda s, a: s.push_layer(Stroke(14.0), MIX_COLOR_BURN, COMPOSE_SRC_IN, a, Affine.IDENTITY,
                                                         Circle(dx + 60, 120, 40))))
    c = col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Rect(dx + 10, 70, 110, 170)))
    pop()
    if full_clip:
        pop()
    return ops


def alphas_of(ops, rows):
    """The alpha each call of `ops` encodes with under rows: the clamped row for a layer, clip layer or image whose row is
    finite, else its encoded alpha (None for other draws and pops)."""
    rows = np.asarray(rows, dtype=np.float32).reshape(-1)
    out = []
    for k, (kind, enc, _) in enumerate(ops):
        if kind in ("layer", "clip", "image") and k < len(rows) and np.isfinite(rows[k]):
            out.append(clamp01(rows[k]))
        else:
            out.append(None if enc is None else f32(enc))
    return out


def build(ops, rows=(), s=None):
    """The scene of `ops` re-encoded with `rows` applied (nothing bound: rows=()); every call encodes one draw object."""
    s = Scene() if s is None else s
    for k, ((_, _, f), a) in enumerate(zip(ops, alphas_of(ops, rows))):
        n0 = s.n_draw_objects
        f(s, a)
        assert s.n_draw_objects == n0 + 1, k
    return s


def rand_rows(n, seed, lo=-0.2, hi=1.2):
    """Rows across [0, 1], with some below 0 and above 1 (clamped), and some exactly 0, 1 and NaN."""
    g = np.random.default_rng(seed)
    rows = g.uniform(lo, hi, n).astype(np.float32)
    pick = g.uniform(size=n)
    rows[pick < 0.1] = 1.0
    rows[(pick >= 0.1) & (pick < 0.15)] = 0.0
    rows[(pick >= 0.15) & (pick < 0.2)] = np.nan
    return rows


def front_ends():
    from vello_b200.scene_native import NativeScene
    return [("python", Scene, lambda s: resolve(s.encoding)), ("native", NativeScene, lambda s: s.resolve())]


# ---- the restatement against both encoders -----------------------------------------------------------------------------------
def edge_rows():
    """The float32 neighbours (up to 2 ulp either side) of every image-byte tie (k + 0.5) / 255, then 0, -0.0, tiny and
    denormal values, 1 and its neighbours, values above 1 and below 0."""
    ties = []
    for k in range(256):
        t = f32((k + 0.5) / 255)
        for d in (-2, -1, 0, 1, 2):
            x = t
            for _ in range(abs(d)):
                x = np.nextafter(x, f32(np.inf) if d > 0 else f32(-np.inf), dtype=np.float32)
            ties.append(x)
    odd = [0.0, -0.0, 1e-30, 1.4e-45, 1e-38, 1.0, 0.99999994, 1.0000001, 2.0, 3e38, -0.5, -1e-30, -3e38, 0.5]
    return np.concatenate([np.array(ties, dtype=np.float32), np.array(odd, dtype=np.float32)])


def test_edge_rows_straddle_the_ties():
    """The rows do sit on both sides of the byte boundaries, so that a contracted multiply-add would show."""
    rows = edge_rows()
    b = np.array([image_byte(clamp01(x)) for x in rows[:1280]]).reshape(256, 5)
    assert len(np.unique(b)) == 256 and (b[:, 0] != b[:, 4]).sum() > 200


@pytest.mark.parametrize("front", front_ends(), ids=lambda f: f[0])
def test_restatement_is_both_encoders_conversion(front):
    """Per row: a blend layer, a luminance mask, a clip layer and an image re-encoded with the row give the words the
    restatement writes over the encoded scene (layer alpha word, clip blend word, image sample byte)."""
    _, make, packed_of = front
    rows = edge_rows()
    enc = make()
    for _ in rows:
        enc.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 0.3, Affine.IDENTITY, Rect(0, 0, 4, 4))
        enc.pop_layer()
        enc.push_luminance_mask_layer(FILL_NON_ZERO, 0.6, Affine.IDENTITY, Rect(0, 0, 4, 4))
        enc.pop_layer()
        enc.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Rect(0, 0, 4, 4))
        enc.pop_layer()
        enc.draw_image(Image(**IMAGES[1], alpha=0.25), Affine.IDENTITY)
    base = packed_of(enc)
    want = make()
    bound = np.full(base.layout.n_draw_objects, np.nan, dtype=np.float32)
    for i, x in enumerate(rows):
        a = clamp01(x)
        want.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, float(x), Affine.IDENTITY, Rect(0, 0, 4, 4))  # the encoder clamps
        want.pop_layer()
        want.push_luminance_mask_layer(FILL_NON_ZERO, float(x), Affine.IDENTITY, Rect(0, 0, 4, 4))
        want.pop_layer()
        if a < 1:
            want.push_layer(FILL_NON_ZERO, MIX_NORMAL, COMPOSE_SRC_OVER, float(x), Affine.IDENTITY, Rect(0, 0, 4, 4))
        else:
            want.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Rect(0, 0, 4, 4))
        want.pop_layer()
        want.draw_image(Image(**IMAGES[1], alpha=float(a)), Affine.IDENTITY)  # Image.alpha is not clamped by the encoders
        bound[7 * i:7 * i + 7] = x  # rows of END_CLIPs are ignored
    packed = packed_of(want)
    L = packed.layout
    got = patched_draw_data(base, bound)
    assert np.array_equal(got, np.asarray(packed.scene[L.draw_data_base:L.transform_base], dtype=np.uint32))
    # the bytes themselves: every value 0 .. 255 and both sides of each tie
    slots = opacity_slots(base)
    img = [w for (w, kind) in (s for s in slots if s) if kind == "image"]
    assert len(img) == len(rows)
    assert sorted(set(int(got[w]) & 0xFF for w in img)) == list(range(256))
    # NaN and infinite rows keep the encoded words
    for bad in (np.nan, np.inf, -np.inf):
        assert np.array_equal(patched_draw_data(base, np.full(L.n_draw_objects, bad, np.float32)),
                              np.asarray(base.scene[base.layout.draw_data_base:base.layout.transform_base], dtype=np.uint32))


@pytest.mark.parametrize("front", front_ends(), ids=lambda f: f[0])
def test_patched_scene_is_the_reencoded_scene(front):
    """The host route of the GPU tests: the packed scene with the rows patched in is, word for word, the scene re-encoded with
    the rows' alphas, in both front ends, for random, partial, NaN and clip-converting rows."""
    _, make, packed_of = front
    ops = opacity_ops(seed=3, full_clip=True)
    packed = packed_of(build(ops, s=make()))
    n = packed.layout.n_draw_objects
    kinds = [s[1] if s else None for s in opacity_slots(packed)]
    assert kinds.count("clip") == 4 and kinds.count("image") == 4 and kinds.count("layer") == 9
    for seed, rows in enumerate([rand_rows(n, 1), rand_rows(n, 2)[:n // 2], np.full(n, 0.5, np.float32), np.ones(n, np.float32)]):
        want = packed_of(build(ops, rows, s=make()))
        got = patched(packed, rows)
        assert np.array_equal(np.asarray(got.scene, dtype=np.uint32), np.asarray(want.scene, dtype=np.uint32)), seed
    # a clip layer's row of 1 (or more) leaves it exactly as encoded
    rows = np.array([2.0 if k == "clip" else np.nan for k in kinds], dtype=np.float32)
    assert np.array_equal(patched(packed, rows).scene, np.asarray(packed.scene, dtype=np.uint32))


def test_rows_of_other_draws_are_ignored():
    ops = opacity_ops(seed=4)
    packed = resolve(build(ops).encoding)
    slots = opacity_slots(packed)
    rows = np.array([np.nan if s else 0.25 for s in slots], dtype=np.float32)
    assert np.array_equal(patched(packed, rows).scene, np.asarray(packed.scene, dtype=np.uint32))
    assert all(s is None for s, (kind, _, _) in zip(slots, ops) if kind in ("draw", "pop"))


# ---- the Python row checks ---------------------------------------------------------------------------------------------------
def _renderer(lib=None):
    from vello_b200.renderer import Renderer
    return Renderer._borrowed(lib or _NoLib(), 1, owner=object())


@pytest.mark.parametrize("t, err", [
    (np.ones(4, np.float32), TypeError),              # host memory: no __cuda_array_interface__
    (_Cai((5, 2), "<f4"), ValueError),                # two columns
    (_Cai((), "<f4"), ValueError),                    # a scalar
    (_Cai((0,), "<f4"), ValueError),                  # no rows
    (_Cai((0, 1), "<f4"), ValueError),
    (_Cai((5,), "<f8"), ValueError),                  # float64
    (_Cai((5,), "<f2"), ValueError),                  # float16
    (_Cai((5,), "|u1"), ValueError),                  # uint8
    (_Cai((5,), "<f4", strides=(0,)), ValueError),    # every row the same float
    (_Cai((5,), "<f4", strides=(-4,)), ValueError),   # reversed
    (_Cai((5,), "<f4", strides=(6,)), ValueError),    # not a multiple of 4 bytes
    (_Cai((5, 1), "<f4", strides=(8, 2)), ValueError),
])
def test_python_checks_refuse_before_the_library(t, err):
    with pytest.raises(err):
        _renderer().bind_draw_opacity(t)


def test_python_messages():
    r = _renderer()
    with pytest.raises(TypeError) as e:
        r.bind_draw_opacity(np.ones(2, np.float32))
    assert str(e.value) == "ndarray has no __cuda_array_interface__: device alphas are needed"
    with pytest.raises(ValueError) as e:
        r.bind_draw_opacity(_Cai((2, 3), "<f4"))
    assert str(e.value) == "bind_draw_opacity: alphas must be (n,) or (n, 1) float32, not (2, 3) <f4"
    with pytest.raises(ValueError) as e:
        r.bind_draw_opacity(_Cai((4,), "<f4", strides=(6,)))
    assert str(e.value) == "bind_draw_opacity: columns 4 bytes apart and rows a multiple of 4 bytes, at least 4, apart; not strides (6, 4)"


def test_python_accepts_vectors_columns_and_strided_rows():
    """A float32 vector, an (n, 1) array, or a column of a wider float32 state tensor reaches the library with its row pitch."""
    got = []

    class Lib:
        def vb_bind_draw_opacity(self, handle, ptr, n, pitch):
            got.append((None if ptr is None else ptr.value, n, pitch))
            return 0

    r = _renderer(Lib())
    t = _Cai((7,), "<f4", strides=(40,))  # state[:, 5] of a (7, 10) float32 tensor
    r.bind_draw_opacity(t)
    assert got == [(1 << 20, 7, 40)] and r._opacity is t
    r.bind_draw_opacity(_Cai((9,), "<f4"))
    assert got[-1] == (1 << 20, 9, 4)
    r.bind_draw_opacity(_Cai((9, 1), "<f4"))
    assert got[-1] == (1 << 20, 9, 4)
    r.bind_draw_opacity(_Cai((6, 1), "<f4", strides=(24, 4)))
    assert got[-1] == (1 << 20, 6, 24)
    r.bind_draw_opacity(None)
    assert got[-1] == (None, 0, 0) and r._opacity is None
