"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle and the golden
vectors. Run on an H100 with `pytest -m gpu`.

Bar: bit-exact for every integer / index buffer and for MSAA pixels (integer sample counts). Area-AA pixels are
compared twice: byte for byte with the oracle's `fine` replayed on the GPU's own command lists and segments
(`parity.replay_fine`), and within +-1 LSB per 8-bit channel of the oracle's full pipeline, on a bounded number of channel
values. The +-1 remains only because segment order inside a tile's slice comes from path_tiling's atomics, so the float
sums run in a different order; `compare_all` pins those slices as multisets.
"""
import os

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, Color, EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT, Scene, TRANSPARENT, WHITE, resolve

from . import parity

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def gold(name):
    return np.load(os.path.join(G, f"smoke_{name}.npy"))


def render_both(renderer, oracle, scene, w, h, aa=AA_AREA, base=BLACK):
    packed = resolve(scene.encoding) if isinstance(scene, Scene) else scene
    img = renderer.render_to_texture(packed, RenderParams(base, w, h, aa))
    ref = oracle.render(packed, w, h, base.premul_rgba8_u32(), aa)
    return packed, img, ref


# area AA against the oracle's full pipeline: at most this share of channel values (and never fewer than
# AREA_OFF_BY_ONE_MIN) may differ, by 1. A defect that moves every edge pixel by one LSB moves far more.
AREA_OFF_BY_ONE_SHARE = 1e-4
AREA_OFF_BY_ONE_MIN = 16


def assert_pixels(img, ref, aa):
    d = np.abs(img.astype(np.int32) - ref.astype(np.int32))
    tol = 1 if aa == AA_AREA else 0
    assert d.max() <= tol, f"aa={aa}: max diff {d.max()}, {int((d > tol).sum())} channel values out of tolerance"
    off = int((d > 0).sum())
    bound = max(AREA_OFF_BY_ONE_MIN, int(d.size * AREA_OFF_BY_ONE_SHARE))
    assert off <= bound, f"aa={aa}: {off} channel values differ by 1 (bound {bound} of {d.size})"
    return off


# ---- golden vectors of the reference, through the CUDA path ------------------------------------
def test_golden_filled_square_circle(renderer):
    for name, fn in (("filled_square", scenes.filled_square), ("filled_circle", scenes.filled_circle)):
        s, w, h = fn()
        img = renderer.render_to_texture(s, RenderParams(BLACK, w, h, AA_AREA))
        assert np.array_equal(img[..., :3], gold(name)[..., :3]), name


@pytest.mark.parametrize("premul", [True, False])
def test_golden_gradients(renderer, premul):
    s, w, h = scenes.gradient_color_alpha(premul)
    name = "gradient_color_alpha_premultiplied" if premul else "gradient_color_alpha_unpremultiplied"
    img = renderer.render_to_texture(s, RenderParams(WHITE, w, h, AA_AREA))
    assert np.array_equal(img[..., :3], gold(name)[..., :3])


@pytest.mark.parametrize("extend", [EXTEND_PAD, EXTEND_REFLECT, EXTEND_REPEAT])
def test_golden_image_roundtrip(renderer, extend):
    im = gold("data_image_roundtrip")
    s, w, h = scenes.image_roundtrip(im, extend)
    assert np.array_equal(renderer.render_to_texture(s, RenderParams(BLACK, w, h, AA_AREA)), im)


def test_property_simple_square_and_empty(renderer):
    s, w, h = scenes.simple_square()
    for aa in (AA_AREA, AA_MSAA8, AA_MSAA16):
        img = renderer.render_to_texture(s, RenderParams(BLACK, w, h, aa))
        red = (img == np.array([255, 0, 0, 255], dtype=np.uint8)).all(axis=2)
        black = (img == np.array([0, 0, 0, 255], dtype=np.uint8)).all(axis=2)
        assert red.sum() == 2500 and black.sum() == 150 * 150 - 2500
    plum = Color.from_rgba8(221, 160, 221)
    img = renderer.render_to_texture(Scene(), RenderParams(plum, 150, 150, AA_AREA))
    assert (img == np.array([221, 160, 221, 255], dtype=np.uint8)).all()


# ---- stage-by-stage + pixel parity with the oracle -------------------------------------------------
SCENES = ["filled_circle", "robust_paths", "funky_paths", "fill_types", "stroke_styles", "many_clips", "deep_blend", "brushes",
          # the reference's own scene recipes (examples/scenes/src/test_scenes.rs), restated in vello_b200/scenes.py
          "blend_grid", "compose_grid", "tricky_strokes", "gradient_extend", "two_point_radial", "conflation_artifacts", "longpathdash"]


@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_scene_parity(renderer, oracle, name, aa):
    s, w, h = getattr(scenes, name)()
    packed, img, ref = render_both(renderer, oracle, s, w, h, aa)
    parity.compare_all(renderer, oracle, packed.layout, w, h)
    parity.assert_replay(renderer, oracle, packed, img, w, h, aa, BLACK)
    assert_pixels(img, ref, aa)


@pytest.mark.parametrize("quality", [0, 1, 2])
def test_image_extend_modes(renderer, oracle, quality):
    """test_scenes.rs:2168-2213 at the three sampling qualities (nearest / bilinear / bicubic), white base colour."""
    s, w, h = scenes.image_extend_modes(quality)
    for aa in (AA_AREA, AA_MSAA16):
        packed, img, ref = render_both(renderer, oracle, s, w, h, aa, base=WHITE)
        assert_pixels(img, ref, aa)
        if aa == AA_AREA:  # the MSAA16 leg's buffers are compared below
            parity.assert_replay(renderer, oracle, packed, img, w, h, aa, WHITE)
    parity.compare_all(renderer, oracle, packed.layout, w, h)


def test_many_draw_objects(renderer, oracle):
    """test_scenes.rs:1928-1948: 90,000 draw objects = 352 partitions of the draw / binning / tile_alloc scans and a
    2000x1500 target (8x6 bins)."""
    s, w, h = scenes.many_draw_objects()
    for aa in (AA_MSAA16, AA_AREA):
        packed, img, ref = render_both(renderer, oracle, s, w, h, aa)
        assert_pixels(img, ref, aa)
    parity.compare_all(renderer, oracle, packed.layout, w, h, check_ptcl_tiles=range(0, ((w + 15) // 16) * ((h + 15) // 16), 7))


def test_large_bin_count(renderer, oracle):
    """vello_tests/tests/compare_gpu_cpu.rs:102-109 (`compare_large_bin_count`): 8192x2304 is 32x9 = 288 bins, more than
    one 256-wide binning workgroup covers."""
    w, h = 8192, 2304
    s = scenes.paris_like(3000, 4096, seed=17)
    s2 = Scene()
    from vello_b200.shapes import Affine
    s2.append(s, Affine.scale(2.0, 0.5625))
    packed, img, ref = render_both(renderer, oracle, s2, w, h, AA_MSAA16)
    assert_pixels(img, ref, AA_MSAA16)
    parity.compare_all(renderer, oracle, packed.layout, w, h, check_ptcl_tiles=range(0, (w // 16) * (h // 16), 37))


@pytest.mark.parametrize("size,aa", [(512, AA_AREA), (512, AA_MSAA16), ((1920, 1080), AA_AREA), ((1920, 1080), AA_MSAA16)])
def test_tiger_parity(renderer, oracle, size, aa):
    w, h = (size, size) if isinstance(size, int) else size
    packed, img, ref = render_both(renderer, oracle, scenes.tiger(w, h), w, h, aa)
    parity.compare_all(renderer, oracle, packed.layout, w, h)
    parity.assert_replay(renderer, oracle, packed, img, w, h, aa, BLACK)
    assert_pixels(img, ref, aa)


@pytest.mark.parametrize("seed", range(12))
def test_random_scene_parity(renderer, oracle, seed):
    s, w, h = scenes.random_small(seed)
    aa = (AA_AREA, AA_MSAA8, AA_MSAA16)[seed % 3]
    packed, img, ref = render_both(renderer, oracle, s, w, h, aa)
    parity.compare_all(renderer, oracle, packed.layout, w, h)
    parity.assert_replay(renderer, oracle, packed, img, w, h, aa, BLACK)
    assert_pixels(img, ref, aa)


def test_odd_sizes_and_transparent_base(renderer, oracle):
    s, _, _ = scenes.stroke_styles()
    for (w, h) in [(1, 1), (17, 33), (255, 257), (561, 479)]:
        for aa in (AA_AREA, AA_MSAA16):
            packed, img, ref = render_both(renderer, oracle, s, w, h, aa, base=TRANSPARENT)
            parity.assert_replay(renderer, oracle, packed, img, w, h, aa, TRANSPARENT)
            assert_pixels(img, ref, aa)


def test_paris_like_small(renderer, oracle):
    """A 2000-path cut of the paris-like generator at 1024^2: all stages + pixels."""
    s = scenes.paris_like(2000, 1024, seed=30000)
    for aa in (AA_MSAA16, AA_AREA):
        packed, img, ref = render_both(renderer, oracle, s, 1024, 1024, aa)
        parity.compare_all(renderer, oracle, packed.layout, 1024, 1024)
        parity.assert_replay(renderer, oracle, packed, img, 1024, 1024, aa, BLACK)
        assert_pixels(img, ref, aa)


def test_beziers_clips_small(renderer, oracle):
    s = scenes.beziers_clips(3000, 60, 1024, seed=100000)
    packed, img, ref = render_both(renderer, oracle, s, 1024, 1024, AA_MSAA16)
    parity.compare_all(renderer, oracle, packed.layout, 1024, 1024)
    assert_pixels(img, ref, AA_MSAA16)


def test_deep_clip_nesting(renderer, oracle):
    """Nesting deeper than the reference GPU path's 256 limit (clip_leaf.wgsl:102); the CPU shader and
    this implementation have no limit."""
    from vello_b200.encoding import FILL_NON_ZERO
    from vello_b200.shapes import Affine, Rect
    s = Scene()
    for i in range(300):
        s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Rect(i * 0.2, i * 0.1, 300 - i * 0.2, 300 - i * 0.1))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 100, 50), None, Rect(0, 0, 300, 300))
    for i in range(300):
        s.pop_layer()
    packed, img, ref = render_both(renderer, oracle, s, 300, 300, AA_MSAA16)
    parity.compare_all(renderer, oracle, packed.layout, 300, 300)
    assert_pixels(img, ref, AA_MSAA16)


def test_stripes_equal_full_frame(renderer):
    """Bin-row stripes (the multi-GPU partition) reproduce the full frame exactly."""
    w = h = 1024
    packed = resolve(scenes.paris_like(1500, 1024, seed=7).encoding)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    full = renderer.render_to_texture(packed, p)
    parts = [renderer.render_to_texture(packed, p, bin_rows=(b, b + 1)) for b in range(4)]
    assert np.array_equal(np.concatenate(parts, axis=0), full)
    parts = [renderer.render_to_texture(packed, p, bin_rows=br) for br in ((0, 3), (3, 4))]
    assert np.array_equal(np.concatenate(parts, axis=0), full)
    # curves, strokes with round / miter joins and caps, rotated transforms: flatten skips the segments that cannot
    # reach a stripe's rows (k_flatten.cu, win_cull), which must not move a pixel
    from vello_b200.shapes import Affine
    for scene, (sw, sh) in ((scenes.tiger(1024, 1024), (1024, 1024)), (scenes.stroke_styles(Affine.translate(180.0, -40.0) * Affine.rotate(0.31) * Affine.scale(1.7, 1.5))[0], (1024, 768))):
        pk = resolve(scene.encoding)
        for aa in (AA_MSAA16, AA_MSAA8):
            pp = RenderParams(BLACK, sw, sh, aa)
            whole = renderer.render_to_texture(pk, pp)
            rows = (sh + 255) // 256
            stripes = [renderer.render_to_texture(pk, pp, bin_rows=(b, b + 1)) for b in range(rows)]
            assert np.array_equal(np.concatenate(stripes, axis=0), whole)


def test_arena_growth_and_retry(oracle):
    """Tiny initial arenas: the frame overflows, the renderer grows and re-runs (the reference leaves
    this as a TODO, vello/src/lib.rs:762) and the result is still exact."""
    from vello_b200.renderer import Renderer
    r = Renderer()
    small, w, h = scenes.filled_square()
    r.render_to_texture(small, RenderParams(BLACK, w, h, AA_AREA))  # arenas sized for a tiny scene
    s = scenes.paris_like(3000, 1024, seed=3)
    packed = resolve(s.encoding)
    img = r.render_to_texture(packed, RenderParams(BLACK, 1024, 1024, AA_MSAA16))
    # the first attempt overflows `lines` (VB_STAGE_FLATTEN: 426,866 lines against a first guess sized from the tag count)
    assert r.last_stats.retries >= 1
    ref = oracle.render(packed, 1024, 1024, BLACK.premul_rgba8_u32(), AA_MSAA16)
    assert np.array_equal(img, ref)
    r.close()


def test_oracle_lines_into_gpu_tile_stages(renderer, oracle):
    """Feed the ORACLE's line soup to the CUDA tile stages (path_count .. fine): everything downstream
    of flatten is bit-exact given identical lines (SURVEY.md section 7 'flatten parity')."""
    s, w, h = scenes.stroke_styles()
    packed = resolve(s.encoding)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    ref = oracle.render(packed, w, h, BLACK.premul_rgba8_u32(), AA_MSAA16)
    renderer.upload(packed)
    renderer.run_stages(p, "pathtag", "flatten")
    renderer.upload_buffer("lines", oracle.buffer("lines"))
    renderer.run_stages(p, "draw", "fine")
    img = renderer.download_target(p)
    assert np.array_equal(img, ref)


def test_flatten_fill_line_fast_path_extremes(renderer, oracle):
    """k_flatten short-cuts line-to segments of fills (one line, no Euler machinery). The oracle has no such
    shortcut, so bit-identical `lines` on adversarial inputs -- tiny segments at large coordinates, skewed /
    scaled transforms, near-degenerate and huge lines, coordinates beyond the guard -- proves the equivalence."""
    from vello_b200.encoding import FILL_NON_ZERO, FILL_EVEN_ODD
    from vello_b200.shapes import Affine, BezPath
    from oracle.vbo import DTYPES
    rng = np.random.default_rng(123)
    s = Scene()
    for k in range(400):
        p = BezPath()
        mag = [1.0, 100.0, 4000.0, 60000.0, 3.0e5, 2.0e7][k % 6]
        step = [1e-4, 1e-3, 1e-2, 0.3, 5.0, 300.0, 5e4][k % 7]
        x, y = rng.uniform(-mag, mag, 2)
        p.move_to(x, y)
        for _ in range(int(rng.integers(2, 9))):
            x += rng.normal(0, step)
            y += rng.normal(0, step)
            p.line_to(x, y)
        p.close_path()
        if k % 5 == 0:
            t = Affine((rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 50), rng.normal(0, 50)))
        elif k % 5 == 1:
            t = Affine.scale(float(rng.uniform(1e-3, 50)))
        else:
            t = Affine.translate(*rng.uniform(-10, 10, 2))
        s.fill(FILL_NON_ZERO if k % 2 else FILL_EVEN_ODD, t, Color.from_rgba8(200, 50, 50, 128), None, p)
    packed = resolve(s.encoding)
    p = RenderParams(BLACK, 256, 256, AA_AREA)
    renderer.upload(packed)
    renderer.run_stages(p, "pathtag", "flatten")
    oracle.bind(packed, 256, 256)
    oracle.run("pathtag", "flatten")
    g, c = renderer.download("lines", DTYPES["lines"]), oracle.buffer("lines")
    assert g.shape == c.shape and g.tobytes() == c.tobytes()
    assert renderer.download("path_bboxes", DTYPES["path_bboxes"]).tobytes() == oracle.buffer("path_bboxes").tobytes()


def test_occlusion_cull_is_invisible(renderer, oracle):
    """fine's occlusion pre-scan (start at the last opaque full-tile cover) must not change a single pixel: opaque
    covers at depth 0, inside clip layers (must NOT be used), translucent covers, covers followed by more content,
    and a command list long enough to need PTCL chunk links between the covers."""
    from vello_b200.encoding import FILL_NON_ZERO
    from vello_b200.shapes import Affine, Rect, Circle
    rng = np.random.default_rng(5)
    s = Scene()
    w = h = 256
    full = Rect(-10, -10, 300, 300)

    def clutter(n):
        for _ in range(n):
            x, y = rng.uniform(0, 256, 2)
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(*[int(v) for v in rng.integers(0, 256, 3)], int(rng.choice([255, 255, 120]))),
                   None, Circle(float(x), float(y), float(rng.uniform(3, 40))))
    clutter(150)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(10, 200, 30, 255), None, full)          # opaque cover
    clutter(30)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 20, 30, 128), None, full)          # translucent cover
    s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Circle(128.0, 128.0, 100.0))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(0, 0, 250, 255), None, full)            # opaque, but clipped
    clutter(10)
    s.pop_layer()
    clutter(20)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(90, 90, 90, 255), None, Rect(0, 0, 128, 300))  # covers half the tiles
    clutter(15)
    packed = resolve(s.encoding)
    for aa in (AA_AREA, AA_MSAA8, AA_MSAA16):
        p = RenderParams(Color.from_rgba8(7, 7, 7, 255), w, h, aa)
        ref = oracle.render(packed, w, h, p.base_color.premul_rgba8_u32(), aa)
        renderer.set_occlusion_cull(False)
        off = renderer.render_to_texture(packed, p)
        renderer.set_occlusion_cull(True)
        on = renderer.render_to_texture(packed, p)
        assert np.array_equal(on, off)
        assert_pixels(on, ref, aa)
        parity.assert_replay(renderer, oracle, packed, on, w, h, aa, p.base_color)
    # and on the map-like workload, where most tiles have an opaque cover somewhere in their list
    packed = resolve(scenes.paris_like(3000, 1024, seed=11).encoding)
    p = RenderParams(BLACK, 1024, 1024, AA_MSAA16)
    renderer.set_occlusion_cull(False)
    off = renderer.render_to_texture(packed, p)
    renderer.set_occlusion_cull(True)
    assert np.array_equal(renderer.render_to_texture(packed, p), off)


def test_streaming_readback_matches_blocking(renderer):
    """vb_render_begin / vb_readback_wait (read-back of frame n overlapping frame n+1, alternating targets) deliver
    exactly the frames the blocking vb_render does, in order."""
    p = RenderParams(BLACK, 1024, 1024, AA_MSAA16)
    seq = [resolve(scenes.paris_like(400 + 150 * k, 1024, seed=20 + k).encoding) for k in range(5)]
    want = [renderer.render_to_texture(s, p) for s in seq]
    got = list(renderer.render_stream(seq, p))
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_flatten_stroke_line_fast_path_extremes(renderer, oracle):
    """k_flatten short-cuts stroked line-to segments (one line per side instead of the Euler machinery) behind a guard
    on chord / coordinate magnitude / width / transform scale. The oracle has no shortcut: bit-identical `lines` and
    path bboxes on strokes built to sit on both sides of that guard proves the equivalence where it is taken."""
    from vello_b200.encoding import Stroke, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND, STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE
    from vello_b200.shapes import Affine, BezPath
    from oracle.vbo import DTYPES
    rng = np.random.default_rng(321)
    s = Scene()
    joins, caps = (STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND), (STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE)
    for k in range(1500):
        p = BezPath()
        mag = [0.0, 1.0, 100.0, 4000.0, 16000.0, 60000.0, 3.0e5][k % 7]
        step = [1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 0.05, 0.3, 5.0, 300.0, 5e4][k % 10]
        width = [1e-3, 0.05, 1.0, 6.0, 40.0, 500.0, 1e4][(k // 3) % 7]
        x, y = rng.uniform(-mag, mag, 2) if mag else (0.0, 0.0)
        p.move_to(x, y)
        for _ in range(int(rng.integers(1, 7))):
            x += rng.normal(0, step)
            y += rng.normal(0, step)
            p.line_to(x, y)
        if k % 4 == 0:
            p.close_path()
        if k % 5 == 0:
            t = Affine((rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 2), rng.normal(0, 50), rng.normal(0, 50)))
        elif k % 5 == 1:
            t = Affine.scale(float(rng.choice([1e-3, 0.1, 0.999, 1.0, 3.7, 50.0, 2000.0])))
        else:
            t = Affine.translate(*rng.uniform(-10, 10, 2))
        # keep round joins / caps to a few hundred lines each (an arc of radius r px takes ~ pi / (2 acos(1 - 0.25 / r)) lines)
        norm = float(np.abs(np.array(t.coeffs[:4])).sum())
        width = min(width, 8000.0 / max(norm, 1e-6))
        st = Stroke(width, join=joins[k % 3], start_cap=caps[(k // 2) % 3], end_cap=caps[(k // 5) % 3], miter_limit=float(rng.choice([1.0, 4.0, 20.0])))
        s.stroke(st, t, Color.from_rgba8(50, 200, 50, 200), None, p)
    packed = resolve(s.encoding)
    p = RenderParams(BLACK, 256, 256, AA_AREA)
    renderer.render_to_texture(packed, p)  # sizes the arenas (grow-and-retry); run_stages below is a single attempt
    renderer.upload(packed)
    renderer.run_stages(p, "pathtag", "flatten")
    oracle.bind(packed, 256, 256)
    oracle.run("pathtag", "flatten")
    g, c = renderer.download("lines", DTYPES["lines"]), oracle.buffer("lines")
    assert g.shape == c.shape, (g.shape, c.shape)
    # degenerate strokes (zero-length tangents) yield NaN points on both sides; NaN payload bits differ between x86 and
    # the GPU (0xffc00000 vs 0x7fffffff), so NaNs are matched by position and everything else by bits
    gf = np.concatenate([g["p0"], g["p1"]], axis=1)
    cf = np.concatenate([c["p0"], c["p1"]], axis=1)
    assert np.array_equal(g["path_ix"], c["path_ix"])
    assert np.array_equal(np.isnan(gf), np.isnan(cf))
    same = (gf.view(np.uint32) == cf.view(np.uint32)) | np.isnan(gf)
    bad = np.nonzero(~same.all(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(g)} lines differ; first: {[(int(i), g[i], c[i]) for i in bad[:3]]}"
    assert int(np.isnan(gf).any(axis=1).sum()) < len(g) // 50
    assert renderer.download("path_bboxes", DTYPES["path_bboxes"]).tobytes() == oracle.buffer("path_bboxes").tobytes()


def test_native_scene_to_pixels(renderer, oracle):
    """Shapes -> pixels through the C ABI alone: a scene built with the native front end (vb_scene_*) and rendered with
    vb_render_scene gives the image the Python-encoded scene gives, which in turn matches the oracle."""
    import ctypes as C
    from vello_b200.renderer import FrameStats, _params_struct
    from vello_b200.scene_native import NativeScene
    from vello_b200.shapes import Affine, Circle, Rect
    from vello_b200.encoding import FILL_NON_ZERO, Gradient, Stroke, EXTEND_REFLECT, MIX_MULTIPLY, COMPOSE_SRC_OVER
    stops = [(0.0, Color.from_rgba8(255, 40, 0)), (0.6, Color.from_rgba8(0, 200, 90, 160)), (1.0, Color.from_rgba8(20, 0, 255))]
    py, nat = Scene(), NativeScene()
    for s in (py, nat):
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (300, 200), stops, EXTEND_REFLECT), None, Rect(10, 10, 290, 190))
        s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.rotate(0.2), Circle(150.0, 90.0, 80.0))
        s.stroke(Stroke(7.5), Affine.translate(20.0, 15.0), Color.from_rgba8(250, 250, 30, 220), None, Circle(120.0, 80.0, 60.0))
        s.fill(FILL_NON_ZERO, Affine.scale(1.5), Gradient.sweep((80, 60), 0.0, 6.0, stops), None, Rect(30, 20, 150, 110))
        s.pop_layer()
        s.draw_blurred_rounded_rect(Affine.translate(200.0, 150.0), Rect(-40, -20, 40, 20), Color.from_rgba8(255, 255, 255, 200), 6.0, 4.0)
    w, h = 300, 200
    for aa in (AA_AREA, AA_MSAA16):
        p = RenderParams(Color.from_rgba8(12, 12, 12), w, h, aa)
        packed = resolve(py.encoding)
        want = renderer.render_to_texture(packed, p)
        got = np.zeros((h, w, 4), dtype=np.uint8)
        ps, st = _params_struct(p, (0, 0)), FrameStats()
        rc = renderer.lib.vb_render_scene(renderer.handle, nat.handle, C.byref(ps), C.c_void_p(got.ctypes.data), 0, C.byref(st))
        assert rc == 0
        assert np.array_equal(got, want)
        assert_pixels(got, oracle.render(packed, w, h, p.base_color.premul_rgba8_u32(), aa), aa)


def test_cuda_graph_replay_is_invisible(oracle):
    """Whole frames are replayed as CUDA graphs, re-captured when anything a launch depends on changes. Alternating
    scenes, frame sizes, AA modes, stripes and host/device destinations must give the frames plain launches give."""
    from vello_b200.renderer import Renderer
    rg, rd = Renderer(), Renderer()
    rd.set_cuda_graph(False)
    a = resolve(scenes.paris_like(800, 512, seed=5).encoding)
    b = resolve(scenes.stroke_styles()[0].encoding)
    plan = [(a, 512, 512, AA_MSAA16, (0, 0)), (a, 512, 512, AA_MSAA16, (0, 0)), (b, 560, 480, AA_AREA, (0, 0)), (a, 512, 512, AA_MSAA16, (0, 0)),
            (a, 512, 512, AA_MSAA8, (0, 0)), (a, 512, 512, AA_MSAA16, (1, 2)), (b, 300, 200, AA_MSAA16, (0, 0)), (a, 512, 512, AA_MSAA16, (0, 0))]
    for packed, w, h, aa, rows in plan:
        p = RenderParams(BLACK, w, h, aa)
        g = rg.render_to_texture(packed, p, bin_rows=rows)
        d = rd.render_to_texture(packed, p, bin_rows=rows)
        assert np.array_equal(g, d)
        rg.upload(packed)
        rd.upload(packed)
        for _ in range(3):  # resident replays of the cached graph
            rg.render_resident(p, 0, rows)
        rd.render_resident(p, 0, rows)
        assert np.array_equal(rg.download_target(p, rows), rd.download_target(p, rows))
    full = oracle.render(a, 512, 512, BLACK.premul_rgba8_u32(), AA_MSAA16)
    assert np.array_equal(rg.render_to_texture(a, RenderParams(BLACK, 512, 512, AA_MSAA16)), full)
    rg.close()
    rd.close()


@pytest.fixture(scope="module")
def big_oracle():
    from oracle.vbo import Oracle
    return Oracle(threads=min(os.cpu_count() or 1, 64))


@pytest.mark.parametrize("workload", ["paris-30k", "beziers-100k-clips-1k"])
def test_full_size_parity(workload, big_oracle):
    """BASELINE.json configs[2] and [4] at their FULL size (4096x4096 MSAA16) against the oracle: every pixel identical,
    every bump total equal, every deterministic buffer byte-identical, the command streams of 2,000 tiles equal -- and the
    size-independent properties on top (run-to-run, bin-row stripes == rows of the full frame, occlusion start and graph
    replay invisible, no arena failure left behind)."""
    from vello_b200.renderer import Renderer
    if workload == "paris-30k":
        packed = resolve(scenes.paris_like(30000, 4096, seed=30000).encoding)
    else:
        packed = resolve(scenes.beziers_clips(100000, 1000, 4096, seed=100000).encoding)
    p = RenderParams(BLACK, 4096, 4096, AA_MSAA16)
    r = Renderer()
    full = r.render_to_texture(packed, p)
    assert r.last_stats.as_dict()["failed"] == 0
    ref = big_oracle.render(packed, 4096, 4096, BLACK.premul_rgba8_u32(), AA_MSAA16)
    assert np.array_equal(full, ref), f"{int((full != ref).any(axis=2).sum())} pixels differ from the oracle"
    rng = np.random.default_rng(1)
    parity.compare_all(r, big_oracle, packed.layout, 4096, 4096, check_ptcl_tiles=[int(t) for t in rng.choice(65536, 2000, replace=False)])
    assert np.array_equal(r.render_to_texture(packed, p), full)  # run-to-run: integer sample counts, no order dependence
    for b in (0, 7, 15):
        assert np.array_equal(r.render_to_texture(packed, p, bin_rows=(b, b + 1)), full[b * 256:(b + 1) * 256]), b
    r.set_occlusion_cull(False)
    r.set_cuda_graph(False)
    assert np.array_equal(r.render_to_texture(packed, p, bin_rows=(4, 8)), full[1024:2048])
    assert full[..., 3].min() == 255 and len(np.unique(np.ascontiguousarray(full).view(np.uint32))) > 1000
    # area AA on the same frame: exact against the oracle's fine on the GPU's command lists, within 1 LSB of its pipeline
    ref0 = big_oracle.render(packed, 4096, 4096, BLACK.premul_rgba8_u32(), AA_AREA)
    r.set_occlusion_cull(True)
    img0 = r.render_to_texture(packed, RenderParams(BLACK, 4096, 4096, AA_AREA))
    assert_pixels(img0, ref0, AA_AREA)
    parity.assert_replay(r, big_oracle, packed, img0, 4096, 4096, AA_AREA, BLACK)
    r.close()


def test_c4_stripes_against_oracle(big_oracle):
    """BASELINE.json configs[3]: paris-30k at 16384x16384 MSAA16 in bin-row stripes. Two of the 64 bin rows (one rank's
    share on a 32-way split; the 8-GPU split renders 8 such rows per rank) are rendered by the GPU as stripes and by the
    oracle with the same window: pixels identical. A fresh renderer is used per stripe, as a rank of the multi-GPU run
    would start (this is also a regression test of the stale failure flag: an attempt of each stripe overflows an arena).
    Bin row 21's first attempt overflows `tiles` (VB_STAGE_TILE_ALLOC: 622,840 tiles against a first guess sized from the
    draw count); bin row 63's first guesses hold it, so its second frame is forced to overflow `tiles` by one tile."""
    from vello_b200.renderer import Renderer
    size = 16384
    packed = resolve(scenes.paris_like(30000, size, seed=30000).encoding)
    p = RenderParams(BLACK, size, size, AA_MSAA16)
    for b in (21, 63):
        r = Renderer()
        got = r.render_to_texture(packed, p, bin_rows=(b, b + 1))
        st = r.last_stats.as_dict()
        assert st["failed"] == 0
        if b == 21:
            assert st["retries"] >= 1
        ref = big_oracle.render(packed, size, size, BLACK.premul_rgba8_u32(), AA_MSAA16, bin_rows=(b, b + 1))[b * 256:(b + 1) * 256]
        assert got.shape == ref.shape
        assert np.array_equal(got, ref), f"bin row {b}: {int((got != ref).any(axis=2).sum())} pixels differ (retries={st['retries']})"
        if b == 63:
            r.limit_arena("tiles", st["tile"] - 1)
        again = r.render_to_texture(packed, p, bin_rows=(b, b + 1))
        assert np.array_equal(again, ref)
        assert r.last_stats.retries == (1 if b == 63 else 0)
        r.close()


def test_failed_attempt_leaves_no_flag_in_a_stripe(oracle):
    """A stripe that does not contain tile 0 and whose first attempt overflows an arena: the successful re-run (and every
    later frame) must paint. The reference signals failure to fine through ptcl[0] (path_tiling_setup.wgsl:25), which only
    tile 0's owner rewrites; this implementation reads bump.failed."""
    from vello_b200.renderer import Renderer
    small, w0, h0 = scenes.filled_square()
    packed = resolve(scenes.paris_like(4000, 1024, seed=9).encoding)
    p = RenderParams(BLACK, 1024, 1024, AA_MSAA16)
    ref = oracle.render(packed, 1024, 1024, BLACK.premul_rgba8_u32(), AA_MSAA16)
    r = Renderer()
    r.upload(resolve(small.encoding))
    r.render_resident(RenderParams(BLACK, w0, h0, AA_AREA), 0, (0, 0))  # arenas sized for a tiny scene, nothing else
    # the first guesses, sized from this scene, hold the stripe: the overflow is forced on `lines` (VB_STAGE_FLATTEN) with a
    # limit one line below the stripe's need, on arenas that already held it
    assert np.array_equal(r.render_to_texture(packed, p, bin_rows=(1, 2)), ref[256:512])
    r.limit_arena("lines", int(r.last_stats.lines) - 1)
    for k, rows in enumerate(((1, 2), (2, 4), (1, 2))):
        got = r.render_to_texture(packed, p, bin_rows=rows)
        assert np.array_equal(got, ref[rows[0] * 256:rows[1] * 256]), (rows, r.last_stats.as_dict()["retries"])
        assert r.last_stats.retries == (1 if k == 0 else 0), (rows, r.last_stats.retries)
    r.close()
    r2 = Renderer()  # completely fresh: first-guess arenas from the scene itself
    assert np.array_equal(r2.render_to_texture(packed, p, bin_rows=(3, 4)), ref[768:1024])
    r2.close()


def test_gpu_against_libm_oracle(renderer, oracle_libm):
    """The product and the default oracle share vb_detmath.h (bit-reproducible transcendentals); a wrong polynomial there
    would be common-mode. The libm build of the oracle is the literal arithmetic of vello_shaders/src/cpu (Rust std ->
    platform libm): the GPU must stay within the bound tests/test_oracle_libm.py sets between the two oracle builds."""
    names = ("stroke_styles", "fill_types", "many_clips", "two_point_radial", "blend_grid", "tricky_strokes")
    cases = [("tiger", scenes.tiger(512, 512), 512, 512)] + [(n,) + getattr(scenes, n)() for n in names]
    for name, s, w, h in cases:
        packed = resolve(s.encoding)
        for aa in (AA_AREA, AA_MSAA16):
            img = renderer.render_to_texture(packed, RenderParams(BLACK, w, h, aa))
            ref = oracle_libm.render(packed, w, h, BLACK.premul_rgba8_u32(), aa)
            d = np.abs(img.astype(int) - ref.astype(int))
            if name == "tricky_strokes":
                # exact and near cusps turn a last-ulp difference of atan2 / sincos into a visibly different join on a few
                # hundred pixels of one 200x200 cell (the two ORACLE builds differ by the same 1158 / 696 channel values)
                assert (d > 1).mean() < 5e-4, (name, aa, int((d > 1).sum()))
                continue
            assert (d > 1).mean() < 2e-4, f"{name} aa={aa}: {(d > 1).sum()} channel values differ by more than 1 LSB from the libm oracle"
            assert d.max() <= 40
        gl = int(renderer.download("bump", np.uint32)[7])
        ol = int(oracle_libm.buffer("bump")["lines"][0])
        assert abs(gl - ol) <= max(4, ol // 2000)


def test_tile_row_stripes_equal_full_frame(renderer, oracle):
    """Stripes in TILE rows (vb_params.tile_row0/1, the granularity the cost-balanced multi-GPU split uses): any cut of the
    frame reproduces the full frame's rows exactly, including cuts inside a bin row and one-tile-row stripes."""
    w, h = 1024, 1000
    packed = resolve(scenes.paris_like(1500, 1024, seed=7).encoding)
    for aa in (AA_MSAA16, AA_AREA):
        p = RenderParams(BLACK, w, h, aa)
        full = renderer.render_to_texture(packed, p)
        for cuts in ([0, 5, 23, 24, 40, 63], [0, 1, 17, 31, 32, 33, 62, 63], [0, 63]):
            parts = [renderer.render_to_texture(packed, p, tile_rows=(a, b)) for a, b in zip(cuts, cuts[1:])]
            assert np.array_equal(np.concatenate(parts, axis=0), full), (aa, cuts)
    ref = oracle.render(packed, w, h, BLACK.premul_rgba8_u32(), AA_MSAA16)
    assert np.array_equal(renderer.render_to_texture(packed, RenderParams(BLACK, w, h, AA_MSAA16), tile_rows=(10, 30)), ref[160:480])
    s = scenes.tiger(512, 512)
    pk = resolve(s.encoding)
    pp = RenderParams(BLACK, 512, 512, AA_MSAA16)
    whole = renderer.render_to_texture(pk, pp)
    parts = [renderer.render_to_texture(pk, pp, tile_rows=(a, a + 3)) for a in range(0, 32, 3)]
    assert np.array_equal(np.concatenate(parts, axis=0)[:512], whole)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_group_one_call_one_frame(oracle, n):
    """vb_group: ONE call renders ONE frame on n renderers (here all on device 0 -- the multi-device path with every piece
    but the NVLink hop; bench.py and tests/test_multi_gpu.py run it on real devices). Host destination and device frame,
    with the cost balancing moving the stripe boundaries between frames: always the oracle's frame."""
    from vello_b200.renderer import RendererGroup
    packed = resolve(scenes.paris_like(2500, 1024, seed=4).encoding)
    p = RenderParams(BLACK, 1024, 1024, AA_MSAA16)
    ref = oracle.render(packed, 1024, 1024, BLACK.premul_rgba8_u32(), AA_MSAA16)
    g = RendererGroup([0] * n)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    g.upload(packed)
    seen = set()
    for k in range(6):
        st = g.render_resident(p)
        assert all(int(s.failed) == 0 for s in st)
        assert np.array_equal(g.frame_to_host(p), ref), k
        b, ms = g.stripes()
        assert b[0] == 0 and b[-1] == 64 and all(x < y for x, y in zip(b, b[1:]))
        seen.add(tuple(b))
    other = resolve(scenes.tiger(700, 500).encoding)
    p2 = RenderParams(BLACK, 700, 500, AA_AREA)
    got = g.render_to_texture(other, p2)
    assert_pixels(got, oracle.render(other, 700, 500, BLACK.premul_rgba8_u32(), AA_AREA), AA_AREA)
    g.close()


def test_device_resolve_equals_host_resolve(renderer, oracle):
    """Resolver::resolve on the device (vb_scene_upload_streams: stream copies to their Layout offsets + the patch / padding /
    ramp kernels, k_resolve.cu): packed scene, gradient ramps and image atlas are byte-identical to the host-side resolve --
    all brush kinds, duplicated gradients (one ramp) and images (one atlas slot), premultiplied and straight interpolation,
    unclosed clips (trailing PATH / END_CLIP tags), dashed strokes -- and so are the pixels. Stops are compared as floats with
    ==, by both resolves: -0 equals 0, and a stop holding a NaN equals nothing, itself included."""
    from vello_b200.scene_native import NativeScene
    from vello_b200.shapes import Affine, Circle, Rect, RoundedRect
    from vello_b200.encoding import FILL_NON_ZERO, FILL_EVEN_ODD, Gradient, Image, Stroke, EXTEND_REPEAT, MIX_SCREEN, COMPOSE_SRC_OVER
    rng = np.random.default_rng(8)
    stops = [(0.0, Color.from_rgba8(255, 40, 0)), (0.3, Color.from_rgba8(0, 200, 90, 100)), (0.31, Color.from_rgba8(20, 0, 255)), (1.0, Color.from_rgba8(250, 250, 0, 30))]
    img_a = rng.integers(0, 256, (9, 14, 4), dtype=np.uint8)
    img_b = rng.integers(0, 256, (30, 5, 4), dtype=np.uint8)
    nat = NativeScene()
    for k in range(3):
        g = Gradient.linear((0, 0), (300, 200), stops, EXTEND_REPEAT, premul_interp=(k != 1))
        nat.fill(FILL_NON_ZERO, Affine.translate(10.0 * k, 0.0), g, None, Rect(10, 10, 290, 190))
    nat.fill(FILL_EVEN_ODD, Affine.IDENTITY, Gradient.radial((150, 100), 5.0, (160, 110), 80.0, stops[:2]), None, Circle(150.0, 100.0, 90.0))
    nat.fill(FILL_NON_ZERO, Affine.scale(1.2), Gradient.sweep((80, 60), 0.0, 6.0, stops), None, RoundedRect(30, 20, 150, 110, 9.0))
    # the stops of the first ramp but for the sign of a zero, in an offset and in a colour channel: the same ramp
    c1 = stops[1][1]
    assert stops[0][0] == 0.0 and c1.r == 0.0
    for zs in ([(-0.0, stops[0][1])] + stops[1:], stops[:1] + [(0.3, Color(-0.0, c1.g, c1.b, c1.a))] + stops[2:]):
        nat.fill(FILL_NON_ZERO, Affine.translate(0.0, 15.0), Gradient.linear((0, 0), (300, 200), zs, EXTEND_REPEAT), None, Rect(20, 150, 120, 190))
    for im in (img_a, img_b, img_a):
        nat.draw_image(Image(im), Affine.translate(float(rng.uniform(0, 200)), float(rng.uniform(0, 100))) * Affine.scale(3.0))
    nat.stroke(Stroke(3.0, dash_pattern=(9.0, 4.0, 2.0), dash_offset=3.0), Affine.IDENTITY, Color.from_rgba8(255, 255, 255), None, Circle(200.0, 120.0, 60.0))
    nat.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 0.7, Affine.IDENTITY, Circle(100.0, 100.0, 80.0))
    nat.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(30, 90, 200, 180), None, Rect(40, 40, 260, 160))
    nat.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Rect(60, 60, 200, 140))  # both layers left open on purpose
    nat.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (300, 200), stops, EXTEND_REPEAT), None, Rect(0, 0, 300, 200))
    host = nat.resolve()
    layout = nat.upload_device(renderer)
    assert layout.as_array().tolist() == host.layout.as_array().tolist()
    assert renderer.download("scene", np.uint32).tobytes() == host.scene.tobytes()
    assert renderer.download("ramps", np.uint32).tobytes() == host.ramps.tobytes()
    assert host.ramps.shape[0] == 3  # (stops, premultiplied), (stops, straight), (first two stops): de-duplicated by (stops, space)
    assert renderer.download("atlas", np.uint8).tobytes() == host.atlas.tobytes()
    w, h = 300, 200
    for aa in (AA_MSAA16, AA_AREA):
        p = RenderParams(Color.from_rgba8(12, 12, 12), w, h, aa)
        want = renderer.render_to_texture(host, p)
        nat.upload_device(renderer)
        got = renderer.render_resident(p) and renderer.download_target(p)
        assert np.array_equal(got, want)
        assert_pixels(got, oracle.render(host, w, h, p.base_color.premul_rgba8_u32(), aa), aa)
    # two patches with the same NaN-holding stops: two ramps (their texels are not compared: host make_ramp and k_make_ramps
    # are not promised to agree on NaN)
    nan_stops = [(0.0, Color(float("nan"), 0.5, 0.5)), (1.0, Color.from_rgba8(0, 0, 255))]
    nan = NativeScene()
    for k in range(2):
        nan.fill(FILL_NON_ZERO, Affine.translate(20.0 * k, 0.0), Gradient.linear((0, 0), (100, 0), nan_stops), None, Rect(0, 0, 100, 50))
    host = nan.resolve()
    assert host.ramps.shape[0] == 2
    assert nan.upload_device(renderer).as_array().tolist() == host.layout.as_array().tolist()
    assert renderer.download("scene", np.uint32).tobytes() == host.scene.tobytes()
    assert renderer.download("ramps", np.uint32).size == host.ramps.size


@pytest.mark.parametrize("n", [2, 3, 5])
def test_group_with_sharded_flatten(oracle, n):
    """SURVEY.md 8(e) option B: every renderer of the group flattens only its share of the tag stream; lines (routed by the
    stripes they touch) and partial path boxes are exchanged through peer memory with epoch flags (k_exchange.cu). The
    assembled frame is the oracle's, for a host destination and for the device frame, across re-balanced stripes, new scenes
    (arenas rebuilt) and frames whose first attempt overflows an arena (re-issued on every renderer together)."""
    from vello_b200.renderer import RendererGroup
    packed = resolve(scenes.paris_like(2500, 1024, seed=4).encoding)
    p = RenderParams(BLACK, 1024, 1024, AA_MSAA16)
    ref = oracle.render(packed, 1024, 1024, BLACK.premul_rgba8_u32(), AA_MSAA16)
    g = RendererGroup([0] * n)
    g.set_exchange(True)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    g.upload(packed)
    for k in range(5):
        st = g.render_resident(p)
        assert all(int(s.failed) == 0 for s in st)
        assert np.array_equal(g.frame_to_host(p), ref), k
    total = sum(int(s.lines) for s in st)  # lines pulled by the stripes: all lines that touch the frame's rows (some twice)
    assert 0.8 * int(oracle.buffer("bump")["lines"][0]) < total < 1.3 * int(oracle.buffer("bump")["lines"][0])
    # strokes with round joins / caps (arcs), curves, clips and blends; area AA within 1 LSB
    for name in ("stroke_styles", "many_clips", "blend_grid"):
        s, w, h = getattr(scenes, name)()
        pk = resolve(s.encoding)
        for aa in (AA_MSAA16, AA_AREA):
            got = g.render_to_texture(pk, RenderParams(BLACK, w, h, aa))
            assert_pixels(got, oracle.render(pk, w, h, BLACK.premul_rgba8_u32(), aa), aa)
    big = resolve(scenes.paris_like(9000, 1024, seed=5).encoding)  # much larger: arenas overflow and the frame is re-issued
    assert np.array_equal(g.render_to_texture(big, p), oracle.render(big, 1024, 1024, BLACK.premul_rgba8_u32(), AA_MSAA16))
    g.set_exchange(False)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    g.close()
