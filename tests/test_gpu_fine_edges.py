"""Scenes aimed at the edges of `fine` (k_fine.cu) that ordinary scenes do not reach, each in area AA, MSAA8 and MSAA16:

1. winding numbers past what a biased byte holds (tile backdrops of +-126 .. +-457, more than 127 crossings in one tile row),
   where the MSAA resolve's byte arithmetic wraps and the WGSL's answer is not the geometric one;
2. the first-touch pixel list saturated: one fill with more than 1,000 segments in one tile, every pixel touched;
3. commands that start at the last offsets of a 256-byte command window and lists of several PTCL chunks;
4. the blend stack on both sides of VB_BLEND_STACK_SPLIT, with nesting depths 0-12 in neighbouring tiles;
5. scenes 1 and 3 in an odd-sized frame and in tile-row stripes that cut through them.

Each test first shows from the GPU's own buffers that the frame reached its edge, so that a change upstream (coarse,
path_tiling) cannot quietly make it a no-op. Then: `compare_all` against the oracle, pixels byte for byte against the
oracle's fine replayed on the GPU's buffers (every AA mode), and for MSAA byte for byte against the oracle's full pipeline."""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (BLACK, COMPOSE_DEST_OVER, COMPOSE_PLUS, COMPOSE_SRC_ATOP, COMPOSE_SRC_IN, COMPOSE_SRC_OVER,
                                 COMPOSE_XOR, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_COLOR_BURN, MIX_COLOR_DODGE, MIX_DIFFERENCE,
                                 MIX_HARD_LIGHT, MIX_HUE, MIX_LUMINOSITY, MIX_MULTIPLY, MIX_NORMAL, MIX_OVERLAY, MIX_SCREEN,
                                 MIX_SOFT_LIGHT, TRANSPARENT, Color, Scene, resolve)
from vello_b200.shapes import Affine, BezPath, Circle, Rect

from . import parity
from .test_gpu_parity import assert_pixels

pytestmark = pytest.mark.gpu

AAS = [AA_AREA, AA_MSAA8, AA_MSAA16]
CMD_FILL, CMD_SOLID, CMD_COLOR, CMD_BEGIN_CLIP, CMD_END_CLIP, CMD_JUMP, CMD_END = 1, 3, 5, 10, 11, 12, 0
WIN_WORDS = 64  # k_fine.cu: a command window is 256 bytes
PTCL_INITIAL_ALLOC = 64


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def render_and_check(renderer, oracle, packed, w, h, aa, base=BLACK):
    """Render on the GPU and in the oracle; compare stage by stage, then pixels. Returns the GPU image and the GPU's
    ptcl / segments / bump of that frame."""
    img = renderer.render_to_texture(packed, RenderParams(base, w, h, aa))
    g = parity.gpu_buffers(renderer, ["ptcl", "segments", "bump"])
    ref = oracle.render(packed, w, h, base.premul_rgba8_u32(), aa)
    parity.compare_all(renderer, oracle, packed.layout, w, h)
    if aa == AA_AREA:
        assert_pixels(img, ref, aa)
    else:
        assert np.array_equal(img, ref), f"aa={aa}: {int((img != ref).any(axis=2).sum())} pixels differ from the oracle"
    parity.assert_replay(renderer, oracle, packed, img, w, h, aa, base)
    return img, g


def walk_tile(ptcl, tile):
    """The commands of one tile as fine reads them with occlusion cull off (k_fine.cu, tile loop): start after the blend
    offset at the tile's head, window base = start & ~3, a re-stage whenever the offset into the window exceeds
    WIN_WORDS - 4 (which includes every CMD_JUMP target outside the window). Yields (tag, index, offset into the window
    before the re-stage check)."""
    cmd_ix = tile * PTCL_INITIAL_ALLOC + 1
    win_base = cmd_ix & ~3
    while True:
        off = (cmd_ix - win_base) & 0xFFFFFFFF
        if off > WIN_WORDS - 4:
            win_base = cmd_ix & ~3
        tag = int(ptcl[cmd_ix])
        yield tag, cmd_ix, off
        if tag == CMD_END:
            return
        if tag == CMD_JUMP:
            cmd_ix = int(ptcl[cmd_ix + 1])
        else:
            cmd_ix += parity.CMD_SIZES[tag]


def fills(ptcl, n_tiles):
    """Every FILL of the frame: (tile, n_segs, even_odd, seg_ix, backdrop)."""
    out = []
    for t in range(n_tiles):
        for tag, ix, _ in walk_tile(ptcl, t):
            if tag == CMD_FILL:
                sr = int(ptcl[ix + 1])
                out.append((t, sr >> 1, sr & 1, int(ptcl[ix + 2]), int(np.int32(np.uint32(ptcl[ix + 3])))))
    return out


def n_tiles_of(w, h):
    return ((w + 15) // 16) * ((h + 15) // 16)


# ---- 1. winding beyond a byte -------------------------------------------------------------------------------------------
# left edges per tile column: the backdrop of a tile is the number of edges left of it, so interior tiles of columns 1..7
# and 31 hold 126, 127, 128, 129, 255, 256, 456 and 457; column 6 holds 200 edges (200 crossings in every pixel row)
EDGES_PER_COLUMN = [126, 1, 1, 1, 126, 1, 200, 1]


def winding_scene(rule, y0=20.0, y1=108.0):
    """One path: 457 rectangles with integer corners, all wound the same way, sharing their right edge x = 500 and top /
    bottom rows y0 / y1 (which cross the left boundary of every tile they pass at local row 4 and 12), their left edges
    spread over tile columns 0-7. Inside column 3 (backdrop 128) 128 rectangles x 50-60 are wound the other way, so pixels
    51-59 have a winding of 0 -- and a winding byte of 128 - 128 = 0 against a backdrop of 128, the case where fine.wgsl
    reports full coverage and k_fine.cu's test of untouched pixels takes its out-of-range branch. Then the mirror image of
    all of it about y = 128, wound the opposite way (backdrop -128 against a winding byte of 0: uncovered)."""
    p = BezPath()

    def rect(xa, xb, ya, yb):
        p.move_to(xa, ya)
        p.line_to(xb, ya)
        p.line_to(xb, yb)
        p.line_to(xa, yb)
        p.close_path()

    for c, n in enumerate(EDGES_PER_COLUMN):
        for j in range(n):
            x = 62 if c == 3 else 16 * c + 1 + j % 14
            rect(x, 500.0, y0, y1)
            rect(x, 500.0, 256.0 - y0, 256.0 - y1)
    for _ in range(128):
        rect(60.0, 50.0, y0, y1)
        rect(60.0, 50.0, 256.0 - y0, 256.0 - y1)
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(30, 60, 90), None, Rect(0, 0, 600, 500))
    s.fill(rule, Affine.IDENTITY, Color.from_rgba8(250, 200, 40, 230), None, p)
    return s


def assert_winding_edges(g, w, h):
    fl = fills(g["ptcl"], n_tiles_of(w, h))
    bds = {f[4] for f in fl}
    for v in (126, 127, 128, 129, 255, 256):
        assert v in bds and -v in bds, (v, sorted(bds))
    assert max(abs(b) for b in bds) > 300
    segs = g["segments"]
    row_crossings, left_edge = 0, 0
    for _, n, _, ix, _ in fl:
        s = segs[ix:ix + n]
        lo, hi = np.minimum(s["p0"][:, 1], s["p1"][:, 1]), np.maximum(s["p0"][:, 1], s["p1"][:, 1])
        centres = np.arange(16) + 0.5
        row_crossings = max(row_crossings, int(((lo[None, :] < centres[:, None]) & (hi[None, :] > centres[:, None])).sum(1).max()))
        left_edge = max(left_edge, int((s["y_edge"] < 1e9).sum()))  # segments ending on the tile's left edge (wind_y)
    assert row_crossings > 127, row_crossings  # packed_w bytes wrap
    assert left_edge > 127, left_edge          # wind_y bytes wrap
    return bds


@pytest.mark.parametrize("rule", [FILL_NON_ZERO, FILL_EVEN_ODD])
@pytest.mark.parametrize("aa", AAS)
def test_winding_beyond_a_byte(renderer, oracle, rule, aa):
    w, h = 512, 256
    packed = resolve(winding_scene(rule).encoding)
    img, g = render_and_check(renderer, oracle, packed, w, h, aa)
    assert_winding_edges(g, w, h)
    if aa != AA_AREA:
        # where the winding fits a byte the MSAA answer is geometric: in pixel row 85 (both loop sets' rows are 20-108 and
        # 148-236) pixel 0 lies left of every edge (winding 0) and pixel 24 right of 127 of them (x <= 17): odd, so it is
        # covered under both rules; so is its mirror image in row 170 (winding -127)
        bg, fg = np.array([30, 60, 90]), np.array([250, 200, 40])
        for y in (85, 170):
            assert (img[y, 0, :3] == bg).all()
            assert np.abs(img[y, 24, :3].astype(int) - (fg * 230 + bg * 25) / 255).max() <= 1, img[y, 24]
        if rule == FILL_NON_ZERO:
            # pixels 51-59 have a winding of 0. Against a backdrop of -128 the winding byte 0 is expected_zero = 128:
            # uncovered. Against +128, expected_zero = -128 is out of a byte's range and fine.wgsl:452 reports full
            # coverage: the WGSL's answer, not the geometric one, and the one the kernel must give.
            assert (img[170, 51:60] == img[170, 0]).all()
            assert (img[85, 51:60] == img[85, 24]).all()


# ---- 2. the first-touch list saturated ------------------------------------------------------------------------------------
def touch_scene(rule):
    """A zigzag of 1,200 random lines confined to tile (1, 1) plus a sweep along every pixel row of it, then a triangle of
    3 lines in the same tile."""
    rng = np.random.default_rng(17)
    p = BezPath()
    p.move_to(16.3, 16.5)
    for r in range(16):
        p.line_to(31.7, 16.5 + r)
        p.line_to(16.3, 16.9 + r)
    for x, y in rng.uniform(16.1, 31.9, (1200, 2)):
        p.line_to(float(x), float(y))
    p.close_path()
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(20, 20, 60), None, Rect(0, 0, 64, 64))
    s.fill(rule, Affine.IDENTITY, Color.from_rgba8(240, 120, 30, 200), None, p)
    s.fill(rule, Affine.IDENTITY, Color.from_rgba8(40, 220, 120, 160), None,
           BezPath([("M", 18.2, 18.7), ("L", 24.6, 19.1), ("L", 20.3, 26.4), ("Z",)]))
    return s


@pytest.mark.parametrize("rule", [FILL_NON_ZERO, FILL_EVEN_ODD])
@pytest.mark.parametrize("aa", AAS)
def test_first_touch_list_saturated(renderer, oracle, rule, aa):
    w = h = 64
    packed = resolve(touch_scene(rule).encoding)
    img, g = render_and_check(renderer, oracle, packed, w, h, aa)
    tile = 1 * (w // 16) + 1
    fl = [f for f in fills(g["ptcl"], n_tiles_of(w, h)) if f[0] == tile]
    assert len(fl) == 2 and fl[0][1] >= 1000 and fl[1][1] <= 4, [f[:3] for f in fl]
    segs = g["segments"][fl[0][3]:fl[0][3] + fl[0][1]]
    tt = np.linspace(0.0, 1.0, 400)[None, :]
    xs = segs["p0"][:, :1] + (segs["p1"][:, :1] - segs["p0"][:, :1]) * tt
    ys = segs["p0"][:, 1:] + (segs["p1"][:, 1:] - segs["p0"][:, 1:]) * tt
    touched = np.unique(np.clip(ys.astype(int), 0, 15) * 16 + np.clip(xs.astype(int), 0, 15))
    assert len(touched) == 256


# ---- 3. command-window boundaries -----------------------------------------------------------------------------------------
def command_scene(n_draws=1500, size=128, seed=3):
    """Random draws over a size x size frame that interleave every kind of command in every tile: whole-frame fills
    (SOLID + COLOR, mostly translucent so that occlusion cull keeps some lists long), circles and rectangles that cover
    parts of tiles (FILL + COLOR), and clip / blend layers up to 3 deep (BEGIN_CLIP; FILL or SOLID + END_CLIP)."""
    rng = np.random.default_rng(seed)
    s = Scene()
    depth = 0
    mixes = [MIX_NORMAL, MIX_MULTIPLY, MIX_SCREEN, MIX_DIFFERENCE]

    def color():
        a = 255 if rng.random() < 0.04 else int(rng.integers(40, 230))
        return Color.from_rgba8(*[int(v) for v in rng.integers(0, 256, 3)], a)

    for _ in range(n_draws):
        k = rng.random()
        if k < 0.35:
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, color(), None, Rect(-4, -4, size + 4, size + 4))
        elif k < 0.75:
            x, y = rng.uniform(0, size, 2)
            if rng.random() < 0.5:
                shape = Circle(float(x), float(y), float(rng.uniform(4, size / 2)))
            else:
                shape = Rect(float(x), float(y), float(x + rng.uniform(5, size)), float(y + rng.uniform(5, size)))
            s.fill(FILL_NON_ZERO if rng.random() < 0.7 else FILL_EVEN_ODD, Affine.IDENTITY, color(), None, shape)
        elif k < 0.87 and depth < 3:
            x, y = rng.uniform(-10, size / 2, 2)
            clip = Rect(float(x), float(y), float(x + rng.uniform(size / 2, size + 20)), float(y + rng.uniform(size / 2, size + 20)))
            if rng.random() < 0.5:
                s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, clip)
            else:
                s.push_layer(FILL_NON_ZERO, mixes[int(rng.integers(0, 4))], COMPOSE_SRC_OVER, float(rng.uniform(0.3, 1.0)), Affine.IDENTITY, clip)
            depth += 1
        elif depth > 0:
            s.pop_layer()
            depth -= 1
    for _ in range(depth):
        s.pop_layer()
    return s


def assert_window_edges(ptcl, w, h):
    kinds = (CMD_FILL, CMD_COLOR, CMD_SOLID, CMD_BEGIN_CLIP, CMD_END_CLIP)
    seen, jumps, max_jumps = set(), 0, 0
    for t in range(n_tiles_of(w, h)):
        tj = 0
        for tag, _, off in walk_tile(ptcl, t):
            if 57 <= off <= 63:
                seen.add((tag, off))
            tj += tag == CMD_JUMP
        jumps += tj
        max_jumps = max(max_jumps, tj)
    missing = [(k, o) for k in kinds for o in range(57, 64) if (k, o) not in seen]
    assert not missing, missing
    assert jumps > 0 and max_jumps >= 3, (jumps, max_jumps)  # some tile's list spans 3 or more 256-word chunks


@pytest.mark.parametrize("cull", [True, False])
@pytest.mark.parametrize("aa", AAS)
def test_command_window_boundaries(renderer, oracle, cull, aa):
    w = h = 128
    packed = resolve(command_scene().encoding)
    renderer.set_occlusion_cull(cull)
    try:
        img, g = render_and_check(renderer, oracle, packed, w, h, aa, base=Color.from_rgba8(9, 9, 9))
    finally:
        renderer.set_occlusion_cull(True)
    assert_window_edges(g["ptcl"], w, h)


# ---- 4. the blend stack across the split ----------------------------------------------------------------------------------
LAYER_MODES = {  # depth (1-based) -> (mix, compose); depth 9 is a luminance mask
    1: None, 2: (MIX_NORMAL, COMPOSE_SRC_OVER), 3: None, 4: (MIX_MULTIPLY, COMPOSE_SRC_OVER), 5: (MIX_SCREEN, COMPOSE_SRC_ATOP),
    6: (MIX_OVERLAY, COMPOSE_XOR), 7: (MIX_COLOR_DODGE, COMPOSE_DEST_OVER), 8: (MIX_DIFFERENCE, COMPOSE_PLUS), 9: "luminance",
    10: (MIX_HARD_LIGHT, COMPOSE_SRC_IN), 11: (MIX_HUE, COMPOSE_SRC_OVER), 12: (MIX_LUMINOSITY, COMPOSE_SRC_ATOP),
}
EXTRA_MIXES = [MIX_SOFT_LIGHT, MIX_COLOR_BURN]


def blend_scene():
    """12 nested layers over a 256 x 64 frame; layer k clips to x >= 16k + 3, so tile column c is nested min(c, 12) deep
    and its neighbours one level less or more. Every layer paints a translucent rectangle and a circle per tile row."""
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 180, 40), None, Rect(0, 0, 256, 64))
    for k in range(1, 13):
        clip = Rect(16 * k + 3, 1.5, 300, 62.5)
        m = LAYER_MODES[k]
        if m is None:
            s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, clip)
        elif m == "luminance":
            s.push_luminance_mask_layer(FILL_NON_ZERO, 0.9, Affine.IDENTITY, clip)
        else:
            s.push_layer(FILL_NON_ZERO, m[0], m[1], 0.85, Affine.IDENTITY, clip)
        c = Color.from_rgba8((37 * k) % 256, (91 * k) % 256, (53 * k + 100) % 256, 120 + 10 * k)
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Rect(16 * k - 5, 4 + k, 250 - 3 * k, 60 - k))
        for ty in range(4):
            s.fill(FILL_EVEN_ODD, Affine.IDENTITY, Color.from_rgba8(255 - 20 * k, 30 * (k % 8), 200, 180), None,
                   Circle(16.0 * k + 20.0 + 7 * ty, 16.0 * ty + 8.0, 6.0 + k % 3))
        if k in (6, 11):  # two more mixes at depth >= 4
            s.push_layer(FILL_NON_ZERO, EXTRA_MIXES[k == 11], COMPOSE_SRC_OVER, 0.7, Affine.IDENTITY, Rect(16 * k + 6, 20, 200, 44))
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(90, 200, 250, 200), None, Circle(16.0 * k + 30.0, 32.0, 12.0))
            s.pop_layer()
    for _ in range(12):
        s.pop_layer()
    return s


def tile_depths(ptcl, n_tiles):
    out = []
    for t in range(n_tiles):
        d = dmax = 0
        for tag, _, _ in walk_tile(ptcl, t):
            if tag == CMD_BEGIN_CLIP:
                d += 1
                dmax = max(dmax, d)
            elif tag == CMD_END_CLIP:
                d -= 1
        assert d == 0
        out.append(dmax)
    return out


@pytest.mark.parametrize("aa", AAS)
def test_blend_stack_across_the_split(renderer, oracle, aa):
    w, h = 256, 64
    packed = resolve(blend_scene().encoding)
    img, g = render_and_check(renderer, oracle, packed, w, h, aa)
    assert int(g["bump"]["blend"][0]) > 0
    depths = tile_depths(g["ptcl"], n_tiles_of(w, h))
    for d in (0, 3, 4, 5):
        assert d in depths, depths
    assert max(depths) >= 8, depths
    row = depths[:16]
    assert all(a != b for a, b in zip(row[:12], row[1:13])), row  # neighbouring tiles at different depths


# ---- 5. odd frame and stripes ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["winding", "commands"])
@pytest.mark.parametrize("aa", AAS)
def test_odd_frame_and_stripes(renderer, oracle, which, aa):
    """Scenes 1 and 3 at 561 x 479 (30 tile rows, the last one partial) on a transparent base, then in two tile-row stripes
    cut inside the scene: each stripe equals the matching rows of the full frame."""
    w, h = 561, 479
    if which == "winding":
        packed, cut = resolve(winding_scene(FILL_NON_ZERO).encoding), 4
    else:
        packed, cut = resolve(command_scene(n_draws=900, size=200, seed=8).encoding), 7
    img, g = render_and_check(renderer, oracle, packed, w, h, aa, base=TRANSPARENT)
    if which == "winding":
        assert_winding_edges(g, w, h)
    else:
        seen = {(tag, off) for t in range(n_tiles_of(w, h)) for tag, _, off in walk_tile(g["ptcl"], t) if off > WIN_WORDS - 4}
        assert {t for t, _ in seen} >= {CMD_FILL, CMD_COLOR, CMD_SOLID}, seen  # commands past the window's end re-stage
    p = RenderParams(TRANSPARENT, w, h, aa)
    parts = [renderer.render_to_texture(packed, p, tile_rows=rows) for rows in ((0, cut), (cut, 30))]
    assert parts[0].shape[0] == 16 * cut and parts[1].shape[0] == h - 16 * cut
    assert np.array_equal(np.concatenate(parts, axis=0), img)
