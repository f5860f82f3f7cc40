"""k_backdrop (k_tile.cu) against a serial reference of the same operation, at the edges of its chunked look-back.

backdrop cuts the tile arena into 4096-tile chunks; a thread walks 16 consecutive tiles, a warp 512, and a decoupled
look-back over the chunks carries a segmented sum (row start seen, backdrop since it) and the crossing count. Each tile
leaves as {backdrop summed along its row, ~first slot of its segment slice}. A wrong carry only shows on an arena that puts
a boundary in exactly the wrong place, so:

1. CPU: `backdrop_ref` (tests/backdrop_ref.py) equals the oracle's backdrop stage on the parity scenes and a plain per-row
   loop on the crafted arenas, and every crafted arena reaches the edges it is named for.
2. GPU: backdrop alone on crafted arenas (paths and tiles uploaded, the arena limited to its end so that a write past it
   shows in the guard region), every tile word compared with the reference.
3. GPU: whole frames at the same edges (frames up to 65536 px wide, arenas at chunk multiples, chunks over more than 256
   paths) through `compare_all`, the replayed fine and the pixel bar of test_gpu_parity, in area AA and MSAA16.
"""
import numpy as np
import pytest

from oracle.vbo import DTYPES
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_EVEN_ODD, FILL_NON_ZERO, Color, Scene, Stroke, resolve
from vello_b200.shapes import Affine, BezPath, Ellipse, Rect

from . import parity
from .backdrop_ref import BD_CHUNK, BD_STAGE, BD_WARP_TILES, backdrop_ref, cases, chunk_paths, reaches, row_layout

CASES = cases()


# ---- CPU: the reference itself ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["filled_circle", "robust_paths", "funky_paths", "fill_types", "stroke_styles", "many_clips",
                                  "deep_blend", "brushes", "blend_grid", "compose_grid", "tricky_strokes", "gradient_extend",
                                  "two_point_radial", "conflation_artifacts", "longpathdash"])
def test_backdrop_ref_matches_oracle(oracle, name):
    """The reference applied to the oracle's tiles after path_count equals the oracle's tiles after backdrop; the oracle's
    `tile_counts` are the counts path_count left in the tiles."""
    from vello_b200 import scenes
    s, w, h = getattr(scenes, name)()
    packed = resolve(s.encoding)
    oracle.bind(packed, w, h)
    oracle.run("pathtag", "path_count")
    n_draw = packed.layout.n_draw_objects
    paths = oracle.buffer("paths")[:n_draw]
    tiles = oracle.buffer("tiles")
    end = int(oracle.buffer("bump")["tile"][0])
    assert tiles.shape == (end,)
    assert np.array_equal(oracle.buffer("tile_counts"), tiles["segment_count_or_ix"])
    want, total = backdrop_ref(paths, tiles, end)
    oracle.run("backdrop", "backdrop")
    after = oracle.buffer("tiles")
    assert np.array_equal(want["backdrop"], after["backdrop"]), name
    assert total == int(tiles["segment_count_or_ix"].astype(np.int64).sum())


def _loop_ref(paths, tiles, arena_end):
    """backdrop as the oracle's serial stage states it: per path, per row, a running sum; the slices by a running count."""
    bd = tiles["backdrop"][:arena_end].astype(np.int64).copy()
    for p in paths:
        w, h, start = int(p["bbox"][2] - p["bbox"][0]), int(p["bbox"][3] - p["bbox"][1]), int(p["tiles"])
        for r0 in range(start, start + w * h, max(w, 1)):
            bd[r0:r0 + w] = np.cumsum(bd[r0:r0 + w])
    words, slot = np.zeros(arena_end, np.uint32), 0
    counts = tiles["segment_count_or_ix"][:arena_end]
    for t in range(arena_end):
        words[t] = ~np.uint32(slot)
        slot = (slot + int(counts[t])) & 0xFFFFFFFF
    return (bd & 0xFFFFFFFF).astype(np.uint32).view(np.int32), words, slot


@pytest.mark.parametrize("case", [c for c in CASES if c.arena_end <= 120_000], ids=repr)
def test_backdrop_ref_matches_a_loop(case):
    """The vectorised reference equals a plain loop over each path's rows on the crafted arenas."""
    paths, tiles = case.build()
    want, total = backdrop_ref(paths, tiles, case.arena_end)
    bd, words, slot = _loop_ref(paths, tiles, case.arena_end)
    assert np.array_equal(want["backdrop"], bd)
    assert np.array_equal(want["segment_count_or_ix"], words)
    assert total == slot


@pytest.mark.parametrize("case", CASES, ids=repr)
def test_crafted_case_reaches_its_edges(case):
    """Each crafted arena reaches the boundaries it is named for, so that an edit to the generator cannot silently lose
    them."""
    paths, _ = case.build()
    got = reaches(paths, case.arena_end)
    assert case.expect, "every case names what it reaches"
    assert case.expect <= got, (case.name, sorted(case.expect - got))


def test_crafted_cases_cover_every_edge():
    """Together the cases reach every edge the kernel has: odd ends and chunk-multiple ends, row starts at thread, warp and
    chunk seams, warps and chunks without a row start, chunks over more than BD_STAGE paths, empty paths at the ends and at
    chunk edges, and a look-back over more than 1000 chunks."""
    seen = set().union(*(c.expect for c in CASES))
    need = {"empty", "end%16=1", "end%16=0", "end%4096=0", "end%4096=4095", "end%4096=1", "start%16=0", "start%16=1",
            "start%16=15", "start%512=511", "start%512=0", "start%4096=4095", "start%4096=0", "row-spans-chunk",
            "warp-no-start", "chunk-no-start", "unstaged", "empty-first", "empty-last", "empty-at-chunk-first",
            "empty-at-chunk-last", "1000-chunks"}
    assert need <= seen, sorted(need - seen)
    big = [c for c in CASES if c.values == "big"]
    assert big and any(c.arena_end >= 1000 * BD_CHUNK for c in big)
    paths, tiles = big[0].build()
    assert int(tiles["segment_count_or_ix"].astype(np.uint64).sum()) > 0xFFFFFFFF, "the total of the counts wraps u32"
    assert np.abs(tiles["backdrop"].astype(np.int64)).max() >= (1 << 30) - 4096


# ---- GPU: backdrop alone on crafted arenas ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


_FILLS = {}


def fills(n):
    """A scene of n small fills (n draw objects, each over one tile, each with crossings): it sizes the per-draw buffers
    backdrop reads, and its own frame leaves a non-zero bump.segments for the crafted arena to overwrite."""
    if n not in _FILLS:
        s = Scene()
        for i in range(n):
            x, y = 16.0 * (i % 16) + 3.0, 16.0 * ((i // 16) % 16) + 3.0
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 100, 50), None, Rect(x, y, x + 9.5, y + 7.25))
        _FILLS[n] = resolve(s.encoding)
        assert _FILLS[n].layout.n_draw_objects == n
    return _FILLS[n]


def run_backdrop(r, paths, tiles, arena_end):
    """backdrop alone on the uploaded paths and tiles (vb_debug_upload's protocol). Returns the tiles, bump and seg_holes
    after it, and the guard region past arena_end."""
    p = RenderParams(BLACK, 256, 256, AA_AREA)
    r.limit_arena("tiles", r.NO_LIMIT)
    r.upload(fills(len(paths)))
    r.run_stages(p, "pathtag", "path_count")  # per-draw buffers of n draw objects
    r.upload_buffer("tiles", tiles)  # grows the arena (without copying)
    r.run_stages(p, "pathtag", "backdrop")  # control block sized from the tile capacity and zeroed; the fills' own slices
    b = r.download("bump", DTYPES["bump"])[0]
    assert int(b["failed"]) == 0 and int(b["segments"]) > 0
    r.upload_buffer("paths", paths)
    r.upload_buffer("tiles", tiles)  # also sets bump.tile = arena_end
    if arena_end:
        r.limit_arena("tiles", arena_end)  # the kernel sees the same end, and bytes past it become the guard
    r.run_stages(p, "backdrop", "backdrop")
    got = r.download("tiles", DTYPES["tiles"])
    bump = r.download("bump", DTYPES["bump"])[0]
    holes = int(r.download("seg_holes", np.uint32)[0])
    guard = r.download_guard("tiles") if arena_end else None
    r.limit_arena("tiles", r.NO_LIMIT)
    return got, bump, holes, guard


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_backdrop_crafted(renderer, case):
    paths, tiles = case.build()
    want, total = backdrop_ref(paths, tiles, case.arena_end)
    got, bump, holes, guard = run_backdrop(renderer, paths, tiles, case.arena_end)
    assert int(bump["failed"]) == 0
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.nonzero((got["backdrop"] != want["backdrop"]) | (got["segment_count_or_ix"] != want["segment_count_or_ix"]))[0]
    if len(bad):
        t = int(bad[0])
        raise AssertionError(f"{case.name}: {len(bad)} of {case.arena_end} tiles differ, first at tile {t} (chunk {t // BD_CHUNK}, "
                             f"offset {t % BD_CHUNK}): got {got[t]}, want {want[t]}")
    assert int(bump["segments"]) == total and holes == total, (int(bump["segments"]), holes, total)
    if guard is not None:
        assert len(guard) > 0
        over = np.nonzero(guard != renderer.GUARD_BYTE)[0]
        assert len(over) == 0, f"backdrop wrote {len(over)} bytes past the arena's end, first at byte {int(over[0])}"


# ---- GPU: whole frames at the same edges -------------------------------------------------------------------------------
def check_frame(renderer, oracle, packed, w, h):
    """compare_all, the replayed fine and the pixel bar of test_gpu_parity, in area AA and MSAA16. Returns the GPU's paths,
    tiles and bump of the last frame."""
    from .test_gpu_parity import assert_pixels
    for aa in (AA_AREA, AA_MSAA16):
        img = renderer.render_to_texture(packed, RenderParams(BLACK, w, h, aa))
        ref = oracle.render(packed, w, h, BLACK.premul_rgba8_u32(), aa)
        parity.compare_all(renderer, oracle, packed.layout, w, h)
        parity.assert_replay(renderer, oracle, packed, img, w, h, aa, BLACK)
        assert_pixels(img, ref, aa)
    g = parity.gpu_buffers(renderer, ["paths", "tiles", "bump"])
    return g["paths"], g["tiles"], g["bump"][0]


def carried(paths, tiles, span):
    """Tiles at a multiple of `span` that do not start a row and carry a non-zero backdrop into it."""
    end = len(tiles)
    _, _, start = row_layout(paths, end)
    t = np.arange(span, end, span)
    return t[~start[t] & (tiles["backdrop"][t] != 0)]


def wide_scene(w, h):
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(40, 90, 200, 200), None, Rect(3.5, 2.25, w - 2.5, h * 0.4))
    zig = BezPath()  # an even-odd band that crosses itself along the whole width
    zig.move_to(1.0, h * 0.5)
    for k in range(1, 41):
        zig.line_to(w * k / 40.0, h * (0.3 if k % 2 else 0.95))
    zig.line_to(w - 1.0, h * 0.1)
    zig.line_to(2.0, h * 0.9)
    zig.close_path()
    s.fill(FILL_EVEN_ODD, Affine.IDENTITY, Color.from_rgba8(220, 200, 30, 160), None, zig)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(30, 220, 90, 128), None, Ellipse(w * 0.5, h * 0.6, w * 0.47, h * 0.35))
    s.stroke(Stroke(3.0), Affine.IDENTITY, Color.from_rgba8(250, 250, 250), None, Ellipse(w * 0.45, h * 0.5, w * 0.44, h * 0.4))
    return resolve(s.encoding)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(8208, 48), (20000, 40), (65536, 32)])
def test_wide_frames(renderer, oracle, w, h):
    """Rows wider than a warp's 512 tiles (8208 px = 513 tiles), than several warps (20000 px), and of a whole chunk
    (65536 px = 4096 tiles, the widest frame): non-zero backdrops cross warp and, in the wider two, chunk boundaries."""
    packed = wide_scene(w, h)
    paths, tiles, bump = check_frame(renderer, oracle, packed, w, h)
    widths = paths["bbox"][:, 2] - paths["bbox"][:, 0]
    assert int(widths.max()) > BD_WARP_TILES
    assert len(carried(paths, tiles, BD_WARP_TILES)) > 0, "a non-zero backdrop crosses a warp boundary inside a row"
    if w >= 20000:
        assert len(carried(paths, tiles, BD_CHUNK)) > 0, "a non-zero backdrop crosses a chunk boundary inside a row"
    assert int(bump["tile"]) == len(tiles)


# tile-aligned fills of a 64 x 64-tile frame whose tile counts sum to each arena end: (x0, y0, x1, y1) in tiles
BLOCKS = {4095: [(0, 0, 64, 63), (0, 0, 63, 1)], 4096: [(0, 0, 64, 64)], 4097: [(0, 0, 64, 64), (5, 7, 6, 8)],
          8191: [(0, 0, 64, 64), (0, 1, 64, 64), (1, 0, 64, 1)], 8192: [(0, 0, 64, 64), (0, 0, 64, 64)],
          8193: [(0, 0, 64, 64), (0, 0, 64, 64), (63, 63, 64, 64)]}


@pytest.mark.gpu
@pytest.mark.parametrize("end", sorted(BLOCKS))
def test_arena_at_chunk_multiples(renderer, oracle, end):
    """1024 x 1024 (64 x 64 tiles) with tile-aligned fills whose tiles sum to an arena end at, or one either side of, one
    and two chunks: the odd ends take the int2 tails of k_tile_zero and backdrop."""
    s = Scene()
    for k, (x0, y0, x1, y1) in enumerate(BLOCKS[end]):
        # edges just inside the tile boundaries: the same tiles, with crossings along the borders
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(60 * k + 40, 200 - 50 * k, 90, 150), None,
               Rect(16.0 * x0 + 0.5 + k, 16.0 * y0 + 0.25, 16.0 * x1 - 0.75, 16.0 * y1 - 1.5 - k))
    packed = resolve(s.encoding)
    paths, tiles, bump = check_frame(renderer, oracle, packed, 1024, 1024)
    assert int(bump["tile"]) == end == len(tiles)
    assert int(bump["segments"]) > 0


@pytest.mark.gpu
def test_many_paths_per_chunk(renderer, oracle):
    """4096 one-tile squares, every one next to an off-frame (empty) path, the first and last draw objects empty: each chunk
    overlaps far more than BD_STAGE paths and searches paths[] in global memory."""
    s = Scene()
    off = Rect(-100.0, -100.0, -60.0, -60.0)
    col = Color.from_rgba8(200, 60, 120, 220)
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, col, None, off)
    for i in range(4096):
        x, y = 16.0 * (i % 64), 16.0 * (i // 64)
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, col, None, Rect(x + 2.5, y + 3.25, x + 13.0 + (i % 3), y + 12.5))
        s.fill(FILL_EVEN_ODD, Affine.IDENTITY, col, None, off)
    packed = resolve(s.encoding)
    paths, _, bump = check_frame(renderer, oracle, packed, 1024, 1024)
    n = len(paths)
    cnt = np.diff(np.append(paths["tiles"].astype(np.int64), int(bump["tile"])))
    assert n == 2 * 4096 + 1 and cnt[0] == 0 and cnt[-1] == 0
    assert max(chunk_paths(paths, int(bump["tile"]))) > BD_STAGE
    assert "unstaged" in reaches(paths, int(bump["tile"]))
