"""k_path_count's crossing phase against the oracle's path_count, at the edges of the way it spreads crossings over a CTA.

k_path_count takes its lines 256 at a time. After the per-line setup it lays the block's crossings end to end (an
exclusive scan of each line's count) and its threads take them in strides of 256: the crossing's line by a search over the
scan, its step `i` from the offset. Each warp reserves the slots of a tile's crossings with one atomic per (warp, tile) and
hands them out in lane order. So the edges are: one line whose crossings span several strides and warps; blocks whose
crossing total is just under, at or just over one and two strides; more than 32 crossings of one tile in one warp and
across CTAs; lines without crossings between others; and lines left of their path's tile box, which only add backdrop.

Checks, after path_count alone on the GPU and on the oracle: the tiles' backdrop deltas and crossing counts are equal, the
records are the same multiset of (line, i, outside the box), and in every tile the slots of its crossings are exactly
0..count-1. The slot order within a tile depends on atomic order, so only that permutation is compared. The tile of a
record comes from `crossing_tiles`, path_count's walk restated in numpy f32; the CPU tests show that it puts the oracle's
own records in tiles whose slots and counts agree, so it is a sound check of the GPU's.
"""
import numpy as np
import pytest

from oracle.vbo import DTYPES
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Scene, resolve
from vello_b200.shapes import Affine, BezPath

from . import tile_walk_ref as ref

BLOCK = 256  # lines per CTA iteration of k_path_count
SEG_OUTSIDE = 0xFFFFFFFF
F = np.float32


# ---- path_count's walk in f32 -----------------------------------------------------------------------------------------
def _span(a, b):
    return np.maximum(np.ceil(np.maximum(a, b)) - np.floor(np.minimum(a, b)), F(1.0)).astype(np.int64)


def crossing_tiles(lines, paths, seg_counts):
    """The tile (index into the tile arena) each record's crossing falls in, computed as k_path_count's setup and walk do,
    operation by operation in f32 (no fused multiply-adds). Only meaningful for records inside their path's box."""
    p0 = lines["p0"].astype(F)
    p1 = lines["p1"].astype(F)
    down = p1[:, 1] >= p0[:, 1]
    xy0 = np.where(down[:, None], p0, p1)
    xy1 = np.where(down[:, None], p1, p0)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s0x, s0y = xy0[:, 0] * F(0.0625), xy0[:, 1] * F(0.0625)
        s1x, s1y = xy1[:, 0] * F(0.0625), xy1[:, 1] * F(0.0625)
        count_x = _span(s0x, s1x) - 1
        count = count_x + _span(s0y, s1y)
        dx = np.abs(s1x - s0x)
        dy = s1y - s0y
        idxdy = F(1.0) / (dx + dy)
        a = dx * idxdy
        pos = s1x >= s0x
        x_sign = np.where(pos, F(1.0), F(-1.0))
        xt0 = np.floor(s0x * x_sign)
        c = s0x * x_sign - xt0
        y0 = np.floor(s0y)
        ytop = np.where(s0y == s1y, np.ceil(s0y), y0 + F(1.0))
        b = np.minimum((dy * c + dx * (ytop - s0y)) * idxdy, F(0.99999994))
        err = np.floor(a * (count.astype(F) - F(1.0)) + b) - count_x.astype(F)
        a = np.where(err != 0, a - F(2e-7) * np.sign(err).astype(F), a)
        x0 = xt0 * x_sign + np.where(pos, F(0.0), F(-1.0))
        li = seg_counts["line_ix"].astype(np.int64)
        i = seg_counts["seg_within_line"].astype(F)
        z = np.floor(a[li] * i + b[li])
        y = _trunc_i32(y0[li] + i - z)
        x = _trunc_i32(x0[li] + x_sign[li] * z)
    box = paths["bbox"].astype(np.int32).astype(np.int64)[lines["path_ix"][li]]
    base = paths["tiles"].astype(np.int64)[lines["path_ix"][li]]
    return base + (y - box[:, 1]) * (box[:, 2] - box[:, 0]) + (x - box[:, 0])


def _trunc_i32(v):
    return np.clip(np.nan_to_num(np.trunc(v.astype(np.float64))), -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)


def assert_slots(lines, paths, seg_counts, counts):
    """In every tile the slots of the records that fall in it are exactly 0..count-1, and no record inside its box falls
    outside the tile arena."""
    inside = seg_counts["seg_within_slice"] != SEG_OUTSIDE
    sc = seg_counts[inside]
    tile = crossing_tiles(lines, paths, sc)
    assert ((tile >= 0) & (tile < len(counts))).all(), "a record's crossing lies outside the tile arena"
    slot = sc["seg_within_slice"].astype(np.int64)
    order = np.lexsort((slot, tile))
    tile, slot = tile[order], slot[order]
    per_tile = np.bincount(tile, minlength=len(counts))
    bad = np.nonzero(per_tile != counts.astype(np.int64))[0]
    assert len(bad) == 0, f"{len(bad)} tiles hold a number of records other than their count, first tile {int(bad[0])}: " \
                          f"{int(per_tile[bad[0]])} records, count {int(counts[bad[0]])}"
    first = np.concatenate([[0], np.cumsum(per_tile)[:-1]])
    rank = np.arange(len(tile)) - first[tile]
    bad = np.nonzero(slot != rank)[0]
    assert len(bad) == 0, f"tile {int(tile[bad[0]])}: its slots are not 0..count-1 (slot {int(slot[bad[0]])} at rank " \
                          f"{int(rank[bad[0]])}; {len(bad)} records out of place)"
    return len(sc)


# ---- scenes -------------------------------------------------------------------------------------------------------------
def _fill(s, pts, k=0):
    p = BezPath()
    p.move_to(*pts[0])
    for q in pts[1:]:
        p.line_to(*q)
    p.close_path()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(40 + 50 * (k % 4), 200 - 30 * (k % 5), 120, 255), None, p)


def _block_path(col, total):
    """256 points (so 256 lines, the closing one included) inside tile column `col`, rows 1..5, whose lines cross `total`
    tiles in all. Pieces start and end at the base point B (row 1): a 'pair' B -> row 1+d -> B crosses 2(d + 1) tiles in
    two lines; 'zero' B -> (row 2's top edge) -> along that edge -> B crosses 2 in three lines, the middle one horizontal on
    a tile edge (no crossing); 'odd' B -> row 2 -> row 2 -> B crosses 5 in three lines."""
    n_odd = total % 2
    n_zero = 2 + n_odd
    n_pair = (256 - 3 * (n_odd + n_zero)) // 2
    extra = total - (5 * n_odd + 2 * n_zero + 2 * n_pair)
    assert extra >= 0 and extra % 2 == 0, (total, extra)
    ds = np.zeros(n_pair, np.int64)
    for k in range(extra // 2):
        ds[k % n_pair] += 1
    X = 16.0 * col
    B = (X + 3.25, 16.0 + 5.5)
    pieces = [("pair", int(d)) for d in ds]
    for z in range(n_zero):  # the zero-crossing pieces between the others
        pieces.insert(1 + z * (len(pieces) // n_zero), ("zero", 0))
    pieces = [("odd", 0)] * n_odd + pieces
    pts = []
    for j, (kind, d) in enumerate(pieces):
        pts.append(B)
        if kind == "odd":
            pts += [(X + 12.5, 32.0 + 5.5), (X + 7.75, 32.0 + 10.25)]
        elif kind == "zero":
            pts += [(X + 6.0 + (j % 3), 32.0), (X + 11.5, 32.0)]
        else:
            pts.append((X + 4.0 + (j % 9), 16.0 * (1 + d) + 10.25))
    assert len(pts) == 256, len(pts)
    return pts


def _zigzag(n):
    """n lines down and up tile column 1; every one crosses tile (1, 1), and they cross 2, 2, 1, 1, 2, 2, .. tiles."""
    tops = [(20.0 + 0.25 * (k % 7), 18.5 + 0.125 * (k % 5)) for k in range(n // 2)]
    bottoms = [(27.5 - 0.25 * (k % 5), 40.25 if k % 2 == 0 else 29.75) for k in range(n // 2)]
    return [p for tb in zip(tops, bottoms) for p in tb]


def scenes():
    """(name, scene, width, height, edges it must reach)."""
    out = []
    s = Scene()
    for k in range(40):  # short lines, then a triangle of long ones in the same 256-line block, then more short ones
        x, y = 16.0 * (k % 20) + 2.5, 16.0 * (k // 20) + 300.25
        _fill(s, [(x, y), (x + 9.5, y + 3.0), (x + 4.0, y + 11.0)], k)
    _fill(s, [(1.5, 1.5), (4090.5, 3000.25), (10.25, 3050.75)], 1)
    for k in range(80):
        x, y = 16.0 * (k % 20) + 2.5, 16.0 * (k // 20) + 3500.25
        _fill(s, [(x, y), (x + 30.5, y + 17.0), (x + 4.0, y + 40.0)], k)
    out.append(("long-line", s, 4096, 4096, {"line>=300"}))

    s = Scene()
    for c, total in enumerate((255, 256, 257, 511, 512, 513)):
        _fill(s, _block_path(c, total), c)
    out.append(("block-totals", s, 128, 128, {f"block={t}" for t in (255, 256, 257, 511, 512, 513)} | {"zero-between"}))

    s = Scene()
    _fill(s, _zigzag(3000))
    out.append(("crowded-tile", s, 48, 48, {"tile>32-in-warp", "tile-across-ctas"}))

    side = next(c for c in ref.cases() if c.name == "side-left")
    out.append(("left-of-box", side.scene(), side.w, side.h, {"left-of-box"}))
    return out


SCENES = scenes()


def reached(lines, paths, seg_counts):
    """Which of the edges in the module docstring a frame's records reach."""
    tags = set()
    li = seg_counts["line_ix"].astype(np.int64)
    per_line = np.bincount(li, minlength=len(lines))
    if per_line.max() >= 300:
        tags.add("line>=300")
    for t in np.bincount(np.arange(len(lines)) // BLOCK, weights=per_line).astype(np.int64):
        tags.add(f"block={t}")
    for blk in range(0, len(lines), BLOCK):
        c = per_line[blk:blk + BLOCK]
        nz = np.nonzero(c)[0]
        if len(nz) >= 2 and (c[nz[0]:nz[-1]] == 0).any():
            tags.add("zero-between")
    # a block's records lie in line order, so a record's position in its block is its item k, taken by warp (k % 256) / 32
    order = np.lexsort((seg_counts["seg_within_line"], li))
    blk = li[order] // BLOCK
    k = np.arange(len(order)) - np.searchsorted(blk, blk)
    warp = (k % BLOCK) // 32
    inside = seg_counts["seg_within_slice"][order] != SEG_OUTSIDE
    if inside.any():
        t = crossing_tiles(lines, paths, seg_counts[order][inside])
        b, w = blk[inside], warp[inside]
        key = (b * (BLOCK // 32) + w) * (int(t.max()) + 1) + t
        if np.unique(key, return_counts=True)[1].max() > 32:
            tags.add("tile>32-in-warp")
        if max(len(np.unique(b[t == v])) for v in np.unique(t)) >= 3:
            tags.add("tile-across-ctas")
    for tags_line, _ in ref.classify(lines, paths):
        tags |= tags_line & {"left-of-box"}
    return tags


def oracle_after_path_count(oracle, packed, w, h):
    oracle.bind(packed, w, h)
    oracle.run("pathtag", "path_count")
    bump = oracle.buffer("bump")[0]
    n_draw = packed.layout.n_draw_objects
    return dict(lines=oracle.buffer("lines")[: int(bump["lines"])], paths=oracle.buffer("paths")[:n_draw],
                tiles=oracle.buffer("tiles")[: int(bump["tile"])], seg_counts=oracle.buffer("seg_counts")[: int(bump["seg_counts"])],
                bump=bump)


def gpu_after_path_count(r, packed, w, h, aa=AA_AREA):
    # a whole frame first: it grows any arena the scene overflows (run_stages does not retry)
    r.render_to_texture(packed, RenderParams(BLACK, w, h, aa))
    r.run_stages(RenderParams(BLACK, w, h, aa), "pathtag", "path_count")
    bump = r.download("bump", DTYPES["bump"])[0]
    n_draw = packed.layout.n_draw_objects
    return dict(lines=r.download("lines", DTYPES["lines"])[: int(bump["lines"])], paths=r.download("paths", DTYPES["paths"])[:n_draw],
                tiles=r.download("tiles", DTYPES["tiles"])[: int(bump["tile"])],
                seg_counts=r.download("seg_counts", DTYPES["seg_counts"])[: int(bump["seg_counts"])], bump=bump)


def _crossings(sc):
    k = np.stack([sc["line_ix"], sc["seg_within_line"], sc["seg_within_slice"] == SEG_OUTSIDE], 1).astype(np.uint32)
    return k[np.lexsort(k.T[::-1])]


# ---- CPU: the scenes and the tile restatement on the oracle -----------------------------------------------------------------
@pytest.mark.parametrize("name,scene,w,h,expect", SCENES, ids=[s[0] for s in SCENES])
def test_oracle_reaches_edges_and_slots(oracle, name, scene, w, h, expect):
    """On the oracle: the scene reaches the edges it is named for, and `crossing_tiles` puts the oracle's records in tiles
    whose slots are 0..count-1 and whose numbers of records are the oracle's counts."""
    o = oracle_after_path_count(oracle, resolve(scene.encoding), w, h)
    assert int(o["bump"]["failed"]) == 0
    got = reached(o["lines"], o["paths"], o["seg_counts"])
    assert expect <= got, (name, sorted(expect - got))
    assert assert_slots(o["lines"], o["paths"], o["seg_counts"], o["tiles"]["segment_count_or_ix"]) > 0


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,scene,w,h,expect", SCENES, ids=[s[0] for s in SCENES])
def test_gpu_path_count_matches_oracle(renderer, oracle, name, scene, w, h, expect):
    packed = resolve(scene.encoding)
    o = oracle_after_path_count(oracle, packed, w, h)
    g = gpu_after_path_count(renderer, packed, w, h)
    assert int(g["bump"]["failed"]) == 0
    assert g["lines"].tobytes() == o["lines"].tobytes()
    assert np.array_equal(g["tiles"]["backdrop"], o["tiles"]["backdrop"]), "backdrop deltas differ"
    assert np.array_equal(g["tiles"]["segment_count_or_ix"], o["tiles"]["segment_count_or_ix"]), "crossing counts differ"
    assert int(g["bump"]["seg_counts"]) == int(o["bump"]["seg_counts"])
    assert np.array_equal(_crossings(g["seg_counts"]), _crossings(o["seg_counts"])), "the (line, i, outside) multiset differs"
    assert assert_slots(g["lines"], g["paths"], g["seg_counts"], g["tiles"]["segment_count_or_ix"]) > 0
    assert expect <= reached(g["lines"], g["paths"], g["seg_counts"])


@pytest.mark.gpu
def test_gpu_bench_frame_slots(renderer):
    """The frame bench.py renders (paris-like 30k, 4096 x 4096, MSAA16): after path_count every tile's slots are exactly
    0..count-1, every line has its records i = 0, 1, .. in one run, and the records fill the worklist."""
    from vello_b200 import scenes as sc
    packed = resolve(sc.paris_like(30000, 4096, 30000).encoding)
    g = gpu_after_path_count(renderer, packed, 4096, 4096, AA_MSAA16)
    assert int(g["bump"]["failed"]) == 0
    recs = g["seg_counts"]
    assert len(recs) > 1_000_000
    n = assert_slots(g["lines"], g["paths"], recs, g["tiles"]["segment_count_or_ix"])
    assert n == int(g["tiles"]["segment_count_or_ix"].astype(np.int64).sum())
    # within each line the records are consecutive and their steps count up by one
    li = recs["line_ix"].astype(np.int64)
    i = recs["seg_within_line"].astype(np.int64)
    same = li[1:] == li[:-1]
    assert (i[1:][same] == i[:-1][same] + 1).all()
    assert len(np.unique(li)) == int((~same).sum()) + 1
