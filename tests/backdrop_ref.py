"""A serial statement of what backdrop computes over the tile arena, vectorised with numpy.

tile_alloc lays the rows of all paths end to end in draw order, and path_count leaves in every tile its backdrop delta
(`backdrop`) and its crossing count (`segment_count_or_ix`). backdrop then gives tile t:
- its path: the last path whose first tile (`Path.tiles`) is <= t (an empty path shares its successor's start);
- its column: (t - that start) % max(bbox[2] - bbox[0], 1);
- its backdrop: the deltas of its row summed from the row's first tile through t, in 32-bit wrapping arithmetic;
- its word: ~(the counts of all tiles before it, summed mod 2^32), the first slot of its segment slice.
The total of all counts is bump.segments. Also the crafted arenas the GPU tests feed backdrop, and what each one reaches.
"""
from __future__ import annotations

import numpy as np

from oracle.vbo import DTYPES

M32 = (1 << 32) - 1
BD_CHUNK = 4096      # tiles per backdrop CTA (k_tile.cu)
BD_PER_THREAD = 16   # consecutive tiles per thread
BD_WARP_TILES = 32 * BD_PER_THREAD
BD_STAGE = 256       # paths a chunk stages in shared memory; a chunk over more searches paths[] in global memory


def slice_words(counts: np.ndarray) -> np.ndarray:
    """~(exclusive sum of counts) per tile, u32."""
    c = np.asarray(counts, dtype=np.uint64)
    excl = (np.cumsum(c) - c) & M32
    return (~excl.astype(np.uint32)).astype(np.uint32)


def row_layout(paths: np.ndarray, arena_end: int):
    """(owner path, column, row start) of every tile in [0, arena_end)."""
    starts = paths["tiles"].astype(np.int64)
    assert len(starts) == 0 or starts[0] == 0, "the first path starts at tile 0"
    assert np.all(np.diff(starts) >= 0), "Path.tiles is monotone in draw order"
    t = np.arange(arena_end, dtype=np.int64)
    owner = np.searchsorted(starts, t, side="right") - 1
    width = np.maximum((paths["bbox"][:, 2].astype(np.int64) - paths["bbox"][:, 0].astype(np.int64)) & M32, 1)
    col = (t - starts[owner]) % width[owner] if arena_end else t
    return owner, col, col == 0


def backdrop_ref(paths: np.ndarray, tiles: np.ndarray, arena_end: int):
    """The tiles after backdrop, and bump.segments. `tiles` as path_count leaves them (counts in segment_count_or_ix)."""
    tiles = tiles[:arena_end]
    _, _, start = row_layout(paths, arena_end)
    delta = tiles["backdrop"].astype(np.int64)
    cs = np.cumsum(delta)
    idx = np.arange(arena_end)
    last_start = np.maximum.accumulate(np.where(start, idx, 0)) if arena_end else idx
    before_row = cs[last_start] - delta[last_start]  # the sum of everything ahead of the row's first tile
    out = np.zeros(arena_end, DTYPES["tiles"])
    out["backdrop"] = ((cs - before_row) & M32).astype(np.uint32).view(np.int32)
    counts = tiles["segment_count_or_ix"]
    out["segment_count_or_ix"] = slice_words(counts)
    return out, int(counts.astype(np.uint64).sum() & M32)


# ---- crafted arenas -----------------------------------------------------------------------------------------------------
class Case:
    """A crafted arena: paths (one record per draw object) and tiles as path_count would leave them. `expect` names the edges
    it is built to reach (see `reaches`)."""

    def __init__(self, name, shapes, seed, values="small", expect=()):
        self.name = name
        self.shapes = shapes  # (width, height) per path; width * height tiles each
        self.arena_end = sum(w * h for w, h in shapes)
        self.seed = seed
        self.values = values
        self.expect = set(expect)

    def build(self):
        n = len(self.shapes)
        w = np.array([s[0] for s in self.shapes], np.int64)
        h = np.array([s[1] for s in self.shapes], np.int64)
        count = w * h
        paths = np.zeros(n, DTYPES["paths"])
        paths["tiles"] = (np.cumsum(count) - count).astype(np.uint32)
        x0 = (np.arange(n) * 7) % 50  # the column is relative to bbox[0]
        paths["bbox"][:, 0] = x0
        paths["bbox"][:, 1] = 3
        paths["bbox"][:, 2] = x0 + w
        paths["bbox"][:, 3] = 3 + h
        rng = np.random.default_rng(self.seed)
        m = self.arena_end
        tiles = np.zeros(m, DTYPES["tiles"])
        if self.values == "small":
            tiles["backdrop"] = rng.integers(-4, 5, m)
            c = np.where(rng.random(m) < 0.7, 0, rng.integers(1, 40, m))
        else:  # magnitudes near +-2^30, so that a narrowed accumulator shows; counts up to 2^20 whose total wraps u32
            big = rng.integers((1 << 30) - 4096, (1 << 30) + 4096, m) * rng.choice([-1, 1], m)
            tiles["backdrop"] = np.where(rng.random(m) < 0.5, big, rng.integers(-4, 5, m)).astype(np.int32)
            c = np.where(rng.random(m) < 0.9, 0, rng.integers(1, 1 << 20, m))
            c[rng.integers(0, m, min(m, 8))] = 1 << 20
        tiles["segment_count_or_ix"] = c.astype(np.uint32)
        return paths, tiles

    def __repr__(self):
        return self.name


def _gap(n):
    """Paths over n tiles with one row start, at their first tile, where a frame allows it (rows of at most 4096 tiles):
    one row of n tiles, or rows of 4096 (whose starts keep the first one's residue mod 4096) and one of the rest."""
    if n <= 0:
        return []
    if n <= BD_CHUNK:
        return [(n, 1)]
    return [(BD_CHUNK, n // BD_CHUNK)] + ([(n % BD_CHUNK, 1)] if n % BD_CHUNK else [])


SEAMS = [(16, 0), (16, 1), (16, 15), (512, 511), (512, 0), (4096, 4095), (4096, 0)]


def _seams(width):
    """For each (m, r) of SEAMS, a path of `width` and two rows whose first row starts at a tile offset = r (mod m)."""
    shapes, pos = [], 0
    for m, r in SEAMS:
        o = pos + ((r - pos) % m)
        if o == 0:
            o = m
        shapes += _gap(o - pos) + [(width, 2)]
        pos = o + 2 * width
    return shapes + _gap(37)


def cases():
    out = []
    # arena ends: chunk, warp and thread multiples and one either side (the int2 loads and stores of an odd end)
    for k, end in enumerate([1, 2, 15, 16, 17, 511, 512, 513, 4095, 4096, 4097, 8191, 8192, 8193, 3 * 4096 + 4095]):
        shapes = [(min(37, end), 1)] + _gap(end - min(37, end))
        out.append(Case(f"end-{end}", shapes, seed=k, expect={f"end%16={end % 16}", f"end%4096={end % 4096}"}))
    out.append(Case("end-0", [(3, 0), (0, 5), (7, 0)], seed=99, expect={"empty"}))  # draw objects, no tiles
    # row starts at thread (16), warp (512) and chunk (4096) seams, for every width
    for k, width in enumerate([1, 2, 15, 16, 17, 511, 512, 513, 4095, 4096]):
        expect = {f"start%{m}={r}" for m, r in SEAMS} | ({"row-spans-chunk"} if width > 1 else set())
        if width > 1024:
            expect.add("warp-no-start")
        out.append(Case(f"seams-w{width}", _seams(width), seed=100 + k, expect=expect))
    # many paths per chunk: more than BD_STAGE overlap one chunk, so the chunk searches paths[] in global memory
    out.append(Case("one-tile-4096", [(1, 1)] * 4096, seed=200, expect={"unstaged"}))
    rng = np.random.default_rng(201)
    shapes = [(0, 0)] * 10000
    for i in sorted(rng.choice(np.arange(1, 9999), 300, replace=False)):
        shapes[i] = (int(rng.integers(1, 40)), int(rng.integers(1, 4)))
    out.append(Case("300-among-10000-empty", shapes, seed=202, expect={"unstaged", "empty-first", "empty-last"}))
    # an empty first path, runs of empty paths at a chunk's last (4095) and first (8192) tile, trailing empty paths
    shapes = [(0, 3)] + [(1, 1)] * 4095 + [(0, 0)] * 400 + [(5, 1)] + [(1, 1)] * 4092 + [(0, 2)] * 300 + [(1, 1)] + [(3, 3)] * 50 + [(0, 0)] * 40
    out.append(Case("empty-runs-at-chunk-edges", shapes, seed=203,
                    expect={"unstaged", "empty-first", "empty-last", "empty-at-chunk-first", "empty-at-chunk-last"}))
    # large arena: over 1000 chunks, so that look-backs span more than one 32-chunk window
    rng = np.random.default_rng(204)
    shapes, total = [], 0
    while total < 1000 * BD_CHUNK + 123:
        w, h = int(rng.choice([1, 3, 16, 100, 511, 513, 2000, 4096])), int(rng.integers(1, 12))
        shapes.append((w, h))
        total += w * h
    out.append(Case("large-1000-chunks", shapes, seed=205, expect={"1000-chunks"}))
    out.append(Case("large-1000-chunks-big-values", shapes, seed=206, values="big", expect={"1000-chunks"}))
    # rows no real frame has (a frame is at most 65536 px = 4096 tiles wide): the only inputs that give a chunk no row start,
    # and so drive the chunk-level carry with f = 0 through the real kernel
    out.append(Case("rows-5000-synthetic", [(3596, 1), (5000, 4), (3, 1)], seed=300, expect={"chunk-no-start", "warp-no-start"}))
    out.append(Case("rows-10000-synthetic", [(1, 100), (10000, 3), (4096, 2)], seed=301, values="big",
                    expect={"chunk-no-start", "warp-no-start"}))
    out.append(Case("big-values-4097", [(4097, 1), (1, 5)], seed=302, values="big", expect={"warp-no-start"}))
    return out


def chunk_paths(paths: np.ndarray, arena_end: int):
    """Per chunk: the number of paths it overlaps, as k_backdrop counts them (the first to the last path of its tiles)."""
    starts = paths["tiles"].astype(np.int64)
    res = []
    for c0 in range(0, arena_end, BD_CHUNK):
        c1 = min(c0 + BD_CHUNK, arena_end) - 1
        p0 = np.searchsorted(starts, c0, side="right") - 1
        p1 = np.searchsorted(starts, c1, side="right") - 1
        res.append(int(p1 - p0 + 1))
    return res


def reaches(paths: np.ndarray, arena_end: int) -> set:
    """The edges an arena reaches, by name (see `cases`)."""
    got = set()
    if arena_end == 0:
        return {"empty"}
    got.add(f"end%16={arena_end % 16}")
    got.add(f"end%4096={arena_end % 4096}")
    _, _, start = row_layout(paths, arena_end)
    s = np.nonzero(start)[0]
    for m, r in ((16, 0), (16, 1), (16, 15), (512, 511), (512, 0), (4096, 4095), (4096, 0)):
        if np.any((s % m == r) & (s > 0)):
            got.add(f"start%{m}={r}")
    # a row that spans a chunk boundary: a chunk whose first tile is not a row start
    if any(not start[c0] for c0 in range(BD_CHUNK, arena_end, BD_CHUNK)):
        got.add("row-spans-chunk")
    # a warp's 512 tiles with no row start, and a chunk with none
    for span, tag in ((BD_WARP_TILES, "warp-no-start"), (BD_CHUNK, "chunk-no-start")):
        n_full = arena_end // span
        if n_full and np.any(start[: n_full * span].reshape(n_full, span).sum(axis=1) == 0):
            got.add(tag)
    per_chunk = chunk_paths(paths, arena_end)
    if max(per_chunk) > BD_STAGE:
        got.add("unstaged")
    if len(per_chunk) >= 1000:
        got.add("1000-chunks")
    n = len(paths)
    cnt = np.diff(np.append(paths["tiles"].astype(np.int64), arena_end))
    if n and cnt[0] == 0:
        got.add("empty-first")
    if n and cnt[-1] == 0:
        got.add("empty-last")
    empty_starts = set(int(v) for v in paths["tiles"][cnt == 0])
    if any(v % BD_CHUNK == 0 and v > 0 for v in empty_starts):
        got.add("empty-at-chunk-first")
    if any(v % BD_CHUNK == BD_CHUNK - 1 for v in empty_starts):
        got.add("empty-at-chunk-last")
    return got
