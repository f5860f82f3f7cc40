"""Helpers that compare the CUDA pipeline's buffers with the CPU oracle's.

Deterministic buffers are compared byte for byte. That includes every tile's segment slice start, which backdrop assigns
in tile order (the oracle's coarse allocates slices in its own order, so the GPU's words are compared with the oracle's
crossing counts instead). What depends on atomic order in the GPU design (bin_data chunks, seg_counts order, the order of
segments inside a slice, dynamic PTCL chunks) is compared after canonicalisation: through the headers / per tile,
following jumps, with per-slice segment multisets.
"""
from __future__ import annotations

import numpy as np

from oracle.vbo import DTYPES

from .backdrop_ref import slice_words

CMD_SIZES = {1: 4, 3: 1, 5: 2, 6: 3, 7: 3, 8: 3, 9: 2, 10: 1, 11: 3, 13: 3}


def gpu_buffers(r, names):
    return {n: r.download(n, DTYPES[n]) for n in names}


def tile_streams(ptcl: np.ndarray, segments, n_tiles: int, tiles_subset=None):
    """Per tile: list of commands with FILL's seg_ix replaced by the sorted bytes of its segment slice (by nothing when
    `segments` is None: path_tiling has not written them)."""
    out = {}
    seg_raw = segments.view(np.uint8).reshape(-1, 24) if segments is not None and segments.size else np.zeros((0, 24), np.uint8)
    rng = range(n_tiles) if tiles_subset is None else tiles_subset
    for t in rng:
        ix = t * 64
        cmds = [("blend", None)]  # blend offset is allocation-order dependent: presence only
        ix += 1
        guard = 0
        while True:
            guard += 1
            assert guard < 10_000_000
            tag = int(ptcl[ix])
            if tag == 0:
                break
            if tag == 12:
                ix = int(ptcl[ix + 1])
                continue
            if tag == 1:
                sr, seg_ix, bd = int(ptcl[ix + 1]), int(ptcl[ix + 2]), int(ptcl[ix + 3])
                n = sr >> 1
                if segments is None:
                    cmds.append((1, sr, bd))
                else:
                    sl = seg_raw[seg_ix:seg_ix + n]
                    order = np.lexsort(sl.T[::-1]) if n else np.zeros(0, int)
                    cmds.append((1, sr, bd, sl[order].tobytes()))
                ix += 4
            else:
                size = CMD_SIZES[tag]
                cmds.append((tag,) + tuple(int(v) for v in ptcl[ix + 1: ix + size]))
                ix += size
        out[t] = cmds
    return out


def bins_canonical(headers: np.ndarray, info_bin_data: np.ndarray, bin_data_start: int):
    """(partition, bin) -> tuple of draw indices."""
    res = []
    for h in headers:
        c, o = int(h["element_count"]), int(h["chunk_offset"])
        res.append(tuple(int(v) for v in info_bin_data[bin_data_start + o: bin_data_start + o + c]) if c else ())
    return res


def unpaired_endpoints(lines: np.ndarray) -> np.ndarray:
    """vello/src/debug/validate.rs:47-64 (`validate_line_soup`): end points, compared as (path_ix, x bits, y bits), that occur
    an odd number of times. Flatten's output is watertight iff none is left (every path's lines form closed loops)."""
    if lines.size == 0:
        return np.zeros((0, 3), np.uint32)
    pts = np.concatenate([
        np.stack([lines["path_ix"], np.ascontiguousarray(lines["p0"][:, 0]).view(np.uint32), np.ascontiguousarray(lines["p0"][:, 1]).view(np.uint32)], 1),
        np.stack([lines["path_ix"], np.ascontiguousarray(lines["p1"][:, 0]).view(np.uint32), np.ascontiguousarray(lines["p1"][:, 1]).view(np.uint32)], 1)])
    u, c = np.unique(pts, axis=0, return_counts=True)
    return u[c % 2 == 1]


def replay_fine(r, o, packed, w, h, aa, base, window=None):
    """The oracle's `fine` run on the buffers the GPU's `fine` read in the last frame of renderer r: its `ptcl`, `segments`
    and `info_bin_data`, with the blend spill sized by the GPU's `bump.blend` (the blend offsets in that ptcl were allocated
    against it). Returns the oracle's image (h, w, 4); with a bin-row `window` only that window's rows are painted.

    The GPU's image must equal it byte for byte in every AA mode: the two interpreters then see the same commands and the
    same segments in the same order, so even area AA's float sums agree (both sides are built without FMA contraction).
    The GPU's fine starts a tile at its occlusion start and walks coarse's cost-ordered tile queue; the oracle starts every
    tile at its head, so equality also pins the occlusion start."""
    g = gpu_buffers(r, ["ptcl", "segments", "info_bin_data", "bump"])
    bump = g["bump"][0]
    assert int(bump["failed"]) == 0, "the last GPU frame failed: fine painted nothing"
    base_u32 = base if isinstance(base, int) else base.premul_rgba8_u32()
    o.bind(packed, w, h, base_u32, aa, window or (0, 0))
    for n in ("ptcl", "segments", "info_bin_data"):
        o.set_buffer(n, g[n])
    o.set_buffer("blend_spill", np.zeros(int(bump["blend"]), np.uint32))
    return o.run("fine", "fine")


def assert_replay(r, o, packed, img, w, h, aa, base, window=None):
    """`img`, the last frame of renderer r (the window's rows only, for a bin-row window), equals replay_fine's image."""
    want = replay_fine(r, o, packed, w, h, aa, base, window)
    if window:
        want = want[min(window[0] * 256, h):min(window[1] * 256, h)]
    assert img.shape == want.shape, (img.shape, want.shape)
    bad = (img != want).any(axis=2)
    assert not bad.any(), f"aa={aa}: {int(bad.sum())} pixels differ from the oracle's fine on the GPU's own buffers, first at " \
                          f"{tuple(int(v) for v in np.argwhere(bad)[0])}"


STAGES = ["pathtag", "flatten", "draw", "clip", "binning", "tile_alloc", "path_count", "backdrop", "coarse", "path_tiling", "fine"]
# the stage that writes each compared buffer (info_bin_data: its info part; the bins part belongs to binning) and bump counter
BUFFER_STAGE = {"tag_monoids": "pathtag", "path_bboxes": "flatten", "lines": "flatten", "draw_monoids": "draw", "clip_inp": "draw",
                "info_bin_data": "draw", "clip_bboxes": "clip", "draw_bboxes": "binning", "bin_headers": "binning", "paths": "tile_alloc",
                "seg_counts": "path_count", "tiles": "backdrop", "ptcl": "coarse", "segments": "path_tiling"}
COUNTER_STAGE = {"lines": "flatten", "binning": "binning", "tile": "tile_alloc", "seg_counts": "path_count", "segments": "coarse",
                 "blend": "coarse"}


def compare_all(r, o, layout, width, height, check_ptcl_tiles=None, before=None, info_nan=False):
    """Assert stage-by-stage parity of the last GPU frame (renderer r) with the oracle context o.
    Returns a dict of counters for reporting.

    With `before` (a stage name) only what the stages ahead of it wrote is compared and `failed` is not checked: the
    buffers an attempt that failed in that stage must still have computed exactly. With `info_nan`, info words that hold a
    NaN on both sides compare equal whatever their payload (degenerate paints, where draw_leaf divides 0 by 0 and the GPU
    and the host compiler produce different NaNs); every other word, and every other buffer, still compares exactly."""
    stop = STAGES.index(before) if before else len(STAGES)
    ran = set(STAGES[:stop])
    names = [n for n, s in BUFFER_STAGE.items() if s in ran]
    g = gpu_buffers(r, names + ["bump"])
    c = {n: o.buffer(n) for n in g}
    gb, cb = g["bump"][0], c["bump"][0]
    if before is None:
        assert int(gb["failed"]) == 0
    # coarse reserves segment slices per 256-draw chunk; slots of fills it then skips (zero-coverage clips) stay unused
    holes = int(r.download("seg_holes", np.uint32)[0])
    for f, s in COUNTER_STAGE.items():
        if s not in ran:
            continue
        have = int(gb[f]) - (holes if f == "segments" else 0)
        assert have == int(cb[f]), (f, have, int(cb[f]))
    # exact, order included
    for n in ("tag_monoids", "path_bboxes", "lines", "draw_monoids", "clip_inp", "clip_bboxes", "draw_bboxes", "paths"):
        if n not in g:
            continue
        a, b = g[n], c[n][: g[n].shape[0]] if n == "paths" else c[n]
        assert a.shape == b.shape, (n, a.shape, b.shape)
        assert a.tobytes() == b.tobytes(), f"{n} differs"
    if "lines" in g:
        assert len(unpaired_endpoints(g["lines"])) == 0, "flatten output is not watertight (debug/validate.rs)"
    bds = layout.bin_data_start
    if "info_bin_data" in g:
        gi, ci = g["info_bin_data"][:bds], c["info_bin_data"][:bds]
        if info_nan:
            nan = np.isnan(gi.view(np.float32)) & np.isnan(ci.view(np.float32))
            gi, ci = np.where(nan, 0, gi), np.where(nan, 0, ci)
        assert gi.tobytes() == ci.tobytes(), "info differs"
    if "bin_headers" in g:
        assert bins_canonical(g["bin_headers"], g["info_bin_data"], bds) == bins_canonical(c["bin_headers"], c["info_bin_data"], bds)
    # tiles: backdrop exact, and every tile's word is ~(the first slot of its slice): the exclusive sum of the crossing counts
    # path_count left in the tiles before it, in u32. The oracle's coarse overwrites its own words in allocation order, so the
    # GPU's are compared with the oracle's counts. This pins every count too (a tile's count is the next word's start minus its
    # own), also for the tiles coarse turns into no CMD_FILL, and bump.segments is their total.
    if "tiles" in g:
        assert np.array_equal(g["tiles"]["backdrop"], c["tiles"]["backdrop"]), "tile backdrops differ"
        counts = o.buffer("tile_counts")
        assert counts.shape == g["tiles"].shape, ("tile_counts: run the oracle's path_count on this scene", counts.shape, g["tiles"].shape)
        want = slice_words(counts)
        bad = np.nonzero(g["tiles"]["segment_count_or_ix"] != want)[0]
        assert len(bad) == 0, f"{len(bad)} of {len(want)} tile slice words differ from the oracle's counts, first at tile {int(bad[0])}"
        total = int(counts.astype(np.uint64).sum() & 0xFFFFFFFF)
        assert int(gb["segments"]) == total, ("bump.segments is not the total of the crossing counts", int(gb["segments"]), total)
    # crossing worklist as a multiset of (line, i, outside the path's tile box); the slot in the slice is atomic-order dependent
    if "seg_counts" in g:
        def crossings(sc):
            return np.stack([sc["line_ix"], sc["seg_within_line"], sc["seg_within_slice"] == 0xFFFFFFFF], 1).astype(np.uint32)
        gs, cs = crossings(g["seg_counts"]), crossings(c["seg_counts"])
        assert np.array_equal(gs[np.lexsort(gs.T[::-1])], cs[np.lexsort(cs.T[::-1])]), "seg_counts multiset differs"
    # per-tile command streams (+ segment slices as multisets, once path_tiling has written them)
    if "ptcl" in g:
        n_tiles = ((width + 15) // 16) * ((height + 15) // 16)
        subset = check_ptcl_tiles
        ts_g = tile_streams(g["ptcl"], g.get("segments"), n_tiles, subset)
        ts_c = tile_streams(c["ptcl"], c.get("segments"), n_tiles, subset)
        assert ts_g == ts_c, "PTCL / segment slices differ"
    return dict(lines=int(gb["lines"]), seg_counts=int(gb["seg_counts"]), segments=int(gb["segments"]), tiles=int(gb["tile"]))
