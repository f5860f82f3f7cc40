"""Helpers that compare the CUDA pipeline's buffers with the CPU oracle's.

Deterministic buffers are compared byte for byte. Buffers whose absolute offsets depend on atomic
allocation order in BOTH implementations' GPU design (bin_data chunks, seg_counts order, segment
slices, dynamic PTCL chunks) are compared after canonicalisation: through the headers / per tile,
following jumps, with per-slice segment multisets.
"""
from __future__ import annotations

import numpy as np

from oracle.vbo import DTYPES

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


STAGES = ["pathtag", "flatten", "draw", "clip", "binning", "tile_alloc", "path_count", "backdrop", "coarse", "path_tiling", "fine"]
# the stage that writes each compared buffer (info_bin_data: its info part; the bins part belongs to binning) and bump counter
BUFFER_STAGE = {"tag_monoids": "pathtag", "path_bboxes": "flatten", "lines": "flatten", "draw_monoids": "draw", "clip_inp": "draw",
                "info_bin_data": "draw", "clip_bboxes": "clip", "draw_bboxes": "binning", "bin_headers": "binning", "paths": "tile_alloc",
                "seg_counts": "path_count", "tiles": "backdrop", "ptcl": "coarse", "segments": "path_tiling"}
COUNTER_STAGE = {"lines": "flatten", "binning": "binning", "tile": "tile_alloc", "seg_counts": "path_count", "segments": "coarse",
                 "blend": "coarse"}


def compare_all(r, o, layout, width, height, check_ptcl_tiles=None, before=None):
    """Assert stage-by-stage parity of the last GPU frame (renderer r) with the oracle context o.
    Returns a dict of counters for reporting.

    With `before` (a stage name) only what the stages ahead of it wrote is compared and `failed` is not checked: the
    buffers an attempt that failed in that stage must still have computed exactly."""
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
        assert g["info_bin_data"][:bds].tobytes() == c["info_bin_data"][:bds].tobytes(), "info differs"
    if "bin_headers" in g:
        assert bins_canonical(g["bin_headers"], g["info_bin_data"], bds) == bins_canonical(c["bin_headers"], c["info_bin_data"], bds)
    # tiles: backdrop exact; the count/index word is ~seg_ix after coarse (allocation order) -> compare via PTCL
    if "tiles" in g:
        assert np.array_equal(g["tiles"]["backdrop"], c["tiles"]["backdrop"]), "tile backdrops differ"
    # crossing worklist as a multiset of (line, i)
    if "seg_counts" in g:
        gs = np.stack([g["seg_counts"]["line_ix"], g["seg_counts"]["counts"] & 0xFFFF], 1)
        cs = np.stack([c["seg_counts"]["line_ix"], c["seg_counts"]["counts"] & 0xFFFF], 1)
        assert np.array_equal(gs[np.lexsort(gs.T[::-1])], cs[np.lexsort(cs.T[::-1])]), "seg_counts multiset differs"
    # per-tile command streams (+ segment slices as multisets, once path_tiling has written them)
    if "ptcl" in g:
        n_tiles = ((width + 15) // 16) * ((height + 15) // 16)
        subset = check_ptcl_tiles
        ts_g = tile_streams(g["ptcl"], g.get("segments"), n_tiles, subset)
        ts_c = tile_streams(c["ptcl"], c.get("segments"), n_tiles, subset)
        assert ts_g == ts_c, "PTCL / segment slices differ"
    return dict(lines=int(gb["lines"]), seg_counts=int(gb["seg_counts"]), segments=int(gb["segments"]), tiles=int(gb["tile"]))
