"""What vb_hit_test answers, stated from geometry rather than from the kernel's arithmetic.

For a point (x, y) of a frame the answer is the index of the last draw object in draw order that covers it, or -1:

* A draw covers the point when the winding number of its path's lines (the frame's own `lines`, so flatten's output under
  the frame's view) at the point is nonzero, or odd when the draw's flags (info word bit 0) say even-odd. The winding
  number is `tile_walk_ref._winding_and_near`'s: float64 on the f32 end points, a line counting when it crosses the
  point's row left of the point.
* The point must also lie inside the clip path of every enclosing BEGIN_CLIP, each with its own fill rule. The nesting
  comes from the draw tags: a BEGIN_CLIP that does not cover the point hides everything up to its END_CLIP.
* BEGIN_CLIP / END_CLIP / NOP objects are never answers. Points outside the frame and NaN points answer -1.
* A point within `line_tolerance` of a line of any draw it evaluates (every draw outside a hidden clip range, clips
  included) is *ambiguous*: there the tile walk's f32 clipping may decide either way.

In a batch the frame is the tall [n_cells * H, W] one: a point of cell c is tested at y - c * H against the draws
cell_draw[c] .. cell_draw[c + 1] only.
"""
from __future__ import annotations

import numpy as np

from .tile_walk_ref import _winding_and_near, line_tolerance

DRAWTAG_NOP = 0
DRAWTAG_BEGIN_CLIP = 0x49
DRAWTAG_END_CLIP = 0x21


def frame_from_oracle(o, packed):
    """The buffers hit testing reads, from the oracle after a full render of `packed`."""
    bump = o.buffer("bump")[0]
    return _frame(o.buffer("lines")[: int(bump["lines"])], o.buffer("draw_monoids"), o.buffer("info_bin_data"), packed)


def frame_from_gpu(r, packed):
    """The same from a renderer after a frame (vb_debug_download)."""
    from oracle.vbo import DTYPES
    bump = r.download("bump", DTYPES["bump"])[0]
    return _frame(r.download("lines", DTYPES["lines"])[: int(bump["lines"])], r.download("draw_monoids", DTYPES["draw_monoids"]),
                  r.download("info_bin_data", DTYPES["info_bin_data"]), packed)


def _frame(lines, draw_monoids, info, packed):
    L = packed.layout
    n = int(L.n_draw_objects)
    dm = draw_monoids[:n]
    tags = np.asarray(packed.scene, np.uint32)[int(L.draw_tag_base): int(L.draw_tag_base) + n].astype(np.int64)
    even_odd = (np.asarray(info, np.uint32)[dm["info_offset"].astype(np.int64)] & 1).astype(bool) if n else np.zeros(0, bool)
    order = np.argsort(lines["path_ix"], kind="stable")
    ln = lines[order]
    return dict(tags=tags, path_ix=dm["path_ix"].astype(np.int64), even_odd=even_odd, lines_path=ln["path_ix"].astype(np.int64),
                p0=ln["p0"].astype(np.float64), p1=ln["p1"].astype(np.float64))


def _cover(frame, d, sx, sy, order_y, sorted_y):
    """For the points (sx, sy) (order_y sorts them by y; sorted_y = sy[order_y]): the covered mask of draw d's path and the
    near-a-line mask. Only points within the y range of the path's lines and right of their left end can be covered or
    near one; the rest are skipped without arithmetic."""
    n = len(sx)
    cov, near = np.zeros(n, bool), np.zeros(n, bool)
    pi = frame["path_ix"][d]
    lo, hi = np.searchsorted(frame["lines_path"], [pi, pi + 1])
    if hi <= lo:
        return cov, near
    p0, p1 = frame["p0"][lo:hi], frame["p1"][lo:hi]
    tol = float(line_tolerance(p0, p1).max())
    y0 = min(p0[:, 1].min(), p1[:, 1].min()) - tol
    y1 = max(p0[:, 1].max(), p1[:, 1].max()) + tol
    x0 = min(p0[:, 0].min(), p1[:, 0].min()) - tol
    cand = order_y[np.searchsorted(sorted_y, y0, side="left"): np.searchsorted(sorted_y, y1, side="right")]
    cand = cand[sx[cand] >= x0]
    if len(cand) == 0:
        return cov, near
    w, nr = _winding_and_near(p0, p1, sx[cand], sy[cand])
    cov[cand] = (w & 1) != 0 if frame["even_odd"][d] else w != 0
    near[cand] = nr
    return cov, near


def hit_ref(frame, xy, width, height, cell_draw=None):
    """(answers int32 (n,), ambiguous bool (n,)) for the points xy ((n, 2) f32) of a width x height frame, or of a batch of
    len(cell_draw) - 1 such frames stacked (cell_draw: the draw-object offsets of the cells)."""
    xy = np.asarray(xy, np.float32).astype(np.float64).reshape(-1, 2)
    n_draw = len(frame["tags"])
    cells = [0, n_draw] if cell_draw is None else [int(v) for v in cell_draw]
    n_cells = len(cells) - 1
    out = np.full(len(xy), -1, np.int32)
    amb = np.zeros(len(xy), bool)
    x, y = xy[:, 0], xy[:, 1]
    with np.errstate(invalid="ignore"):
        inside = (x >= 0) & (y >= 0) & (x < width) & (y < n_cells * height)
    cell = np.where(inside, np.floor(np.where(inside, y, 0) / height), -1).astype(np.int64)
    for c in range(n_cells):
        sel = np.nonzero(cell == c)[0]
        if len(sel) == 0:
            continue
        sx, sy = x[sel], y[sel] - c * height
        order_y = np.argsort(sy, kind="stable")
        sorted_y = sy[order_y]
        best = np.full(len(sel), -1, np.int64)
        near_any = np.zeros(len(sel), bool)
        clip_zero = np.zeros(len(sel), np.int64)  # 0: every enclosing clip covers the point; else the depth of the first that does not
        depth = 0
        for d in range(cells[c], cells[c + 1]):
            tag = int(frame["tags"][d])
            if tag == DRAWTAG_NOP:
                continue
            if tag == DRAWTAG_END_CLIP:
                clip_zero[clip_zero == depth] = 0
                depth -= 1
                continue
            active = clip_zero == 0
            if not active.any():
                if tag == DRAWTAG_BEGIN_CLIP:
                    depth += 1
                continue
            cov, near = _cover(frame, d, sx, sy, order_y, sorted_y)
            near_any |= near & active
            if tag == DRAWTAG_BEGIN_CLIP:
                depth += 1
                clip_zero[active & ~cov] = depth
            else:
                best[active & cov] = d
        out[sel] = best
        amb[sel] = near_any
    return out, amb
