"""Serial reference of the upload diff (vb_set_upload_diff, k_upload_diff.cu): the key of every draw object of a packed scene,
the order-preserving matching of two key lists by common prefix, common suffix and position, and the damaged tiles it gives
with the two frames' clipped draw boxes (k_recompose_damage's rule, one draw object per instance)."""
import numpy as np

from vello_b200.encoding import (DRAWTAG_IMAGE, DRAWTAG_LINEAR_GRADIENT, DRAWTAG_RADIAL_GRADIENT, DRAWTAG_SWEEP_GRADIENT, TAG_PATH,
                                 TAG_STYLE, TAG_TRANSFORM)

NONE = 0xFFFFFFFF
GRADIENTS = (DRAWTAG_LINEAR_GRADIENT, DRAWTAG_RADIAL_GRADIENT, DRAWTAG_SWEEP_GRADIENT)


class _Unequal:
    """A key part that equals nothing, itself included (a ramp row or atlas rectangle outside its buffer)."""

    def __eq__(self, other):
        return False

    def __hash__(self):
        return id(self)


def records(scene, layout):
    """Per draw object: (tag0, tag1, pd0, pd1, t0, t1, s0, s1, draw tag, draw-data offset), as VbUdRec."""
    L = layout
    scene = np.asarray(scene, dtype=np.uint32)
    tags = scene[L.path_tag_base:L.path_data_base].view(np.uint8).astype(np.int64)
    seg = tags & 3
    n_points = seg + ((tags >> 2) & 1)
    off_inc = np.where(tags & 8, 2 * n_points, n_points)
    ex = lambda v: np.concatenate([[0], np.cumsum(v)])  # exclusive prefix at every byte, and the total
    trans, off, style = ex((tags & TAG_TRANSFORM) != 0), ex(off_inc), ex(2 * ((tags & TAG_STYLE) != 0))
    ends = np.flatnonzero(tags & TAG_PATH)
    dt = scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects].astype(np.int64)
    path_ix = ex(dt != 0)[:-1]
    dd = ex((dt >> 2) & 7)[:-1]
    out = []
    for i in range(L.n_draw_objects):
        if dt[i] == 0:
            out.append((0, 0, 0, 0, 0, 0, 0, 0, int(dt[i]), int(dd[i])))
            continue
        p = int(path_ix[i])
        b = int(ends[p])
        a = int(ends[p - 1]) + 1 if p else 0
        t0 = max(int(trans[a]), 1) - 1
        s0 = max(int(style[a]), 2) - 2
        out.append((a, b + 1, int(off[a]), int(off[b + 1]), t0, max(int(trans[b]), t0), s0, max(int(style[b]), s0), int(dt[i]), int(dd[i])))
    return out


def keys(scene, layout, ramps, atlas):
    """One hashable key per draw object: equal keys <=> eq() of k_upload_diff.cu. `ramps` is (n, 512) u32, `atlas` (h, w, 4)
    u8 (None: the scene draws no image)."""
    L = layout
    scene = np.asarray(scene, dtype=np.uint32)
    tag_bytes = scene[L.path_tag_base:L.path_data_base].view(np.uint8)
    ramps = np.asarray(ramps, dtype=np.uint32).reshape(-1, 512)
    out = []
    for (tag0, tag1, pd0, pd1, t0, t1, s0, s1, dtag, dd) in records(scene, L):
        words = scene[L.draw_data_base + dd:L.draw_data_base + dd + ((dtag >> 2) & 7)].copy()
        extra = b""
        if dtag in GRADIENTS:
            row = int(words[0]) >> 2
            words[0] &= 3
            extra = ramps[row].tobytes() if row < ramps.shape[0] else _Unequal()
        elif dtag == DRAWTAG_IMAGE:
            if atlas is None:
                raise ValueError("an image needs the atlas")
            x, y, w, h = int(words[0]) >> 16, int(words[0]) & 0xFFFF, int(words[1]) >> 16, int(words[1]) & 0xFFFF
            extra = atlas[y:y + h, x:x + w].tobytes() if x + w <= atlas.shape[1] and y + h <= atlas.shape[0] else _Unequal()
        out.append((dtag, words.tobytes(), extra, tag_bytes[tag0:tag1].tobytes(), scene[L.path_data_base + pd0:L.path_data_base + pd1].tobytes(),
                    scene[L.transform_base + 6 * t0:L.transform_base + 6 * t1].tobytes(), scene[L.style_base + s0:L.style_base + s1].tobytes()))
    return out


def match(old, new, eq=None):
    """(map, unmatched): map[j] = the old index new j is paired with, or NONE; unmatched[i] for every old i. The common prefix
    p, the common suffix s capped at m - p, and the middle by position."""
    eq = eq or (lambda i, j: old[i] == new[j])
    n_o, n_n = len(old), len(new)
    m = min(n_o, n_n)
    p = 0
    while p < m and eq(p, p):
        p += 1
    s = 0
    if n_o != n_n:
        while s < m - p and eq(n_o - 1 - s, n_n - 1 - s):
            s += 1
    mp = np.full(n_n, NONE, dtype=np.int64)
    for j in range(n_n):
        if j < p:
            mp[j] = j
        elif j >= n_n - s:
            mp[j] = j + n_o - n_n
        elif j < m - s and eq(j, j):
            mp[j] = j
    unmatched = np.ones(n_o, dtype=bool)
    unmatched[mp[mp != NONE]] = False
    return mp, unmatched


def _or_box(mask, box):
    x0, y0, x1, y1 = (np.float32(v) for v in box)
    if not (x0 < x1 and y0 < y1):
        return
    ht, wt = mask.shape
    S = np.float32(1.0 / 16.0)

    def t(v, f, hi):
        v = f(v * S)
        return int(min(max(v, -1.0), hi + 1.0)) if np.isfinite(v) else (hi if v > 0 else 0)

    tx0, tx1 = min(max(t(x0, np.floor, wt), 0), wt), min(max(t(x1, np.ceil, wt), 0), wt)
    ty0, ty1 = min(max(t(y0, np.floor, ht), 0), ht), min(max(t(y1, np.ceil, ht), 0), ht)
    mask[ty0:ty1, tx0:tx1] = True


def damage(old_keys, new_keys, old_boxes, new_boxes, width, height):
    """The damaged tiles of the frame after the upload: bool [tiles_h, tiles_w]."""
    mp, unmatched = match(old_keys, new_keys)
    mask = np.zeros(((height + 15) // 16, (width + 15) // 16), dtype=bool)
    ob = np.asarray(old_boxes, dtype=np.float32).reshape(-1, 4)
    nb = np.asarray(new_boxes, dtype=np.float32).reshape(-1, 4)
    for j, i in enumerate(mp):
        if i == NONE:
            _or_box(mask, nb[j])
        elif not np.array_equal(ob[i].view(np.uint32), nb[j].view(np.uint32)):
            _or_box(mask, ob[i])
            _or_box(mask, nb[j])
    for i in np.flatnonzero(unmatched):
        _or_box(mask, ob[i])
    return mask
