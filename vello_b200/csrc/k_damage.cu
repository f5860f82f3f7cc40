// k_damage.cu -- damage tracking: which tiles a frame must paint again when it goes into the destination of the last
// successful frame (vb_set_damage_tracking).
//
// A tile's pixels depend only on the draw objects whose tile box covers it, and every stage is deterministic, so a tile that
// no changed draw object touches gets the same pixels again. The damage of a frame is
//   the caller's rectangles (vb_add_damage, staged into `pending` in stream order)
//   + for every bound instance whose transform words (the ones flatten reads: the bound region, or the viewed one) differ bit
//     for bit from the last successful frame's, the tile boxes of its draw objects in that frame and in this one
//   + for every draw object with a bound colour (vb_bind_draw_colors) whose colour word (the one coarse reads from the frame's
//     draw data) differs bit for bit from the last successful frame's, its tile box in that frame and in this one
//   + for every path with a bound point (vb_bind_path_points) whose two words (the ones flatten reads from the frame's path
//     data) differ bit for bit from the last successful frame's, the tile box of its draw object (path i is draw object i) in
//     that frame and in this one. A changed clip path is covered by its BEGIN_CLIP's boxes, as a moved clip is below
//   + for every bound gradient (vb_bind_gradient_stops) whose ramp row (the 512 texels fine reads) differs bit for bit from the
//     last successful frame's, the tile box of its draw object in that frame and in this one
//   + with bound transforms (vb_bind_transforms), for every path one of whose transforms [t_lo, t_hi] (the binding's range: from
//     the one in effect at its first segment to the one at its TAG_PATH, where draw reads its brush) differs bit for bit from
//     the last successful frame's, the tile box of its draw object in that frame and in this one
//   + with bound visibility (vb_bind_draw_visibility), for every draw object whose bit of the frame's mask (the one flatten
//     reads) differs from the last successful frame's, its tile box in that frame and in this one. A hidden draw object's box
//     is empty, so the union is the box it has while shown; a hidden layer is covered by its BEGIN_CLIP's box, which holds
//     every box inside the layer and the pixels its blend touches
//   + with bound stroke widths (vb_bind_stroke_widths), for every draw object below the bound count whose width (the one
//     flatten used: its snapshot entry, or for an entry of 0 its style's width word) differs bit for bit from the last successful
//     frame's, its tile box in that frame and in this one. A fill's entry is always 0 and its style word never changes, so its
//     row is no change; neither is a row that falls back to an unchanged encoded width. A wider stroke's new box holds it
//   + with bound opacity (vb_bind_draw_opacity), for every draw object below the bound count whose opacity word (the one
//     coarse and fine read from the frame's draw data: a layer's alpha word, an image's sample word) differs bit for bit from the
//     last successful frame's, its tile box in that frame and in this one. A clip layer's blend word follows from its alpha, and
//     a layer is covered by its BEGIN_CLIP's box, which holds everything inside the layer and the pixels its blend touches.
//     Other draw objects have no opacity word, so their rows are no change.
// Draw boxes are binning's clipped boxes, rounded out to tiles exactly as tile_alloc rounds them, so a draw object paints no
// pixel outside its box. A moved open clip changes the boxes of later instances' draw objects, but only inside its own old
// and new box, which its BEGIN_CLIP contributes.
//
// The comparison needs the last successful frame's words and boxes: the snapshot holds two slots behind a generation word.
// A frame reads slot gen & 1 and writes its own words and boxes into the other one; k_damage_commit, the frame's last kernel,
// advances the generation only when bump.failed is 0. A re-run after an arena overflow therefore compares against the same
// slot and computes the same damage, and the frame's launches never change: moving instances keeps replaying one graph.
#include <string.h>

#include <algorithm>

#include "vb_device.cuh"
#include "vb_stages.h"

#define DM_THREADS 256u
#define DM_RECTS 64u // caller rectangles per k_damage_rects launch

// the snapshot slot the last successful frame wrote (old) and the one this frame writes (nxt)
__device__ __forceinline__ void dm_slots(uint32_t *snap, size_t slot_words, const uint32_t **old, uint32_t **nxt) {
    const uint32_t gen = *(volatile uint32_t *)snap;
    *old = snap + VB_DMG_HEADER_WORDS + (gen & 1u) * slot_words;
    *nxt = snap + VB_DMG_HEADER_WORDS + ((gen + 1u) & 1u) * slot_words;
}

// A full frame damages every tile; otherwise the frame starts from the caller's rectangles. No instance or path has changed yet.
__global__ void __launch_bounds__(DM_THREADS) k_damage_begin(uint8_t *mask, const uint8_t *__restrict__ pending, uint32_t n_tiles, uint32_t full,
                                                             uint32_t *changed, uint32_t n_inst, uint32_t *paths, uint32_t n_paths) {
    const uint32_t i = blockIdx.x * DM_THREADS + threadIdx.x;
    if (i < n_tiles) mask[i] = full ? 1u : pending[i];
    if (i < n_inst) changed[i] = 0u;
    if (i < n_paths) paths[i] = 0u;
}

// The inputs of k_damage_mark and k_damage: the snapshot `snap`, laid out by L (its flag arrays: L.changed, L.paths, L.xf), the
// frame's mask, the words the frame reads and the bindings' tables (VbBound). The mask words `vis` are null without bound
// visibility, `grad` (VbBound::rs_draw) without a bound gradient, `xf_range` without bound transforms, the stroke-width
// snapshot `widths` without bound widths (`styles`: the scene's n_style style words, `path_draw`: pathtag's path table). The
// frame's draw data `dd` has n_dd words.
struct DmArgs {
    VbDmgLayout L;
    uint32_t *snap;
    uint8_t *mask;
    const uint32_t *xf, *pd, *vis, *draw_tags, *dd; // transforms, path data, visibility mask, draw tags, draw data
    const VbBbox4 *draw_bboxes;
    const VbDrawMonoid *draw_monoids;
    const uint32_t *inst_prefix, *inst_draw, *pt_first, *grad, *ramps; // ramps: the bound gradients' rows
    const uint2 *xf_range;
    const float *widths;
    const uint2 *path_draw;
    const uint32_t *styles;
    uint32_t compare, wt, ht, n_style, n_dd;
};

// One thread per transform u of the frame: its six words against the snapshot, and into the next slot. A difference marks
// the instance holding u (the binding's prefix of the instances' transform counts). The same thread takes bound point u, when
// there is one: its two words in the frame's path data (`pd`, the bound region). A difference marks the path holding u
// (`pt_first`, the binding's first point of each path). A non-finite row left the encoded words in the region, so it is a
// change only if the words are. With bound transforms, flag u records whether transform u differs (a non-finite row that left
// an unchanged word does not). The same thread takes word u of the visibility mask, when there is one: each bit that differs
// marks its draw object, path d being draw object d. The mask holds normalised bits, so a row going from 1 to 2 is no change.
__global__ void __launch_bounds__(DM_THREADS) k_damage_mark(const DmArgs a) {
    const VbDmgLayout &L = a.L;
    const uint32_t u = blockIdx.x * DM_THREADS + threadIdx.x;
    const uint32_t n_paths = L.paths ? L.n_paths : 0u, n_pt = n_paths ? L.n_pt : 0u;
    if (u >= L.n_xf && u >= n_pt && u >= L.n_vis) return;
    const uint32_t *old;
    uint32_t *nxt;
    dm_slots(a.snap, L.slot_words, &old, &nxt);
    uint32_t *changed = a.snap + L.changed, *paths = a.snap + L.paths, *xf_changed = a.snap + L.xf;
    if (u < L.n_xf) {
        bool diff = false;
#pragma unroll
        for (uint32_t i = 0; i < 6u; i++) {
            const uint32_t w = __ldg(a.xf + 6u * u + i);
            diff = diff || w != old[6u * u + i];
            nxt[6u * u + i] = w;
        }
        if (a.compare && diff && L.n_inst) changed[cp_find(a.inst_prefix, 0u, L.n_inst - 1u, u)] = 1u;
        if (a.compare && L.xf) xf_changed[u] = diff ? 1u : 0u;
    }
    if (u < n_pt) {
        const uint32_t x = __ldg(a.pd + 2u * u), y = __ldg(a.pd + 2u * u + 1u);
        const size_t o = L.pt + 2u * (size_t)u;
        const bool diff = x != old[o] || y != old[o + 1u];
        nxt[o] = x;
        nxt[o + 1u] = y;
        if (a.compare && diff) paths[cp_find(a.pt_first, 0u, n_paths - 1u, u)] = 1u;
    }
    if (u < L.n_vis) {
        const uint32_t w = __ldg(a.vis + u);
        uint32_t flips = a.compare ? w ^ old[L.vis + u] : 0u;
        nxt[L.vis + u] = w;
        while (flips != 0u) {
            const uint32_t d = 32u * u + (uint32_t)(__ffs((int)flips) - 1);
            flips &= flips - 1u;
            if (d < n_paths) paths[d] = 1u;
        }
    }
}

// One warp per draw object: its box, below L.n_col its colour word and, for a bound gradient (`grad`: the draw object's
// gradient g or VB_COLOR_NONE), its ramp row (`ramps` + 512 g) into the next slot; when its instance (L.n_inst > 0), its colour
// word, its ramp row or its path's points (flagged with points or visibility bound) or one of its path's transforms (path d
// reads transforms xf_range[d].x .. .y, each flagged with transforms bound) changed, its old and new boxes into the mask. A draw
// object whose paint is not one colour has colour word 0: its bound row is never read. Its colour word is at its draw monoid's
// offset in the frame's draw data (`dd`, the bound region). Below L.n_wid, its stroke width: the snapshot entry, or for 0 the
// width word of its path's style (path d is draw object d). Below L.n_op, its opacity word in `dd` (a BEGIN_CLIP's alpha word
// right after its draw monoid's offset, an image's sample word two after it), or 0 for any other draw object.
__global__ void __launch_bounds__(DM_THREADS) k_damage(const DmArgs a) {
    const VbDmgLayout &L = a.L;
    const uint32_t d = blockIdx.x * (DM_THREADS / 32u) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (d >= L.n_draw) return;
    const uint32_t *old;
    uint32_t *nxt;
    dm_slots(a.snap, L.slot_words, &old, &nxt);
    const VbBbox4 *box = a.draw_bboxes + d;
    const VbBbox4 now = {__ldg(&box->x0), __ldg(&box->y0), __ldg(&box->x1), __ldg(&box->y1)};
    const VbBbox4 was = reinterpret_cast<const VbBbox4 *>(old + L.box)[d];
    bool hit = false;
    if (d < L.n_col) {
        const uint32_t tag = __ldg(a.draw_tags + d);
        const bool one_colour = tag == VB_DRAWTAG_FILL_COLOR || tag == VB_DRAWTAG_BLURRED_ROUNDED_RECT;
        const uint32_t col = one_colour ? __ldg(a.dd + __ldg(&a.draw_monoids[d].scene_offset)) : 0u;
        hit = col != old[L.col + d];
        if (lane == 0u) nxt[L.col + d] = col;
    }
    if (d < L.n_wid) {
        uint32_t w = __float_as_uint(__ldg(a.widths + d));
        if (w == 0u && d < L.n_paths) {
            const uint32_t s = __ldg(&a.path_draw[d].x) + 1u;
            w = s < a.n_style ? __ldg(a.styles + s) : 0u;
        }
        hit = w != old[L.wid + d] || hit;
        if (lane == 0u) nxt[L.wid + d] = w;
    }
    if (d < L.n_op) {
        const uint32_t tag = __ldg(a.draw_tags + d);
        const uint32_t at = tag == VB_DRAWTAG_BEGIN_CLIP ? 1u : tag == VB_DRAWTAG_FILL_IMAGE ? 2u : 0u;
        const uint32_t o = __ldg(&a.draw_monoids[d].scene_offset) + at;
        const uint32_t w = at && o < a.n_dd ? __ldg(a.dd + o) : 0u;
        hit = w != old[L.op + d] || hit;
        if (lane == 0u) nxt[L.op + d] = w;
    }
    const uint32_t g = a.grad ? __ldg(a.grad + d) : VB_COLOR_NONE;
    if (g != VB_COLOR_NONE) {
        const uint32_t *row = a.ramps + 512u * (size_t)g;
        const size_t at = L.ramp + 512u * (size_t)g;
        bool diff = false;
        for (uint32_t i = lane; i < 512u; i += 32u) {
            const uint32_t w = __ldg(row + i);
            diff = diff || w != old[at + i];
            nxt[at + i] = w;
        }
        hit = __any_sync(0xffffffffu, diff) || hit;
    }
    __syncwarp();
    if (lane == 0u) reinterpret_cast<VbBbox4 *>(nxt + L.box)[d] = now;
    if (!a.compare) return;
    const uint32_t *changed = a.snap + L.changed, *paths = a.snap + L.paths, *xf_changed = a.snap + L.xf;
    if (!hit && L.paths && d < L.n_paths) hit = __ldg(paths + d) != 0u; // path d is draw object d
    if (!hit && a.xf_range && d < L.n_paths && L.n_xf) {
        const uint2 t = __ldg(a.xf_range + d);
        const uint64_t hi = t.y < L.n_xf ? t.y : L.n_xf - 1u;
        bool any = false;
        for (uint64_t i = (uint64_t)t.x + lane; i <= hi; i += 32u) any = any || __ldg(xf_changed + i) != 0u;
        hit = __any_sync(0xffffffffu, any);
    }
    if (!hit) {
        // draw objects past the last instance (the END_CLIPs closing open clips) belong to no instance
        if (L.n_inst == 0u || d >= __ldg(a.inst_draw + L.n_inst)) return;
        if (__ldg(changed + cp_find(a.inst_draw, 0u, L.n_inst - 1u, d)) == 0u) return;
    }
    dm_or_box(a.mask, was, a.wt, a.ht, lane);
    dm_or_box(a.mask, now, a.wt, a.ht, lane);
}

// The frame's last kernel: a frame that succeeded becomes the base of the next one (its snapshot slot is current, the caller's
// rectangles are consumed). A failed attempt changes nothing, so its re-run computes the same damage. An unbound scene keeps
// no snapshot (snap is null).
__global__ void __launch_bounds__(DM_THREADS) k_damage_commit(const VbBump *bump, uint32_t *snap, uint8_t *pending, uint32_t n_tiles) {
    if (bump->failed != 0u) return;
    const uint32_t i = blockIdx.x * DM_THREADS + threadIdx.x;
    if (i == 0u && snap) snap[0] += 1u;
    if (i < n_tiles) pending[i] = 0u;
}

struct DmRects {
    uint32_t r[DM_RECTS][4]; // tile ranges x0 y0 x1 y1, clipped to the frame
    uint32_t wt;
};
// One CTA per rectangle.
__global__ void __launch_bounds__(DM_THREADS) k_damage_rects(uint8_t *pending, DmRects a) {
    const uint32_t *q = a.r[blockIdx.x];
    const uint32_t w = q[2] - q[0], n = w * (q[3] - q[1]);
    for (uint32_t i = threadIdx.x; i < n; i += DM_THREADS) pending[(q[1] + i / w) * a.wt + q[0] + i % w] = 1u;
}

extern "C" uint32_t vb_launch_damage(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbDamage &D = b.dmg;
    if (D.mode == VB_DMG_OFF) return 0u;
    const VbBound &B = b.bound;
    const VbDmgLayout L = vb_dmg_layout(B, cfg.layout, D.n_xf);
    const uint32_t wt = cfg.width_in_tiles, ht = cfg.height_in_tiles, n_tiles = wt * ht, full = D.mode == VB_DMG_FULL;
    const uint32_t n_paths = L.paths ? L.n_paths : 0u, n = std::max(std::max(n_tiles, L.n_inst), n_paths);
    k_damage_begin<<<(n + DM_THREADS - 1u) / DM_THREADS, DM_THREADS, 0, st>>>(D.mask, D.pending, n_tiles, full, D.snap + L.changed, L.n_inst,
                                                                              D.snap + L.paths, n_paths);
    // neither instance transforms, colours, points, stops, transforms, visibility, stroke widths nor opacity bound: nothing
    // changes without a call that makes the frame full
    if (L.n_inst == 0u && L.n_col == 0u && L.n_pt == 0u && L.n_grads == 0u && B.rows[VB_BIND_TRANSFORMS].n == 0u && L.n_vis == 0u &&
        L.n_wid == 0u && L.n_op == 0u)
        return 1u;
    DmArgs a;
    a.L = L, a.snap = D.snap, a.mask = D.mask, a.compare = !full, a.wt = wt, a.ht = ht;
    a.xf = b.scene + cfg.layout.transform_base, a.pd = b.scene + cfg.layout.path_data_base, a.vis = cfg.vis;
    a.draw_tags = b.scene + cfg.layout.draw_tag_base, a.dd = b.scene + cfg.layout.draw_data_base;
    a.draw_bboxes = b.draw_bboxes, a.draw_monoids = b.draw_monoids, a.ramps = b.ramps + 512u * (size_t)B.rs_ramp0;
    a.inst_prefix = B.inst_prefix, a.inst_draw = B.inst_draw, a.pt_first = B.pt_first, a.grad = L.n_grads ? B.rs_draw : nullptr;
    a.xf_range = B.rows[VB_BIND_TRANSFORMS].rows ? B.xf_range : nullptr;
    a.widths = cfg.widths, a.path_draw = b.path_draw, a.styles = b.scene + cfg.layout.style_base;
    a.n_style = cfg.scene_words > cfg.layout.style_base ? cfg.scene_words - cfg.layout.style_base : 0u;
    a.n_dd = b.dd_len;
    uint32_t launches = 1u;
    const uint32_t n_mark = std::max(std::max(L.n_xf, n_paths ? L.n_pt : 0u), L.n_vis);
    if (n_mark) {
        k_damage_mark<<<(n_mark + DM_THREADS - 1u) / DM_THREADS, DM_THREADS, 0, st>>>(a);
        launches++;
    }
    if (L.n_draw) {
        const uint32_t per = DM_THREADS / 32u;
        k_damage<<<(L.n_draw + per - 1u) / per, DM_THREADS, 0, st>>>(a);
        launches++;
    }
    return launches;
}

extern "C" uint32_t vb_launch_damage_commit(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (b.dmg.mode == VB_DMG_OFF) return 0u;
    const uint32_t n_tiles = cfg.width_in_tiles * cfg.height_in_tiles;
    k_damage_commit<<<(n_tiles + DM_THREADS - 1u) / DM_THREADS, DM_THREADS, 0, st>>>(b.bump(), b.dmg.snap, b.dmg.pending, n_tiles);
    return 1u;
}

extern "C" uint32_t vb_launch_damage_rects(uint8_t *pending, uint32_t width_in_tiles, const uint32_t *tile_rects, uint32_t n, cudaStream_t st) {
    uint32_t launches = 0u;
    for (uint32_t i = 0; i < n; i += DM_RECTS) {
        DmRects a;
        const uint32_t m = std::min(DM_RECTS, n - i);
        memcpy(a.r, tile_rects + 4u * (size_t)i, (size_t)m * 16u);
        a.wt = width_in_tiles;
        k_damage_rects<<<m, DM_THREADS, 0, st>>>(pending, a);
        launches++;
    }
    return launches;
}
