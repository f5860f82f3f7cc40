// vb_damage.cu -- damage tracking (k_damage.cu): which frames are incremental, and the C ABI around it.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>

#include "vb_renderer.h"

// ---- damage tracking: vb_set_damage_tracking / vb_add_damage / vb_last_damage (k_damage.cu) -------------------------------
// After prepare, pick_out and resolve_background: is the frame incremental, full, or outside damage tracking (a batch, a window,
// a background, the exchange: mode VB_DMG_OFF, and no base for the next frame)? A background frame is full because nothing tells
// which of the background's pixels changed since the base frame. The decision is the same for every re-run of the frame, because the base
// and the forcing flags change only when a frame succeeds (damage_succeeded). Allocates the mask, the staged rectangles and,
// while anything is bound, the snapshot with its flags (vb_dmg_layout). The mask's size follows from the frame size, which an
// incremental frame shares with its base; the snapshot's from the scene and what is bound, which change only through an
// installation or a binding. Both advance the epoch and so make the next frame full: no buffer moves under an incremental frame.
int vb_host::damage_prepare(vb_renderer *r) {
    vb_renderer::Damage &D = r->dmg;
    const VbConfig &c = r->cfg;
    vb_renderer::DamageFrame f;
    f.w = c.target_width;
    f.h = c.target_height;
    f.aa = r->params.aa;
    f.base_color = c.base_color;
    f.dest = r->dest.dev;
    f.epoch = D.epoch;
    const bool windowed = r->params.bin_row1 > r->params.bin_row0 || r->params.tile_row1 > r->params.tile_row0;
    f.can_base = D.on && c.n_cells == 1u && !windowed && !r->dest.bg.on && !r->xc.enabled && !r->grouped;
    D.frame = f;
    if (!f.can_base) return VB_OK;
    // an overridden image copied again changes pixels nothing here can locate: the frame is full unless the caller named them
    for (const auto &o : r->cur->overridden)
        if (o.dirty && !D.rects) D.force_full = true;
    const vb_renderer::DamageFrame &B = D.base;
    const vb_renderer::Damage::Diff &X = D.diff;
    const bool diff = X.armed && X.epoch == f.epoch; // the scene was diffed against the base's (vb_recompose, vb_set_upload_diff)
    const bool incremental = D.have_base && !D.force_full && !r->dest.host && (B.epoch == f.epoch || diff) && B.w == f.w && B.h == f.h &&
                             B.aa == f.aa && B.base_color == f.base_color && B.dest == f.dest;
    f.mode = incremental ? VB_DMG_INCREMENTAL : VB_DMG_FULL;
    // this frame rewrites the mask: the last successful frame's can be reported again only if this one succeeds (a frame that
    // fails for good, or a streamed one, which the host does not follow frame by frame, leaves nothing to report)
    if (D.last.mode == VB_DMG_INCREMENTAL) D.have_last = false;
    const uint32_t n_tiles = c.width_in_tiles * c.height_in_tiles;
    const VbRows *rows = r->bound.rows;
    const uint32_t n_xf = rows[VB_BIND_INSTANCES].rows || rows[VB_BIND_TRANSFORMS].rows ? n_transforms(r->cur->layout, r->cur->scene_words) : 0u;
    const bool snap = any_binding(r->bound);
    int rc;
    if ((rc = ensure(r, r->dmg_mask, n_tiles))) return rc;
    if ((rc = ensure(r, r->dmg_pending, n_tiles))) return rc;
    if (snap && (rc = ensure(r, r->dmg_snap, vb_dmg_layout(r->bound, r->cur->layout, n_xf).bytes))) return rc;
    VbDamage &dm = r->bufs.dmg;
    dm.mask = (uint8_t *)r->dmg_mask.p;
    dm.pending = (uint8_t *)r->dmg_pending.p;
    if (snap) dm.snap = (uint32_t *)r->dmg_snap.p;
    dm.mode = f.mode;
    dm.n_xf = n_xf;
    if (incremental && diff) { // k_recompose_damage's inputs; an upload's tables are built by the frame (k_upload_diff.cu)
        const char *p = (const char *)r->dmg_diff.p;
        if (X.upload) dm.udiff = (VbUdiff *)r->dmg_diff.p;
        dm.old_boxes = (const VbBbox4 *)(p + X.o_boxes);
        dm.tables = (const uint32_t *)(p + X.o_tables);
        dm.n_old = X.n_old;
        dm.n_new = X.n_new;
        dm.old_draws = X.old_draws;
        dm.new_draws = X.new_draws;
    }
    D.frame = f;
    return VB_OK;
}

// There is a tracked base frame of the current scene (the epoch unchanged since: no installation, binding, view, cells or
// tracking switch), unbound (any_binding: a diff compares scenes, not what a binding made of them), of one cell, whose intermediates are intact: hit tests answer from it (no failed frame, vb_run_stages or debug write
// since).
bool vb_host::base_diffable(const vb_renderer *r) {
    const vb_renderer::Damage &D = r->dmg;
    const vb_renderer::SceneSlot &s = *r->cur;
    return D.on && D.have_base && D.base.epoch == D.epoch && s.have_scene && !any_binding(r->bound) &&
           r->hit.valid && !r->hit.windowed && r->hit.cfg.n_cells == 1u && r->hit.cfg.layout.n_draw_objects == s.layout.n_draw_objects;
}

// Size dmg_diff (an upload's laid out by vb_udiff_layout; a recompose's as [boxes] [tables, 16-byte aligned]), enqueue on st the
// copy of the base frame's draw boxes, before anything can rewrite them, and mark the record pending for set_scene to arm.
int vb_host::diff_begin(vb_renderer *r, cudaStream_t st, bool upload, uint32_t n_old, uint32_t n_new, uint32_t new_draws) {
    const uint32_t old_draws = r->cur->layout.n_draw_objects;
    const size_t box_bytes = (size_t)old_draws * sizeof(VbBbox4);
    const VbUdLayout U = vb_udiff_layout(n_old, n_new);
    const size_t o_boxes = upload ? U.boxes : 0u, o_tables = upload ? U.tables : (box_bytes + 15u) & ~(size_t)15u;
    const size_t bytes = o_tables + vb_rcmp_tables((uint32_t *)nullptr, n_old, n_new).words * 4u;
    if (r->dmg_diff.cap < bytes) CK(cudaStreamSynchronize(st)); // growing: copies enqueued into it may not have run yet
    int rc;
    if ((rc = ensure(r, r->dmg_diff, bytes))) return rc;
    if (old_draws) CK(cudaMemcpyAsync((char *)r->dmg_diff.p + o_boxes, r->hit.bufs.draw_bboxes, box_bytes, cudaMemcpyDeviceToDevice, st));
    r->dmg.diff = vb_renderer::Damage::Diff{true, false, upload, 0u, n_old, n_new, old_draws, new_draws, o_boxes, o_tables}; // pending
    return VB_OK;
}
// The frame prepared last succeeded: it is the one vb_last_damage reports, and the base of the next frame when it was tracked.
void vb_host::damage_succeeded(vb_renderer *r) {
    vb_renderer::Damage &D = r->dmg;
    D.last = D.frame;
    D.have_last = true;
    D.have_base = D.frame.mode != VB_DMG_OFF;
    if (D.have_base) D.base = D.frame;
    D.rects = false;
    D.force_full = false;
    D.diff.armed = false;
}

extern "C" int vb_set_damage_tracking(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    if (on && (r->grouped || r->xc.configured)) {
        r->err = "vb_set_damage_tracking: not available for a renderer of a vb_group or with the exchange";
        return VB_E_INVALID;
    }
    r->dmg.on = on != 0;
    r->dmg.epoch++; // switched on (or on again): the next frame is full
    if (!on) r->dmg.have_base = false;
    return VB_OK;
}

extern "C" int vb_add_damage(vb_renderer *r, const uint32_t *rects, uint32_t n) {
    if (!r) return VB_E_INVALID;
    if (n && !rects) {
        r->err = "vb_add_damage: NULL rectangles";
        return VB_E_INVALID;
    }
    // the rectangles belong to the frame after the one in flight, whose size and success are not known yet
    if (r->frame_pending || r->stream_pending) {
        r->err = "vb_add_damage: a frame is in flight (finish it with vb_frame_finish / vb_readback_wait)";
        return VB_E_INVALID;
    }
    vb_renderer::Damage &D = r->dmg;
    if (!D.on || n == 0u) return VB_OK;
    D.rects = true;
    if (!D.have_base) return VB_OK; // the next frame is a full one
    // clamped to the frame the next incremental frame must match, rounded out to tiles
    const uint32_t w = D.base.w, h = D.base.h, wt = (w + 15u) / 16u;
    std::vector<uint32_t> t;
    t.reserve((size_t)n * 4u);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t *q = rects + 4u * (size_t)i;
        const uint32_t x0 = std::min(q[0], w), y0 = std::min(q[1], h), x1 = std::min(q[2], w), y1 = std::min(q[3], h);
        if (x1 <= x0 || y1 <= y0) continue;
        t.insert(t.end(), {x0 / 16u, y0 / 16u, (x1 + 15u) / 16u, (y1 + 15u) / 16u});
    }
    if (t.empty()) return VB_OK;
    CK(cudaSetDevice(r->device));
    vb_launch_damage_rects((uint8_t *)r->dmg_pending.p, wt, t.data(), (uint32_t)(t.size() / 4u), r->stream); // in stream order
    CK(cudaGetLastError());
    return VB_OK;
}

extern "C" int vb_last_damage(vb_renderer *r, uint8_t *tile_mask, size_t cap, uint32_t *n_damaged) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const char *why) {
        r->err = std::string("vb_last_damage: ") + why;
        return VB_E_INVALID;
    };
    if (r->frame_pending || r->stream_pending) return bad("a frame is in flight (finish it with vb_frame_finish / vb_readback_wait)");
    const vb_renderer::Damage &D = r->dmg;
    if (!D.have_last) return bad("no completed frame to report (none yet, or a later tracked frame failed or was streamed)");
    const size_t n_tiles = (size_t)((D.last.w + 15u) / 16u) * ((D.last.h + 15u) / 16u);
    if (tile_mask && cap < n_tiles) return bad("the mask holds fewer bytes than the frame has tiles");
    std::vector<uint8_t> m(n_tiles, 1u); // a frame that was not incremental rendered every tile
    if (D.last.mode == VB_DMG_INCREMENTAL) {
        CK(cudaSetDevice(r->device));
        CK(cudaMemcpyAsync(m.data(), r->dmg_mask.p, n_tiles, cudaMemcpyDeviceToHost, r->stream));
        CK(cudaStreamSynchronize(r->stream));
    }
    uint32_t count = 0;
    for (uint8_t &v : m) {
        v = v ? 1u : 0u;
        count += v;
    }
    if (tile_mask) memcpy(tile_mask, m.data(), n_tiles);
    if (n_damaged) *n_damaged = count;
    return VB_OK;
}
