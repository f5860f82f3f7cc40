// vb_debug.cu -- the vb_debug_* entry points: downloads and uploads of named buffers, arena limits and their guard regions,
// fine's traffic, the look-back test harness and graph capture counts.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>

#include "vb_device.cuh"
#include "vb_renderer.h"

// Statistics for the roofline of `fine`: PTCL words each tile's interpreter reads and segments it
// references (one thread per tile walks its command stream, as fine does).
// Under damage tracking (`damage` non-null) only the tiles fine painted count.
__global__ void k_ptcl_stats(VbConfig cfg, const uint32_t *__restrict__ ptcl, const uint32_t *__restrict__ tile_start,
                             const uint8_t *__restrict__ damage, unsigned long long *out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t wt = cfg.width_in_tiles, rows = cfg.win_ty1 - cfg.win_ty0;
    if (t >= wt * rows) return;
    uint32_t tile_ix = (cfg.win_ty0 + t / wt) * wt + t % wt;
    if (damage && !damage[tile_ix]) return;
    uint32_t ix = tile_ix * VB_PTCL_INITIAL_ALLOC + 1u;
    unsigned long long words = 1, segs = 0, fills = 0;
    if (tile_start && tile_start[tile_ix]) { // occlusion start: the interpreter begins at the tile's last opaque cover
        ix = tile_start[tile_ix];
        words += 1;
    }
    for (uint32_t guard = 0; guard < (1u << 24); guard++) {
        uint32_t tag = ptcl[ix];
        uint32_t size = 1;
        if (tag == VB_CMD_END) { words += 1; break; }
        if (tag == VB_CMD_JUMP) { words += 2; ix = ptcl[ix + 1]; continue; }
        if (tag == VB_CMD_FILL) { size = 4; segs += ptcl[ix + 1] >> 1; fills++; }
        else if (tag == VB_CMD_COLOR || tag == VB_CMD_IMAGE) size = 2;
        else if (tag == VB_CMD_LIN_GRAD || tag == VB_CMD_RAD_GRAD || tag == VB_CMD_SWEEP_GRAD || tag == VB_CMD_END_CLIP || tag == VB_CMD_BLUR_RECT) size = 3;
        words += size;
        ix += size;
    }
    atomicAdd(out, words);
    atomicAdd(out + 1, segs);
    atomicAdd(out + 2, fills);
}

struct NamedBuf {
    const char *name;
    DevBuf *buf;
    size_t bytes;
    size_t off = 0; // where the bytes start in buf
};
static std::vector<NamedBuf> named(vb_renderer *r) {
    const VbConfig &c = r->cfg;
    std::vector<NamedBuf> v = {
        {"scene", &r->cur->scene, r->cur->scene_words * 4}, // the uploaded / device-resolved inputs
        {"ramps", &r->cur->ramps, (size_t)r->cur->n_ramps * 512 * 4},
        {"atlas", &r->cur->atlas, (size_t)r->cur->atlas_w * r->cur->atlas_h * 4},
    };
    // the ramps the last frame read: with bound gradient stops the binding's, the scene's and then one row per gradient
    if (r->bufs.ramps && r->bufs.ramps == (const uint32_t *)r->stop_ramps.p) v[1] = {"ramps", &r->stop_ramps, (size_t)c.n_ramps * 512 * 4};
    // the fixed-size intermediates of the frame prepared last
    for (int i = 0; i < N_FIXED_BUFS; i++)
        if (FRAME_BUFS[i].downloadable) v.push_back({FRAME_BUFS[i].name, &r->fb[i], FRAME_BUFS[i].bytes(r->counts, true)});
    // the transform words the last frame read from its transform_base: the bound or viewed region, else the scene's stream
    const size_t t_off = (size_t)c.layout.transform_base * 4u, t_cap = r->cur->scene.cap > t_off ? r->cur->scene.cap - t_off : 0u;
    v.push_back({"transforms", &r->cur->scene, std::min<size_t>(24u * (size_t)n_transforms(r->cur->layout, r->cur->scene_words), t_cap), t_off});
    // the draw-data words the last frame read from its draw_data_base: the bound colours' region, else the scene's stream
    const size_t d_off = (size_t)c.layout.draw_data_base * 4u, d_cap = r->cur->scene.cap > d_off ? r->cur->scene.cap - d_off : 0u;
    v.push_back({"draw_data", &r->cur->scene, std::min<size_t>(4u * (size_t)n_draw_data(r->cur->layout, r->cur->scene_words), d_cap), d_off});
    // the path-data words the last frame read from its path_data_base: the bound points' region, else the scene's stream
    const size_t p_off = (size_t)c.layout.path_data_base * 4u, p_cap = r->cur->scene.cap > p_off ? r->cur->scene.cap - p_off : 0u;
    v.push_back({"path_data", &r->cur->scene, std::min<size_t>(4u * (size_t)n_path_data(r->cur->layout, r->cur->scene_words), p_cap), p_off});
    // the stroke widths the last frame read (k_widths.cu): one float per draw object, 0 where the encoded width applies; empty
    // while unbound
    v.push_back({"stroke_widths", &r->width_snap, c.widths ? (size_t)vb_width_entries(c.layout) * 4u : 0u});
    // an arena's buffer up to what the last attempt used of it, at most the capacity the kernels saw
    const uint32_t *size = &c.lines_size;
    for (int a = 0; a < N_ARENAS; a++) {
        const ArenaDesc &d = ARENAS[a];
        const size_t used = (size_t)std::min<uint64_t>(arena_need(r, a), size[a]);
        v.push_back({FRAME_BUFS[d.buf].name, &r->fb[d.buf], (arena_offset(r, a) + used) * d.elem_bytes});
    }
    return v;
}

// The guard region of a limited arena (vb_debug_limit_arena): the bytes of its allocation past the limit. `name` is an arena
// name, or "line_scratch" / "flatten_jobs" (flatten's scratch arenas, sized from the lines capacity). Returns false for an
// unknown name; *buf is nullptr while the arena has no limit.
static bool guard_region(vb_renderer *r, const char *name, DevBuf **buf, size_t *off) {
    DevBuf *scratch = !strcmp(name, "line_scratch") ? &r->fb[FB_LINE_SCRATCH] : !strcmp(name, "flatten_jobs") ? &r->fb[FB_FLATTEN_JOBS] : nullptr;
    const int a = scratch ? ARENA_LINES : arena_index(name);
    if (a < 0) return false;
    *buf = nullptr;
    *off = 0;
    const uint32_t lim = r->limit[a];
    if (lim == UINT32_MAX) return true;
    // ptcl: includes the 512 bytes of window slack that fine reads and never writes
    DevBuf *b = &r->fb[ARENAS[a].buf];
    size_t o = (arena_offset(r, a) + lim) * ARENAS[a].elem_bytes;
    if (scratch) {
        size_t lit_bytes, job_bytes; // flatten sees lits_cap = lines_size, jobs_cap = lines_size / FL_DEFER_MIN + 1
        vb_flatten_arena_bytes(lim, &lit_bytes, &job_bytes);
        b = scratch;
        o = scratch == &r->fb[FB_LINE_SCRATCH] ? lit_bytes : job_bytes;
    }
    *buf = b;
    *off = o < b->cap ? o : b->cap;
    return true;
}

extern "C" int vb_debug_limit_arena(vb_renderer *r, const char *arena, uint32_t limit) {
    if (!r || !arena) return VB_E_INVALID;
    const int a = arena_index(arena);
    if (a < 0) {
        r->err = std::string("vb_debug_limit_arena: unknown arena ") + arena;
        return VB_E_INVALID;
    }
    hit_forget(r);
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    CK(cudaStreamSynchronize(r->upload_stream));
    if (limit == UINT32_MAX) {
        r->limit[a] = UINT32_MAX;
        return VB_OK;
    }
    // 0 is refused too: path_count and path_tiling size their grids from the capacity
    if (limit == 0u || limit > r->cap[a] || (a == ARENA_PTCL && limit < ptcl_static(r->cfg))) {
        r->err = "vb_debug_limit_arena: the limit must be at least 1 (the static area for ptcl) and at most the allocation";
        return VB_E_INVALID;
    }
    r->limit[a] = limit;
    const char *regions[3] = {ARENAS[a].name, "line_scratch", "flatten_jobs"};
    for (int k = 0; k < (a == ARENA_LINES ? 3 : 1); k++) {
        DevBuf *b = nullptr;
        size_t off = 0;
        guard_region(r, regions[k], &b, &off);
        if (b && b->cap > off) CK(cudaMemsetAsync((char *)b->p + off, VB_GUARD_BYTE, b->cap - off, r->stream));
    }
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

extern "C" int vb_debug_download(vb_renderer *r, const char *name, void *dst, size_t cap, size_t *bytes) {
    if (!r || !name) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    const size_t len = strlen(name);
    if (len > 6 && !strcmp(name + len - 6, ".guard")) {
        const std::string base(name, len - 6);
        DevBuf *b;
        size_t off;
        if (!guard_region(r, base.c_str(), &b, &off)) return VB_E_UNKNOWN_BUFFER;
        const size_t n = b ? b->cap - off : 0;
        if (bytes) *bytes = n;
        const size_t c = n < cap ? n : cap;
        if (dst && c) CK(cudaMemcpy(dst, (const char *)b->p + off, c, cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    if (!strcmp(name, "bump")) {
        if (bytes) *bytes = sizeof(VbBump);
        if (dst && cap >= sizeof(VbBump)) CK(cudaMemcpy(dst, r->fb[FB_CTL].p, sizeof(VbBump), cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    // segment slots of the last frame that backdrop assigned and no CMD_FILL uses (k_tile.cu, k_coarse.cu); after an incremental
    // frame (damage tracking) also the slots of the quadrants coarse skipped, so not the reference's count
    if (!strcmp(name, "seg_holes")) {
        if (bytes) *bytes = 4;
        if (dst && cap >= 4) CK(cudaMemcpy(dst, (const uint32_t *)r->fb[FB_CTL].p + VB_CTL_SEG_HOLES, 4, cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    // the tile counts of fine's lists in the last frame (k_coarse.cu): VB_FINE_LISTS words, list 2k + 1 the flagged tiles of class k
    if (!strcmp(name, "fine_lists")) {
        if (bytes) *bytes = VB_FINE_LISTS * 4;
        if (dst && cap >= VB_FINE_LISTS * 4)
            CK(cudaMemcpy(dst, (const uint32_t *)r->fb[FB_CTL].p + VB_CTL_FINE_CLASS, VB_FINE_LISTS * 4, cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    if (!strcmp(name, "config")) {
        if (bytes) *bytes = sizeof(VbConfig);
        if (dst && cap >= sizeof(VbConfig)) memcpy(dst, &r->cfg, sizeof(VbConfig));
        return VB_OK;
    }
    // flatten's device counters of the last attempt (k_flatten.cu FlCtx::ctrs): literal records, jobs, and the length of
    // the general tag kernel's work list; and its two scratch arenas up to their counters (at most their capacity)
    const bool lits = !strcmp(name, "line_scratch"), jobs = !strcmp(name, "flatten_jobs");
    if (!strcmp(name, "flatten_counters") || lits || jobs) {
        uint32_t ctrs[3] = {0u, 0u, 0u};
        if (r->bufs.lb_flatten) CK(cudaMemcpy(ctrs, r->bufs.lb_flatten, sizeof ctrs, cudaMemcpyDeviceToHost));
        size_t n = sizeof ctrs;
        const void *src = ctrs;
        bool host = true;
        if (lits || jobs) {
            size_t lit1, job1, lit_cap, job_cap; // one record of each, and the capacities the kernels saw
            vb_flatten_arena_bytes(1u, &lit1, &job1);
            vb_flatten_arena_bytes(r->cfg.lines_size, &lit_cap, &job_cap);
            const DevBuf &b = r->fb[lits ? FB_LINE_SCRATCH : FB_FLATTEN_JOBS];
            n = std::min({(size_t)ctrs[lits ? 0 : 1] * (lits ? lit1 : job1), lits ? lit_cap : job_cap, b.cap});
            src = b.p;
            host = false;
        }
        if (bytes) *bytes = n;
        const size_t c = n < cap ? n : cap;
        if (dst && c) {
            if (host) memcpy(dst, src, c);
            else CK(cudaMemcpy(dst, src, c, cudaMemcpyDeviceToHost));
        }
        return VB_OK;
    }
    for (auto &nb : named(r))
        if (!strcmp(name, nb.name)) {
            if (bytes) *bytes = nb.bytes;
            size_t n = nb.bytes < cap ? nb.bytes : cap;
            if (dst && n) CK(cudaMemcpy(dst, (const char *)nb.buf->p + nb.off, n, cudaMemcpyDeviceToHost));
            return VB_OK;
        }
    return VB_E_UNKNOWN_BUFFER;
}

extern "C" int vb_debug_graph_captures(vb_renderer *r, uint64_t *captures) {
    if (!r || !captures) return VB_E_INVALID;
    *captures = r->graph_captures;
    return VB_OK;
}

extern "C" int vb_debug_fine_traffic(vb_renderer *r, uint64_t *ptcl_words, uint64_t *segment_refs, uint64_t *fill_cmds) {
    if (!r) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    unsigned long long *d = nullptr, h[3] = {0, 0, 0};
    CK(cudaMalloc(&d, sizeof h));
    CK(cudaMemset(d, 0, sizeof h));
    VbConfig c = r->cfg;
    const FineRows f = fine_rows(c, Dest{});
    c.win_ty0 = f.ty0, c.win_ty1 = f.ty1;
    uint32_t n = c.width_in_tiles * (c.win_ty1 - c.win_ty0);
    const uint8_t *damage = r->dmg.have_last && r->dmg.last.mode == VB_DMG_INCREMENTAL ? (const uint8_t *)r->dmg_mask.p : nullptr;
    if (n) k_ptcl_stats<<<(n + 127) / 128, 128, 0, r->stream>>>(c, (const uint32_t *)r->fb[FB_PTCL].p,
                                                                r->occlusion_cull ? (const uint32_t *)r->fb[FB_TILE_START].p : nullptr, damage, d);
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaMemcpy(h, d, sizeof h, cudaMemcpyDeviceToHost));
    cudaFree(d);
    if (ptcl_words) *ptcl_words = h[0];
    if (segment_refs) *segment_refs = h[1];
    if (fill_cmds) *fill_cmds = h[2];
    return VB_OK;
}

extern "C" int vb_debug_upload(vb_renderer *r, const char *name, const void *src, size_t bytes) {
    if (!r || !name || !src) return VB_E_INVALID;
    hit_forget(r);
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    // "lines" and "tiles": the arena's contents and its bump counter. Growing the arena frees it without copying, and the
    // look-back state of backdrop is sized from the tile capacity when the next frame is prepared.
    for (int a : {ARENA_LINES, ARENA_TILES}) {
        if (strcmp(name, ARENAS[a].name)) continue;
        const uint32_t n = (uint32_t)(bytes / ARENAS[a].elem_bytes);
        if (n > r->cap[a]) {
            r->cap[a] = grow(n);
            int rc = ensure_arena(r, a);
            if (rc) return rc;
        }
        if (n) CK(cudaMemcpy(r->fb[ARENAS[a].buf].p, src, (size_t)n * ARENAS[a].elem_bytes, cudaMemcpyHostToDevice));
        VbBump *bump = (VbBump *)r->fb[FB_CTL].p;
        CK(cudaMemcpy(&(bump->*ARENAS[a].counter), &n, 4, cudaMemcpyHostToDevice));
        r->cur->h_bump->*ARENAS[a].counter = n;
        return VB_OK;
    }
    if (!strcmp(name, "path_bboxes")) {
        if (bytes > r->fb[FB_PATH_BBOXES].cap) return VB_E_INVALID;
        CK(cudaMemcpy(r->fb[FB_PATH_BBOXES].p, src, bytes, cudaMemcpyHostToDevice));
        return VB_OK;
    }
    if (!strcmp(name, "paths")) { // backdrop searches exactly n_draw_objects of them
        if (bytes != (size_t)r->cur->layout.n_draw_objects * sizeof(VbPath) || bytes > r->fb[FB_PATHS].cap) {
            r->err = "vb_debug_upload: \"paths\" takes exactly one record per draw object, after a frame of the scene";
            return VB_E_INVALID;
        }
        if (bytes) CK(cudaMemcpy(r->fb[FB_PATHS].p, src, bytes, cudaMemcpyHostToDevice));
        return VB_OK;
    }
    return VB_E_UNKNOWN_BUFFER;
}

extern "C" int vb_debug_lookback(vb_renderer *r, int op, uint32_t n_parts, const uint32_t *agg, const uint32_t *delay_ns, uint32_t *excl) {
    if (!r) return VB_E_INVALID;
    const uint32_t K = vb_debug_lookback_words(op);
    if (!agg || !excl || K == 0u || n_parts == 0u || n_parts > VB_LOOKBACK_MAX_PARTS) {
        r->err = "vb_debug_lookback: unknown op, no buffers, or n_parts outside 1..VB_LOOKBACK_MAX_PARTS";
        return VB_E_INVALID;
    }
    for (uint32_t p = 0; delay_ns && p < n_parts; p++)
        if (delay_ns[p] > VB_LOOKBACK_MAX_DELAY_NS) {
            r->err = "vb_debug_lookback: a delay exceeds VB_LOOKBACK_MAX_DELAY_NS";
            return VB_E_INVALID;
        }
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    // one allocation: [look-back state][agg: n_parts * K][delays: n_parts][excl: n_parts * K]
    const size_t lb_words = vb_lookback_words(n_parts, (int)K), vec = (size_t)n_parts * K;
    DevBuf d;
    int rc = ensure(r, d, (lb_words + 2 * vec + n_parts) * 4);
    if (rc) return rc;
    uint32_t *lb = (uint32_t *)d.p, *d_agg = lb + lb_words, *d_delay = d_agg + vec, *d_excl = d_delay + n_parts;
    auto run = [&]() -> int {
        CK(cudaMemsetAsync(lb, 0, lb_words * 4, r->stream));
        CK(cudaMemcpyAsync(d_agg, agg, vec * 4, cudaMemcpyHostToDevice, r->stream));
        if (delay_ns) CK(cudaMemcpyAsync(d_delay, delay_ns, (size_t)n_parts * 4, cudaMemcpyHostToDevice, r->stream));
        else CK(cudaMemsetAsync(d_delay, 0, (size_t)n_parts * 4, r->stream));
        vb_launch_debug_lookback(op, n_parts, lb, d_agg, d_delay, d_excl, r->stream);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(excl, d_excl, vec * 4, cudaMemcpyDeviceToHost, r->stream));
        CK(cudaStreamSynchronize(r->stream));
        return VB_OK;
    };
    rc = run();
    cudaFree(d.p);
    return rc;
}
