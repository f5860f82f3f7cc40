// k_coarse.cu -- per-tile command lists (PTCL).
//
// Reference: vello_shaders/shader/coarse.wgsl:156-471 (PTCL layout shared/ptcl.wgsl:6-25, writers
// coarse.wgsl:68-154), CPU twin cpu/coarse.rs. One CTA = one bin (16x16 tiles), one thread = one
// tile, as in the WGSL; log-step shared-memory scans are replaced by warp-shuffle scans.
// The per-tile command SEQUENCE is identical to the reference's; dynamic PTCL chunks come from an
// atomic bump allocator, so their absolute offsets are allocation-order dependent (as in the
// reference), and segment slices are in tile order (see below). Only bins inside the stripe window are launched.
// Parallelism: the WGSL launches one workgroup per bin (256 at 4096^2 -- far fewer than an H100 can hold), and the
// per-bin coverage loop is a chain of dependent global loads. Here every bin is split into four 8x8-tile QUADRANTS,
// each handled by its own CTA (all 256 threads share the (draw, tile) coverage loop, threads 0..63 own a tile each for
// emission), and the coverage loop keeps two independent tile loads in flight.
// Segment slices: the WGSL takes one global atomicAdd per CMD_FILL (coarse.wgsl:100) and writes ~slice into the tile,
// ~1.7 M same-address atomics and scattered stores on a map-like frame. Here k_backdrop has already given every
// (path, tile) its slice in tile order (k_tile.cu), so coarse only reads them: it allocates no segments and writes no
// tile, and k_path_tiling runs beside it. Slices of tiles that coarse turns into no CMD_FILL (a fill inside a
// zero-coverage clip, a clip path whose END_CLIP is not emitted) stay unused: ctl[VB_CTL_SEG_HOLES] starts at
// bump.segments and each CTA subtracts the segments of the fills it emits, so `bump.segments - holes` is the
// reference's number.
#include "vb_device.cuh"
#include "vb_stages.h"

#define CO_THREADS 256
#define CO_MINB 5 // CTAs per SM: 48 registers, no spills
#define CO_N_SLICE 8

struct TileState {
    uint32_t cmd_offset, cmd_limit;
};

// A tile as coarse sees it. k_backdrop wrote ~(first slot of the slice) into every tile of the arena in tile order, so a
// tile's segment count is the distance to the next tile's slice; the arena's last tile ends at bump.segments.
struct CoTile {
    int32_t backdrop;
    uint32_t seg_ix, n_segs;
};
__device__ __forceinline__ CoTile co_load_tile(const VbTile *tiles, uint32_t ix, uint32_t tile_end, uint32_t seg_end) {
    const VbTile t = tiles[ix];
    const uint32_t next = ix + 1u < tile_end ? ~tiles[ix + 1u].segment_count_or_ix : seg_end;
    CoTile c;
    c.backdrop = t.backdrop;
    c.seg_ix = ~t.segment_count_or_ix;
    c.n_segs = next - c.seg_ix;
    return c;
}

__device__ __forceinline__ void co_alloc_cmd(TileState &s, uint32_t size, const VbConfig &cfg, VbBump *bump, uint32_t *ptcl) {
    if (s.cmd_offset + size >= s.cmd_limit) {
        const uint32_t ptcl_dyn_start = cfg.width_in_tiles * cfg.tile_rows * VB_PTCL_INITIAL_ALLOC;
        uint32_t new_cmd = ptcl_dyn_start + atomicAdd(&bump->ptcl, VB_PTCL_INCREMENT);
        if (new_cmd + VB_PTCL_INCREMENT > cfg.ptcl_size) {
            // Out of PTCL space: park this tile's writes in the (unused) first dynamic chunk slot 0 of
            // the static area is not safe, so fall back to the tile's own static chunk start; the
            // frame is discarded and re-run with a bigger arena.
            new_cmd = 0u;
            atomicOr(&bump->failed, VB_STAGE_COARSE);
        }
        ptcl[s.cmd_offset] = VB_CMD_JUMP;
        ptcl[s.cmd_offset + 1u] = new_cmd;
        s.cmd_offset = new_cmd;
        s.cmd_limit = new_cmd + (VB_PTCL_INCREMENT - VB_PTCL_HEADROOM);
    }
}

// Returns the PTCL offset of the CMD_SOLID it wrote, or 0 when it wrote a CMD_FILL (whose segments it adds to `emitted`).
__device__ __forceinline__ uint32_t co_write_path(TileState &s, const CoTile &tile, uint32_t draw_flags, const VbConfig &cfg, VbBump *bump,
                                                  uint32_t *ptcl, uint32_t &emitted, uint32_t &cost) {
    const uint32_t n_segs = tile.n_segs;
    cost += n_segs != 0u ? 8u + n_segs : 1u; // what fine will spend on it, in rough units (a fill: set-up + its segments)
    if (n_segs != 0u) {
        emitted += n_segs;
        co_alloc_cmd(s, 4u, cfg, bump, ptcl);
        ptcl[s.cmd_offset] = VB_CMD_FILL;
        ptcl[s.cmd_offset + 1u] = (n_segs << 1) | (draw_flags & 1u);
        ptcl[s.cmd_offset + 2u] = tile.seg_ix;
        ptcl[s.cmd_offset + 3u] = (uint32_t)tile.backdrop;
        s.cmd_offset += 4u;
        return 0u;
    }
    co_alloc_cmd(s, 1u, cfg, bump, ptcl);
    ptcl[s.cmd_offset] = VB_CMD_SOLID;
    s.cmd_offset += 1u;
    return s.cmd_offset - 1u;
}

__global__ void __launch_bounds__(CO_THREADS, CO_MINB)
k_coarse(VbConfig cfg, const uint32_t *__restrict__ scene, const VbDrawMonoid *__restrict__ draw_monoids,
         const VbBinHeader *__restrict__ bin_headers, const uint32_t *__restrict__ info_bin_data, const VbPath *__restrict__ paths,
         const VbTile *__restrict__ tiles, VbBump *bump, uint32_t *ptcl, uint32_t *tile_start, uint2 *cls_list, uint32_t cls_stride) {
    __shared__ uint32_t sh_bitmaps[CO_N_SLICE][VB_N_TILE];
    __shared__ uint32_t sh_part_count[CO_THREADS];
    __shared__ uint32_t sh_part_offsets[CO_THREADS];
    __shared__ uint32_t sh_drawobj_ix[CO_THREADS];
    __shared__ uint32_t sh_tile_stride[CO_THREADS];
    __shared__ uint32_t sh_tile_width[CO_THREADS];
    __shared__ uint32_t sh_tile_x0y0[CO_THREADS];
    __shared__ uint32_t sh_tile_count[CO_THREADS];
    __shared__ uint32_t sh_tile_base[CO_THREADS];
    // per-draw-object fields cached once per 256-element chunk (the WGSL re-reads them from global memory for
    // every (draw, tile) pair: 3-4 dependent loads per pair -> 1)
    __shared__ uint32_t sh_tag[CO_THREADS];    // draw tag
    __shared__ uint32_t sh_dd[CO_THREADS];     // draw data word offset
    __shared__ uint32_t sh_di[CO_THREADS];     // info word offset
    __shared__ uint32_t sh_dflags[CO_THREADS]; // bit0 even-odd, bit1 non-trivial blend (clip objects)
    __shared__ uint32_t sh_scan[CO_THREADS / 32 + 2];

    const uint32_t lid = threadIdx.x;
    // Only PRIOR stages abort coarse (coarse.wgsl:164-179); read once per CTA so the decision is
    // uniform even while other CTAs of this kernel raise VB_STAGE_COARSE (and k_path_tiling, beside it, FINE_SEGMENTS).
    if (lid == 0) sh_scan[0] = bump->failed & VB_STAGES_BEFORE_COARSE;
    __syncthreads();
    const uint32_t prior_failed = sh_scan[0];
    __syncthreads();
    if (prior_failed != 0u) return;
    const uint32_t tile_end = min(bump->tile, cfg.tiles_size), seg_end = bump->segments; // final since k_backdrop
    const uint32_t wg_x = blockIdx.x >> 1, wg_y = (blockIdx.y >> 1) + cfg.win_by0;
    const int32_t qx0 = (int32_t)(blockIdx.x & 1u) * 8, qy0 = (int32_t)(blockIdx.y & 1u) * 8; // quadrant origin in bin tiles
    const uint32_t width_in_bins = (cfg.width_in_tiles + VB_N_TILE_X - 1u) / VB_N_TILE_X;
    const uint32_t height_in_bins = (cfg.height_in_tiles + VB_N_TILE_Y - 1u) / VB_N_TILE_Y;
    const uint32_t bin_ix = width_in_bins * wg_y + wg_x;
    const uint32_t aligned_n_bins = (width_in_bins * height_in_bins * cfg.n_cells + VB_N_TILE - 1u) & ~(VB_N_TILE - 1u);
    // Batch: the bin row (of the tall frame) names the cell; tiles are cell-local below, except for the frame-wide tile index
    // (PTCL, tile_start, fine's queue). Only the partitions that hold draws of the cell are read: [partition_ix, sh_part_end).
    // (The end lives in shared memory: a register more would spill at this occupancy.)
    __shared__ uint32_t sh_part_end;
    uint32_t cell = 0u, partition_ix = 0u;
    if (cfg.n_cells > 1u) {
        cell = wg_y / height_in_bins;
        const uint32_t d0 = __ldg(cfg.cell_draw + cell), d1 = __ldg(cfg.cell_draw + cell + 1u);
        partition_ix = d0 / VB_N_TILE;
        if (lid == 0u) sh_part_end = d1 > d0 ? (d1 + VB_N_TILE - 1u) / VB_N_TILE : partition_ix;
        __syncthreads(); // uniform: n_cells is the launch's
    }
#define n_partitions (cfg.n_cells > 1u ? sh_part_end : (cfg.layout.n_draw_objects + VB_N_TILE - 1u) / VB_N_TILE)
    const uint32_t bin_tile_x = VB_N_TILE_X * wg_x, bin_tile_y = VB_N_TILE_Y * (wg_y - cell * height_in_bins);
    const bool owns_tile = lid < 64u;
    const uint32_t tile_x = (uint32_t)qx0 + (lid & 7u), tile_y = (uint32_t)qy0 + ((lid >> 3) & 7u);
    const uint32_t this_tile_ix = (cell * cfg.height_in_tiles + bin_tile_y + tile_y) * cfg.width_in_tiles + bin_tile_x + tile_x;
    TileState st;
    st.cmd_offset = this_tile_ix * VB_PTCL_INITIAL_ALLOC;
    st.cmd_limit = st.cmd_offset + (VB_PTCL_INITIAL_ALLOC - VB_PTCL_HEADROOM);
    uint32_t clip_zero_depth = 0u, clip_depth = 0u;
    uint32_t rd_ix = 0u, wr_ix = 0u, part_start_ix = 0u, ready_ix = 0u;
    uint32_t render_blend_depth = 0u, max_blend_depth = 0u;
    uint32_t cull_start = 0u; // PTCL offset of the CMD_SOLID of this tile's last opaque full-tile cover (0: none)
    uint32_t cost = 0u;       // estimated work of fine on this tile from its occlusion start (orders fine's tile queue)
    uint32_t emitted = 0u;    // segments of the CMD_FILLs written for this tile
    const uint32_t blend_offset = st.cmd_offset;
    st.cmd_offset += 1u;

    while (true) {
        for (int i = 0; i < CO_N_SLICE; i++) sh_bitmaps[i][lid] = 0u;
        while (true) {
            if (ready_ix == wr_ix && partition_ix < n_partitions) {
                part_start_ix = ready_ix;
                uint32_t count = 0u;
                if (partition_ix + lid < n_partitions) {
                    VbBinHeader h = bin_headers[(size_t)(partition_ix + lid) * aligned_n_bins + bin_ix];
                    count = h.element_count;
                    sh_part_offsets[lid] = h.chunk_offset;
                }
                uint32_t total;
                uint32_t ex = vb_block_excl_scan(count, sh_scan, &total);
                sh_part_count[lid] = part_start_ix + ex + count;
                __syncthreads();
                ready_ix = sh_part_count[CO_THREADS - 1u];
                partition_ix += CO_THREADS;
            }
            uint32_t ix = rd_ix + lid;
            if (ix >= wr_ix && ix < ready_ix) {
                uint32_t part_ix = 0u;
#pragma unroll
                for (uint32_t i = 0u; i < 8u; i++) {
                    uint32_t probe = part_ix + (128u >> i);
                    if (ix >= sh_part_count[probe - 1u]) part_ix = probe;
                }
                ix -= part_ix > 0u ? sh_part_count[part_ix - 1u] : part_start_ix;
                sh_drawobj_ix[lid] = info_bin_data[cfg.layout.bin_data_start + sh_part_offsets[part_ix] + ix];
            }
            wr_ix = min(rd_ix + VB_N_TILE, ready_ix);
            if (wr_ix - rd_ix >= VB_N_TILE || (wr_ix >= ready_ix && partition_ix >= n_partitions)) break;
            __syncthreads();
        }
        __syncthreads();
        uint32_t tag = VB_DRAWTAG_NOP;
        uint32_t drawobj_ix = 0u;
        if (lid + rd_ix < wr_ix) {
            drawobj_ix = sh_drawobj_ix[lid];
            tag = vb_scene(scene, cfg, cfg.layout.draw_tag_base + drawobj_ix);
        }
        uint32_t tile_count = 0u;
        sh_tag[lid] = tag;
        if (tag != VB_DRAWTAG_NOP) {
            const VbDrawMonoid dm0 = draw_monoids[drawobj_ix];
            const uint32_t path_ix = dm0.path_ix;
            const uint32_t dd0 = cfg.layout.draw_data_base + dm0.scene_offset;
            uint32_t fl = info_bin_data[dm0.info_offset] & 1u;
            if ((tag & 1u) != 0u && vb_scene(scene, cfg, dd0) != ((128u << 8) | 3u)) fl |= 2u;
            sh_dd[lid] = dd0;
            sh_di[lid] = dm0.info_offset;
            sh_dflags[lid] = fl;
            const VbPath path = paths[path_ix];
            const uint32_t stride = path.bbox[2] - path.bbox[0];
            sh_tile_stride[lid] = stride;
            const int32_t dx = (int32_t)path.bbox[0] - (int32_t)bin_tile_x;
            const int32_t dy = (int32_t)path.bbox[1] - (int32_t)bin_tile_y;
            const int32_t x0 = vb_clampi(dx, qx0, qx0 + 8);
            const int32_t y0 = vb_clampi(dy, qy0, qy0 + 8);
            const int32_t x1 = vb_clampi((int32_t)path.bbox[2] - (int32_t)bin_tile_x, qx0, qx0 + 8);
            const int32_t y1 = vb_clampi((int32_t)path.bbox[3] - (int32_t)bin_tile_y, qy0, qy0 + 8);
            sh_tile_width[lid] = (uint32_t)(x1 - x0);
            sh_tile_x0y0[lid] = (uint32_t)x0 | ((uint32_t)y0 << 16);
            tile_count = (uint32_t)(x1 - x0) * (uint32_t)(y1 - y0);
            sh_tile_base[lid] = path.tiles - (uint32_t)(dy * (int32_t)stride + dx);
        }
        uint32_t total_tile_count;
        {
            uint32_t ex = vb_block_excl_scan(tile_count, sh_scan, &total_tile_count);
            sh_tile_count[lid] = ex + tile_count;
        }
        __syncthreads();
        for (uint32_t ix0 = lid; ix0 < total_tile_count; ix0 += 2u * VB_N_TILE) {
            uint32_t el[2], tix[2], bit[2];
            CoTile tl[2];
            bool ok[2];
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const uint32_t ix = ix0 + (uint32_t)u * VB_N_TILE;
                ok[u] = ix < total_tile_count;
                uint32_t el_ix = 0u;
                if (ok[u]) {
#pragma unroll
                    for (uint32_t i = 0u; i < 8u; i++) {
                        uint32_t probe = el_ix + (128u >> i);
                        if (ix >= sh_tile_count[probe - 1u]) el_ix = probe;
                    }
                }
                el[u] = el_ix;
                const uint32_t seq_ix = ix - (el_ix > 0u ? sh_tile_count[el_ix - 1u] : 0u);
                const uint32_t width = ok[u] ? sh_tile_width[el_ix] : 1u;
                const uint32_t x0y0 = sh_tile_x0y0[el_ix];
                const uint32_t x = (x0y0 & 0xffffu) + seq_ix % width;
                const uint32_t y = (x0y0 >> 16) + seq_ix / width;
                tix[u] = sh_tile_base[el_ix] + sh_tile_stride[el_ix] * y + x;
                bit[u] = (y - (uint32_t)qy0) * 8u + (x - (uint32_t)qx0);
            }
#pragma unroll
            for (int u = 0; u < 2; u++)
                if (ok[u]) tl[u] = co_load_tile(tiles, tix[u], tile_end, seg_end); // independent loads in flight
#pragma unroll
            for (int u = 0; u < 2; u++) {
                if (!ok[u]) continue;
                const uint32_t el_ix = el[u];
                const uint32_t dtag = sh_tag[el_ix];
                const bool is_clip = (dtag & 1u) != 0u;
                const uint32_t fl = sh_dflags[el_ix];
                const bool is_blend = (fl & 2u) != 0u;
                const bool even_odd = (fl & 1u) != 0u;
                const bool backdrop_clear = (even_odd ? (abs(tl[u].backdrop) & 1) : tl[u].backdrop) == 0;
                const bool include_tile = tl[u].n_segs != 0u || (backdrop_clear == is_clip) || is_blend;
                if (include_tile) atomicOr(&sh_bitmaps[el_ix / 32u][bit[u]], 1u << (el_ix & 31u));
            }
        }
        __syncthreads();

        // emission: each owner walks the set bits of its tile in draw order. The tile record of the NEXT element is
        // requested before the current one is emitted, so the walk is not a chain of exposed global-load latencies.
        uint32_t slice_ix = 0u;
        uint32_t bitmap = owns_tile ? sh_bitmaps[0][lid] : 0u;
        uint32_t nx_el = 0u;
        CoTile nx_tile;
        nx_tile.backdrop = 0; nx_tile.seg_ix = 0u; nx_tile.n_segs = 0u;
        bool nx_have = false;
        auto advance = [&]() {
            nx_have = false;
            while (owns_tile) {
                if (bitmap == 0u) {
                    slice_ix += 1u;
                    if (slice_ix >= CO_N_SLICE) break;
                    bitmap = sh_bitmaps[slice_ix][lid];
                    continue;
                }
                nx_el = slice_ix * 32u + (uint32_t)(__ffs((int)bitmap) - 1);
                bitmap &= bitmap - 1u;
                nx_tile = co_load_tile(tiles, sh_tile_base[nx_el] + sh_tile_stride[nx_el] * tile_y + tile_x, tile_end, seg_end);
                nx_have = true;
                break;
            }
        };
        advance();
        while (nx_have) {
            const uint32_t el_ix = nx_el;
            const CoTile tile = nx_tile;
            advance();
            const uint32_t drawtag = sh_tag[el_ix];
            const uint32_t dd = sh_dd[el_ix];
            const uint32_t di = sh_di[el_ix];
            const uint32_t draw_flags = sh_dflags[el_ix] & 1u; // only the fill-rule bit is defined (drawtag.wgsl:42)
            if (clip_zero_depth == 0u) {
                switch (drawtag) {
                case VB_DRAWTAG_FILL_COLOR: {
                    const uint32_t solid_at = co_write_path(st, tile, draw_flags, cfg, bump, ptcl, emitted, cost);
                    const uint32_t rgba = vb_scene(scene, cfg, dd);
                    co_alloc_cmd(st, 2u, cfg, bump, ptcl);
                    ptcl[st.cmd_offset] = VB_CMD_COLOR;
                    ptcl[st.cmd_offset + 1u] = rgba;
                    st.cmd_offset += 2u;
                    // an opaque colour over the whole tile, outside any clip: nothing emitted so far can show through
                    cost += 2u;
                    if (solid_at != 0u && (rgba >> 24) == 0xffu && render_blend_depth == 0u) {
                        cull_start = solid_at;
                        cost = 3u; // fine starts here: everything before is never executed
                    }
                    break;
                }
                case VB_DRAWTAG_BLURRED_ROUNDED_RECT:
                    co_write_path(st, tile, draw_flags, cfg, bump, ptcl, emitted, cost);
                    co_alloc_cmd(st, 3u, cfg, bump, ptcl);
                    ptcl[st.cmd_offset] = VB_CMD_BLUR_RECT;
                    ptcl[st.cmd_offset + 1u] = di + 1u;
                    ptcl[st.cmd_offset + 2u] = vb_scene(scene, cfg, dd);
                    st.cmd_offset += 3u;
                    cost += 24u;
                    break;
                case VB_DRAWTAG_FILL_LIN_GRADIENT:
                case VB_DRAWTAG_FILL_RAD_GRADIENT:
                case VB_DRAWTAG_FILL_SWEEP_GRADIENT: {
                    const uint32_t ty = drawtag == VB_DRAWTAG_FILL_LIN_GRADIENT ? VB_CMD_LIN_GRAD
                                        : drawtag == VB_DRAWTAG_FILL_RAD_GRADIENT ? VB_CMD_RAD_GRAD : VB_CMD_SWEEP_GRAD;
                    co_write_path(st, tile, draw_flags, cfg, bump, ptcl, emitted, cost);
                    co_alloc_cmd(st, 3u, cfg, bump, ptcl);
                    ptcl[st.cmd_offset] = ty;
                    ptcl[st.cmd_offset + 1u] = vb_scene(scene, cfg, dd);
                    ptcl[st.cmd_offset + 2u] = di + 1u;
                    st.cmd_offset += 3u;
                    cost += 8u;
                    break;
                }
                case VB_DRAWTAG_FILL_IMAGE:
                    co_write_path(st, tile, draw_flags, cfg, bump, ptcl, emitted, cost);
                    co_alloc_cmd(st, 2u, cfg, bump, ptcl);
                    ptcl[st.cmd_offset] = VB_CMD_IMAGE;
                    ptcl[st.cmd_offset + 1u] = di + 1u;
                    st.cmd_offset += 2u;
                    cost += 16u;
                    break;
                case VB_DRAWTAG_BEGIN_CLIP: {
                    const bool even_odd = (draw_flags & 1u) != 0u;
                    const bool backdrop_clear = (even_odd ? (abs(tile.backdrop) & 1) : tile.backdrop) == 0;
                    if (tile.n_segs == 0u && backdrop_clear) {
                        clip_zero_depth = clip_depth + 1u;
                    } else {
                        co_alloc_cmd(st, 1u, cfg, bump, ptcl);
                        ptcl[st.cmd_offset] = VB_CMD_BEGIN_CLIP;
                        st.cmd_offset += 1u;
                        render_blend_depth += 1u;
                        max_blend_depth = max(max_blend_depth, render_blend_depth);
                        cost += 4u;
                    }
                    clip_depth += 1u;
                    break;
                }
                case VB_DRAWTAG_END_CLIP:
                    clip_depth -= 1u;
                    co_write_path(st, tile, draw_flags, cfg, bump, ptcl, emitted, cost);
                    co_alloc_cmd(st, 3u, cfg, bump, ptcl);
                    ptcl[st.cmd_offset] = VB_CMD_END_CLIP;
                    ptcl[st.cmd_offset + 1u] = vb_scene(scene, cfg, dd);
                    ptcl[st.cmd_offset + 2u] = vb_scene(scene, cfg, dd + 1u);
                    st.cmd_offset += 3u;
                    render_blend_depth -= 1u;
                    cost += 8u;
                    break;
                default: break;
                }
            } else {
                if (drawtag == VB_DRAWTAG_BEGIN_CLIP) {
                    clip_depth += 1u;
                } else if (drawtag == VB_DRAWTAG_END_CLIP) {
                    if (clip_depth == clip_zero_depth) clip_zero_depth = 0u;
                    clip_depth -= 1u;
                }
            }
        }
        rd_ix += VB_N_TILE;
        if (rd_ix >= ready_ix && partition_ix >= n_partitions) break;
        __syncthreads();
    }
    if (owns_tile && bin_tile_x + tile_x < cfg.width_in_tiles && bin_tile_y + tile_y < cfg.height_in_tiles) {
        ptcl[st.cmd_offset] = VB_CMD_END;
        uint32_t blend_ix = 0u;
        if (max_blend_depth > VB_BLEND_STACK_SPLIT) {
            const uint32_t scratch_size = (max_blend_depth - VB_BLEND_STACK_SPLIT) * VB_TILE_WIDTH * VB_TILE_HEIGHT;
            blend_ix = atomicAdd(&bump->blend, scratch_size);
            if (blend_ix + scratch_size > cfg.blend_size) atomicOr(&bump->failed, VB_STAGE_COARSE);
        }
        ptcl[blend_offset] = blend_ix;
        tile_start[this_tile_ix] = cull_start;
    }
    // fine's tile queue, heaviest first: every tile of the window goes into one of VB_FINE_CLASSES lists by its estimated cost
    // (one atomic per warp and class; fine walks the lists in class order, so the long tiles start at time zero instead of
    // turning up at the tail of a persistent kernel that has nothing left to overlap them with)
    if (lid < 64u) { // the two owner warps, whole
        const uint32_t ty = bin_tile_y + tile_y, tx = bin_tile_x + tile_x; // ty: row in the cell; the list takes frame rows
        const bool in_win = tx < cfg.width_in_tiles && ty >= cfg.win_ty0 && ty < cfg.win_ty1 && ty < cfg.height_in_tiles;
        // classes by powers of two of the estimate: >= 1024, 512, 256, 128, 64, 32, 16, rest
        const uint32_t lg = 31u - (uint32_t)__clz((int)max(cost, 1u));
        const uint32_t cls = lg >= 10u ? 0u : (lg <= 3u ? 7u : 10u - lg);
        const uint32_t lane = lid & 31u;
#pragma unroll
        for (uint32_t k = 0; k < VB_FINE_CLASSES; k++) {
            const uint32_t m = __ballot_sync(VB_FULL, in_win && cls == k);
            if (m == 0u) continue;
            uint32_t base = 0u;
            if (lane == (uint32_t)(__ffs((int)m) - 1)) base = atomicAdd(reinterpret_cast<uint32_t *>(bump) + VB_CTL_FINE_CLASS + k, (uint32_t)__popc(m));
            base = __shfl_sync(VB_FULL, base, __ffs((int)m) - 1);
            if (in_win && cls == k) {
                const uint32_t slot = base + (uint32_t)__popc(m & ((1u << lane) - 1u));
                if (slot < cls_stride) cls_list[(size_t)k * cls_stride + slot] = make_uint2(this_tile_ix - cfg.win_ty0 * cfg.width_in_tiles, cull_start);
            }
        }
        // the slots these fills use are not holes (k_backdrop set holes to every slot of the frame)
        const uint32_t used = vb_warp_sum(emitted);
        if (lane == 0u && used != 0u) atomicSub(reinterpret_cast<uint32_t *>(bump) + VB_CTL_SEG_HOLES, used);
    }
#undef n_partitions
}

// The segments-arena overflow check (the reference sizes `segments` statically and never checks) lives at the top of
// k_path_tiling, which runs beside coarse.

extern "C" uint32_t vb_launch_coarse(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    uint32_t width_in_bins = (cfg.width_in_tiles + 15u) / 16u;
    uint32_t rows = cfg.win_by1 - cfg.win_by0;
    if (cfg.n_cells > 1u) rows *= cfg.n_cells; // a batch has no window: every cell's bin rows, stacked
    if (width_in_bins == 0 || rows == 0) return 0;
    dim3 grid(width_in_bins * 2u, rows * 2u); // four quadrant CTAs per bin
    k_coarse<<<grid, CO_THREADS, 0, st>>>(cfg, b.scene, b.draw_monoids, b.bin_headers, b.info_bin_data, b.paths, b.tiles, b.bump(), b.ptcl,
                                          b.tile_start, b.cls_list, cfg.width_in_tiles * cfg.tile_rows);
    return 1;
}
