// k_tile.cu -- tile_alloc and backdrop.
//
// Reference: vello_shaders/shader/tile_alloc.wgsl:36-123 (CPU twin cpu/tile_alloc.rs),
// backdrop_dyn.wgsl:29-86 (CPU twin cpu/backdrop.rs).
//
// Design: tile_alloc's per-workgroup atomicAdd(bump.tile) becomes a decoupled look-back scan,
// so `Path.tiles` offsets are deterministic and equal to the serial CPU shader's -- `tiles[]` can be
// compared byte for byte. The allocated range is zeroed by a grid-wide pass (k_tile_zero). backdrop streams the
// arena as contiguous per-CTA ranges (see k_backdrop).
// Extension: tile rows are clamped to the stripe window [win_ty0, win_ty1).
#include "vb_device.cuh"

#define TA_THREADS 256

__global__ void __launch_bounds__(TA_THREADS)
k_tile_alloc(VbConfig cfg, const uint32_t *__restrict__ scene, const VbBbox4 *__restrict__ draw_bboxes, VbBump *bump, VbPath *paths,
             VbTile *tiles, uint32_t *lb_mem, uint32_t n_parts) {
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_scan[TA_THREADS / 32 + 2];
    __shared__ uint32_t sh_base;
    if (bump->failed & (VB_STAGE_BINNING | VB_STAGE_FLATTEN)) return; // uniform: set only by earlier kernels
    VbLookback lb = vb_lookback_view(lb_mem, n_parts, 1);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t drawobj_ix = part * TA_THREADS + threadIdx.x;
    const float SX = 1.0f / 16.0f, SY = 1.0f / 16.0f;
    uint32_t drawtag = VB_DRAWTAG_NOP;
    if (drawobj_ix < cfg.layout.n_draw_objects) drawtag = vb_scene(scene, cfg, cfg.layout.draw_tag_base + drawobj_ix);
    int32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (drawtag != VB_DRAWTAG_NOP && drawtag != VB_DRAWTAG_END_CLIP) {
        VbBbox4 b = draw_bboxes[drawobj_ix];
        if (b.x0 < b.x1 && b.y0 < b.y1) {
            x0 = vb_f2i_sat(floorf(b.x0 * SX));
            y0 = vb_f2i_sat(floorf(b.y0 * SY));
            x1 = vb_f2i_sat(ceilf(b.x1 * SX));
            y1 = vb_f2i_sat(ceilf(b.y1 * SY));
        }
    }
    const uint32_t ux0 = (uint32_t)vb_clampi(x0, 0, (int32_t)cfg.width_in_tiles);
    const uint32_t ux1 = (uint32_t)vb_clampi(x1, 0, (int32_t)cfg.width_in_tiles);
    const uint32_t uy0 = (uint32_t)vb_clampi(y0, (int32_t)cfg.win_ty0, (int32_t)cfg.win_ty1);
    const uint32_t uy1 = (uint32_t)vb_clampi(y1, (int32_t)cfg.win_ty0, (int32_t)cfg.win_ty1);
    const uint32_t tile_count = (ux1 - ux0) * (uy1 - uy0);
    uint32_t total;
    const uint32_t local_off = vb_block_excl_scan(tile_count, sh_scan, &total);
    if (threadIdx.x < 32) {
        uint32_t agg[1] = {total}, excl[1];
        vb_lookback<1>(lb, part, agg, excl);
        if (threadIdx.x == 0) {
            sh_base = excl[0];
            if (part == n_parts - 1) {
                bump->tile = excl[0] + total;
                if (excl[0] + total > cfg.tiles_size) atomicOr(&bump->failed, VB_STAGE_TILE_ALLOC);
            }
        }
    }
    __syncthreads();
    const uint32_t base = sh_base;
    if (drawobj_ix < cfg.layout.n_draw_objects) {
        VbPath p;
        p.bbox[0] = ux0; p.bbox[1] = uy0; p.bbox[2] = ux1; p.bbox[3] = uy1;
        p.tiles = base + local_off;
        p._pad[0] = p._pad[1] = p._pad[2] = 0;
        paths[drawobj_ix] = p;
    }
}

// Tiles start zeroed (tile_alloc.wgsl:100-107 does this per workgroup). A grid-wide pass instead: a scene with a few
// huge paths (one CTA of tile_alloc owning 500k tiles) is zeroed at full bandwidth.
__global__ void __launch_bounds__(256) k_tile_zero(VbConfig cfg, const VbBump *__restrict__ bump, VbTile *tiles) {
    const uint32_t end = min(bump->tile, cfg.tiles_size);
    uint4 *t4 = reinterpret_cast<uint4 *>(tiles);
    const uint32_t n4 = end / 2u;
    for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n4; i += gridDim.x * 256u) t4[i] = make_uint4(0u, 0u, 0u, 0u);
    if ((end & 1u) != 0u && blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<uint2 *>(tiles)[end - 1u] = make_uint2(0u, 0u);
}

// backdrop: per (path, tile row) inclusive prefix sum along x (backdrop_dyn.wgsl:66-84).
// Design: the WGSL assigns one thread per row, walking 8-byte tiles at a stride of the row width (uncoalesced).
// tile_alloc hands out tiles in draw order, so the tiles of 32 consecutive paths are ONE contiguous range of the arena,
// made of rows laid end to end. A CTA owns that range; it is cut into 8 x gridDim.y pieces of equal size, each piece
// moved to whole-row boundaries, and one warp streams its piece 128 consecutive tiles at a time (four independent
// coalesced loads per lane in flight) through a segmented warp-shuffle scan whose segments are the rows. Groups whose
// deltas are all zero -- most of the arena -- are skipped after the load. Integer sums: identical results.
#define BD_THREADS 256
#define BD_WARPS (BD_THREADS / 32)
#define BD_PATHS 32u // paths per CTA
__global__ void __launch_bounds__(BD_THREADS)
k_backdrop(VbConfig cfg, VbBump *bump, const VbPath *__restrict__ paths, VbTile *tiles) {
    __shared__ uint32_t sh_start[BD_PATHS + 1]; // first tile of each path, then the end of the range
    __shared__ uint32_t sh_width[BD_PATHS];
    // path_count's worklist overflow (the WGSL checks it at the top of coarse) is detected here, by every CTA alike, and
    // published by one thread: a separate one-thread check kernel used to sit on the frame's critical path
    const bool pc_overflow = bump->seg_counts > cfg.seg_counts_size;
    if (pc_overflow && blockIdx.x == 0u && blockIdx.y == 0u && threadIdx.x == 0u) atomicOr(&bump->failed, VB_STAGE_PATH_COUNT);
    if (bump->failed != 0u || pc_overflow) return;
    const uint32_t n_draw = cfg.layout.n_draw_objects;
    const uint32_t p0 = blockIdx.x * BD_PATHS;
    const uint32_t arena_end = min(bump->tile, cfg.tiles_size);
    if (threadIdx.x <= BD_PATHS) {
        const uint32_t p = p0 + threadIdx.x;
        uint32_t start = arena_end, width = 0u;
        if (p < n_draw) {
            const VbPath path = paths[p];
            start = min(path.tiles, arena_end);
            width = path.bbox[2] - path.bbox[0];
        }
        sh_start[threadIdx.x] = start;
        if (threadIdx.x < BD_PATHS) sh_width[threadIdx.x] = width;
    }
    __syncthreads();
    const uint32_t lane = vb_lane();
    const uint32_t r0 = sh_start[0], r1 = sh_start[BD_PATHS];
    if (r1 <= r0) return;
    // the path owning tile t (the last path starting at or before t; empty paths share their successor's start) and
    // t's column inside its row
    auto column = [&](uint32_t t, uint32_t &w) -> uint32_t {
        uint32_t p = 0u;
#pragma unroll
        for (uint32_t step = 16u; step > 0u; step >>= 1)
            if (sh_start[p + step] <= t) p += step;
        w = max(sh_width[p], 1u);
        return (t - sh_start[p]) % w;
    };
    auto row_align = [&](uint32_t t) -> uint32_t { // first row start at or after t
        if (t >= r1) return r1;
        uint32_t w;
        const uint32_t x = column(t, w);
        return x == 0u ? t : min(t + (w - x), r1);
    };
    const uint32_t pieces = BD_WARPS * gridDim.y;
    const uint32_t piece = blockIdx.y * BD_WARPS + (threadIdx.x >> 5);
    const uint32_t len = (r1 - r0 + pieces - 1u) / pieces;
    const uint64_t na = (uint64_t)r0 + (uint64_t)piece * len;
    if (na >= r1) return;
    const uint32_t A = row_align((uint32_t)na);
    const uint32_t B = row_align((uint32_t)min((uint64_t)r1, na + len));
    int32_t carry = 0;
    for (uint32_t base = A; base < B; base += 128u) {
        int32_t v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t idx = base + (uint32_t)k * 32u + lane;
            v[k] = idx < B ? tiles[idx].backdrop : 0;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t idx = base + (uint32_t)k * 32u + lane;
            if (!__any_sync(VB_FULL, v[k] != 0) && carry == 0) continue; // nothing to propagate in these 32 tiles
            const bool valid = idx < B;
            uint32_t w;
            const uint32_t x = valid ? column(idx, w) : 0u;
            const uint32_t reach = min(x, lane); // elements of my row to my left inside this 32-tile group
            int32_t s = v[k];
#pragma unroll
            for (uint32_t o = 1u; o < 32u; o <<= 1) {
                const int32_t t = __shfl_up_sync(VB_FULL, s, o);
                if (o <= reach) s += t;
            }
            if (x > lane) s += carry; // my row started in an earlier group
            if (valid && x != 0u && s != v[k]) tiles[idx].backdrop = s;
            carry = __shfl_sync(VB_FULL, s, 31);
        }
    }
}

extern "C" uint32_t vb_launch_tile_alloc(const VbConfig *cfg, const uint32_t *scene, const VbBbox4 *draw_bboxes, VbBump *bump,
                                     VbPath *paths, VbTile *tiles, uint32_t *lb_mem, uint32_t n_parts, int sm_count, cudaStream_t st) {
    if (n_parts == 0) return 0;
    k_tile_alloc<<<n_parts, TA_THREADS, 0, st>>>(*cfg, scene, draw_bboxes, bump, paths, tiles, lb_mem, n_parts);
    k_tile_zero<<<(uint32_t)sm_count * 4u, 256, 0, st>>>(*cfg, bump, tiles);
    return 2;
}
extern "C" uint32_t vb_tile_alloc_parts(uint32_t n_draw) { return (n_draw + TA_THREADS - 1) / TA_THREADS; }
extern "C" uint32_t vb_launch_backdrop(const VbConfig *cfg, VbBump *bump, const VbPath *paths, VbTile *tiles, int sm_count, cudaStream_t st) {
    uint32_t n = cfg->layout.n_draw_objects;
    if (n == 0) return 0;
    const uint32_t groups = (n + BD_PATHS - 1) / BD_PATHS;
    uint32_t split = ((uint32_t)sm_count * 4u + groups - 1u) / groups;
    if (split > 64u) split = 64u;
    k_backdrop<<<dim3(groups, split), BD_THREADS, 0, st>>>(*cfg, bump, paths, tiles);
    return 1;
}
