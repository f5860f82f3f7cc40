// k_tile.cu -- tile_alloc and backdrop.
//
// Reference: vello_shaders/shader/tile_alloc.wgsl:36-123 (CPU twin cpu/tile_alloc.rs),
// backdrop_dyn.wgsl:29-86 (CPU twin cpu/backdrop.rs).
//
// Design: tile_alloc's per-workgroup atomicAdd(bump.tile) becomes a decoupled look-back scan,
// so `Path.tiles` offsets are deterministic and equal to the serial CPU shader's -- `tiles[]` can be
// compared byte for byte. The allocated range is zeroed by a grid-wide pass (k_tile_zero). backdrop streams the
// arena as contiguous per-CTA ranges and also assigns every tile its segment slice, which the reference leaves to
// coarse, so that path_tiling and coarse can run side by side (see k_backdrop).
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

// backdrop: per (path, tile row) inclusive prefix sum along x (backdrop_dyn.wgsl:66-84), and the segment slices.
// Design: the WGSL assigns one thread per row, walking 8-byte tiles at a stride of the row width (uncoalesced).
// tile_alloc hands out tiles in draw order, so the tiles of 32 consecutive paths are ONE contiguous range of the arena,
// made of rows laid end to end. A group of `split` CTAs owns that range; it is cut into 8 x split pieces of equal size,
// each piece moved to whole-row boundaries, and one warp streams its piece 128 consecutive tiles at a time (four
// independent coalesced loads per lane in flight) through a segmented warp-shuffle scan whose segments are the rows.
// Groups whose deltas are all zero -- most of the arena -- skip the scan. Integer sums: identical results.
// Segment slices (the reference allocates one per CMD_FILL in coarse, coarse.wgsl:100): path_count left each tile's
// crossing count in `segment_count_or_ix`, so an exclusive scan of the counts in tile order gives every (path, tile) its
// slice without waiting for coarse. Each CTA first sums the counts of its pieces, a decoupled look-back over the CTAs
// (ticketed; CTA order = tile order) turns the sums into bases, and the backdrop pass then writes every tile whole:
// {backdrop, ~first slot of its slice}. A tile's count is the difference to the next tile's slice start (the arena's
// last tile ends at bump.segments), so coarse recovers it without another buffer. bump.segments is the total, which
// includes the slices of tiles that coarse turns into no CMD_FILL; ctl[VB_CTL_SEG_HOLES] starts at the total and
// coarse subtracts what its fills take, so `bump.segments - holes` is the reference's count.
#define BD_THREADS 256
#define BD_WARPS (BD_THREADS / 32)
#define BD_PATHS 32u // paths per CTA group
static void bd_grid(uint32_t n_draw, int sm_count, uint32_t *groups, uint32_t *split) {
    *groups = (n_draw + BD_PATHS - 1) / BD_PATHS;
    const uint32_t s = *groups ? ((uint32_t)sm_count * 4u + *groups - 1u) / *groups : 1u;
    *split = s > 64u ? 64u : s;
}
__global__ void __launch_bounds__(BD_THREADS)
k_backdrop(VbConfig cfg, VbBump *bump, const VbPath *__restrict__ paths, VbTile *tiles, uint32_t *lb_mem, uint32_t split) {
    __shared__ uint32_t sh_start[BD_PATHS + 1]; // first tile of each path, then the end of the range
    __shared__ uint32_t sh_width[BD_PATHS];
    __shared__ uint32_t sh_seg[BD_WARPS]; // segments of each warp's piece, then the first slot of the piece
    __shared__ uint32_t sh_ticket;
    // path_count's worklist overflow (the WGSL checks it at the top of coarse) is detected here, by every CTA alike, and
    // published by one thread: a separate one-thread check kernel used to sit on the frame's critical path
    const bool pc_overflow = bump->seg_counts > cfg.seg_counts_size;
    if (pc_overflow && blockIdx.x == 0u && threadIdx.x == 0u) atomicOr(&bump->failed, VB_STAGE_PATH_COUNT);
    if (bump->failed != 0u || pc_overflow) return; // uniform: every CTA returns, or none (the look-back needs all)
    const uint32_t n_parts = gridDim.x;
    const VbLookback lb = vb_lookback_view(lb_mem, n_parts, 1);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t n_draw = cfg.layout.n_draw_objects;
    const uint32_t p0 = (part / split) * BD_PATHS;
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
    // this warp's piece [A, B) (empty when the range has fewer rows than pieces)
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t pieces = BD_WARPS * split;
    const uint32_t piece = (part % split) * BD_WARPS + warp;
    uint32_t A = r1, B = r1;
    if (r1 > r0) {
        const uint32_t len = (r1 - r0 + pieces - 1u) / pieces;
        const uint64_t na = (uint64_t)r0 + (uint64_t)piece * len;
        if (na < r1) {
            A = row_align((uint32_t)na);
            B = row_align((uint32_t)min((uint64_t)r1, na + len));
        }
    }
    // slices: the piece's segment count, the CTA's prefix over its warps, the look-back across CTAs
    uint32_t n_segs = 0u;
    for (uint32_t base = A; base < B; base += 256u) {
        uint32_t c[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint32_t idx = base + (uint32_t)k * 32u + lane;
            c[k] = idx < B ? tiles[idx].segment_count_or_ix : 0u;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) n_segs += c[k];
    }
    n_segs = vb_warp_sum(n_segs);
    if (lane == 0u) sh_seg[warp] = n_segs;
    __syncthreads();
    if (warp == 0u) {
        const uint32_t mine = lane < BD_WARPS ? sh_seg[lane] : 0u;
        const uint32_t incl = vb_warp_incl_scan(mine);
        uint32_t agg[1] = {__shfl_sync(VB_FULL, incl, 31)}, excl[1];
        vb_lookback<1>(lb, part, agg, excl);
        if (lane < BD_WARPS) sh_seg[lane] = excl[0] + incl - mine;
        if (lane == 0u && part == n_parts - 1u) {
            bump->segments = excl[0] + agg[0];
            reinterpret_cast<uint32_t *>(bump)[VB_CTL_SEG_HOLES] = excl[0] + agg[0]; // coarse subtracts its fills
        }
    }
    __syncthreads();
    uint32_t seg_next = sh_seg[warp];
    int32_t carry = 0;
    for (uint32_t base = A; base < B; base += 128u) {
        int2 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t idx = base + (uint32_t)k * 32u + lane;
            v[k] = idx < B ? reinterpret_cast<const int2 *>(tiles)[idx] : make_int2(0, 0);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t idx = base + (uint32_t)k * 32u + lane;
            const bool valid = idx < B;
            const uint32_t count = (uint32_t)v[k].y;
            const uint32_t count_incl = vb_warp_incl_scan(count);
            const uint32_t slice = seg_next + count_incl - count;
            seg_next += __shfl_sync(VB_FULL, count_incl, 31);
            int32_t s = v[k].x;
            if (__any_sync(VB_FULL, s != 0) || carry != 0) { // else nothing to propagate in these 32 tiles
                uint32_t w;
                const uint32_t x = valid ? column(idx, w) : 0u;
                const uint32_t reach = min(x, lane); // elements of my row to my left inside this 32-tile group
#pragma unroll
                for (uint32_t o = 1u; o < 32u; o <<= 1) {
                    const int32_t t = __shfl_up_sync(VB_FULL, s, o);
                    if (o <= reach) s += t;
                }
                if (x > lane) s += carry; // my row started in an earlier group
                carry = __shfl_sync(VB_FULL, s, 31);
            }
            if (valid) reinterpret_cast<int2 *>(tiles)[idx] = make_int2(s, (int32_t)~slice);
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
// look-back partitions of k_backdrop: its CTAs
extern "C" uint32_t vb_backdrop_parts(uint32_t n_draw, int sm_count) {
    uint32_t groups, split;
    bd_grid(n_draw, sm_count, &groups, &split);
    return groups * split;
}
extern "C" uint32_t vb_launch_backdrop(const VbConfig *cfg, VbBump *bump, const VbPath *paths, VbTile *tiles, uint32_t *lb_mem, int sm_count,
                                       cudaStream_t st) {
    uint32_t groups, split;
    bd_grid(cfg->layout.n_draw_objects, sm_count, &groups, &split);
    if (groups == 0) return 0;
    k_backdrop<<<groups * split, BD_THREADS, 0, st>>>(*cfg, bump, paths, tiles, lb_mem, split);
    return 1;
}
