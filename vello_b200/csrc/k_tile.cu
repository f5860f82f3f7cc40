// k_tile.cu -- tile_alloc and backdrop.
//
// Reference: vello_shaders/shader/tile_alloc.wgsl:36-123 (CPU twin cpu/tile_alloc.rs),
// backdrop_dyn.wgsl:29-86 (CPU twin cpu/backdrop.rs).
//
// Design: tile_alloc's per-workgroup atomicAdd(bump.tile) becomes a decoupled look-back scan,
// so `Path.tiles` offsets are deterministic and equal to the serial CPU shader's -- `tiles[]` can be
// compared byte for byte. The allocated range is zeroed by a grid-wide pass (k_tile_zero). backdrop scans the arena
// in one pass of fixed chunks and also assigns every tile its segment slice, which the reference leaves to
// coarse, so that path_tiling and coarse can run side by side (see k_backdrop).
// Extension: tile rows are clamped to the stripe window [win_ty0, win_ty1).
#include "vb_device.cuh"
#include "vb_stages.h"

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
// tile_alloc hands out tiles in draw order, so the arena is the rows of all paths laid end to end, and both results are
// scans over it in tile order: the backdrop a sum segmented at row starts, the slices (the reference allocates one per
// CMD_FILL in coarse, coarse.wgsl:100) an exclusive sum of the crossing counts path_count left in `segment_count_or_ix`.
// ONE pass over the arena: it is cut into fixed chunks of BD_CHUNK tiles, taken by ticket in arena order. A CTA copies its
// chunk into shared memory with coalesced 16-byte loads, and every thread then owns BD_PER_THREAD consecutive tiles: it
// walks them serially (a few integer operations per tile), a warp-shuffle scan combines the threads, and a decoupled
// look-back over the chunks carries {crossings, row start seen, backdrop since the last row start} (BdSegOp). Each thread
// walks its tiles again from its exclusive prefix, and the chunk leaves with coalesced stores, every tile written whole:
// {backdrop, ~first slot of its slice}. Integer sums: the same words whatever the order of evaluation.
// Why serial per thread: a 32-tile warp-shuffle scan costs ~150 warp instructions (two scans, a path search and a modulo
// per tile), and a zero delta does not let a group skip it while a filled row carries a backdrop through it, so the
// scans bounded the kernel; a walk costs a few instructions per tile, there is one shuffle scan per 32 x 16 tiles, and a
// thread's column only needs a path search when its walk reaches the next path.
// A tile's count is the difference to the next tile's slice start (the arena's last tile ends at bump.segments), so
// coarse recovers it without another buffer. bump.segments is the total, which includes the slices of tiles that coarse
// turns into no CMD_FILL; ctl[VB_CTL_SEG_HOLES] starts at the total and coarse subtracts what its fills take, so
// `bump.segments - holes` is the reference's count.
// Row starts: tile t starts a row when (t - first tile of its path) % width == 0, its path being the last one whose first
// tile is <= t (Path.tiles is monotone in draw order; an empty path shares its successor's start, so it never owns a
// tile). A CTA finds the first and last path of its chunk by a 32-ary search of paths[] and stages up to BD_STAGE paths
// in shared memory. A chunk overlaps at most BD_CHUNK non-empty paths but any number of empty ones between them, so a
// chunk over more than BD_STAGE paths searches paths[] in global memory instead (the same answer, slower).
#define BD_THREADS 256
#define BD_WARPS (BD_THREADS / 32)
#define BD_PER_THREAD 16u                          // consecutive tiles of one thread
#define BD_CHUNK (BD_THREADS * BD_PER_THREAD)      // 4096 tiles per CTA
#define BD_ROW4 (BD_PER_THREAD / 2u + 1u)          // int4 per thread in shared memory: one of padding makes the 16-byte
                                                   // accesses of 8 consecutive threads hit distinct banks
#define BD_STAGE 256u

// The last path p < n whose first tile is <= t (paths[0].tiles is 0), by a warp-wide 32-ary search: ceil(log32 n) rounds
// of one load per lane. Call from a whole warp.
__device__ __forceinline__ uint32_t bd_find_path(const VbPath *__restrict__ paths, uint32_t n, uint32_t t) {
    uint32_t lo = 0u, hi = n; // paths[lo].tiles <= t, and paths[hi].tiles > t or hi == n
    while (hi - lo > 1u) {
        const uint32_t step = (hi - lo + 31u) / 32u, q = lo + vb_lane() * step;
        const bool le = q < hi && __ldg(&paths[q].tiles) <= t;
        const uint32_t j = 31u - (uint32_t)__clz(__ballot_sync(VB_FULL, le)); // lane 0 (q = lo) always holds
        lo += j * step;
        hi = min(hi, lo + step);
    }
    return lo;
}

__global__ void __launch_bounds__(BD_THREADS)
k_backdrop(VbConfig cfg, VbBump *bump, const VbPath *__restrict__ paths, VbTile *tiles, uint32_t *lb_mem, uint32_t n_parts) {
    __shared__ int4 sh_tiles[BD_THREADS * BD_ROW4];             // the chunk: thread i's tiles in row i, two per int4
    __shared__ uint32_t sh_start[BD_STAGE], sh_width[BD_STAGE]; // the chunk's paths: first tile, row width
    __shared__ uint32_t sh_pre[BD_WARPS][3];                    // each warp's aggregate, then its exclusive prefix
    __shared__ uint32_t sh_path[2];                             // the chunk's first and last path
    __shared__ uint32_t sh_ticket;
    // path_count's worklist overflow (the WGSL checks it at the top of coarse) is detected here, by every CTA alike, and
    // published by one thread: a separate one-thread check kernel used to sit on the frame's critical path
    const bool pc_overflow = bump->seg_counts > cfg.seg_counts_size;
    if (pc_overflow && blockIdx.x == 0u && threadIdx.x == 0u) atomicOr(&bump->failed, VB_STAGE_PATH_COUNT);
    if (bump->failed != 0u || pc_overflow) return; // uniform: every CTA returns, or none (the look-back needs all)
    // The grid covers the arena's capacity; CTAs past its end take no ticket, so the chunks 0 .. n_chunks - 1 are taken
    // by the first n_chunks CTAs. Chunk 0 always runs: an empty arena still publishes bump.segments.
    const uint32_t arena_end = min(bump->tile, cfg.tiles_size);
    const uint32_t n_chunks = max(arena_end / BD_CHUNK + (arena_end % BD_CHUNK != 0u ? 1u : 0u), 1u);
    if (blockIdx.x >= n_chunks) return;
    const VbLookback lb = vb_lookback_view(lb_mem, n_parts, 3);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t lane = vb_lane(), warp = threadIdx.x >> 5;
    const uint32_t c0 = part * BD_CHUNK, n = min(c0 + BD_CHUNK, arena_end) - c0; // this chunk: tiles [c0, c0 + n)
    // int4 g of the chunk holds its tiles 2g and 2g + 1 (c0 is a multiple of BD_CHUNK: 16-byte aligned)
    int4 in[BD_PER_THREAD / 2u];
#pragma unroll
    for (uint32_t k = 0; k < BD_PER_THREAD / 2u; k++) {
        const uint32_t g = k * BD_THREADS + threadIdx.x;
        if (2u * g + 1u < n) in[k] = reinterpret_cast<const int4 *>(tiles + c0)[g];
        else if (2u * g < n) {
            const int2 t = reinterpret_cast<const int2 *>(tiles)[c0 + 2u * g];
            in[k] = make_int4(t.x, t.y, 0, 0);
        } else in[k] = make_int4(0, 0, 0, 0);
    }
    if (n > 0u && warp < 2u) { // while the loads are in flight
        const uint32_t p = bd_find_path(paths, cfg.layout.n_draw_objects, warp == 0u ? c0 : c0 + n - 1u);
        if (lane == 0u) sh_path[warp] = p;
    }
#pragma unroll
    for (uint32_t k = 0; k < BD_PER_THREAD / 2u; k++) {
        const uint32_t g = k * BD_THREADS + threadIdx.x;
        sh_tiles[(g / (BD_PER_THREAD / 2u)) * BD_ROW4 + g % (BD_PER_THREAD / 2u)] = in[k];
    }
    __syncthreads();
    const uint32_t P0 = sh_path[0], n_stage = n > 0u ? sh_path[1] - P0 + 1u : 0u;
    const bool staged = n_stage <= BD_STAGE;
    if (staged && threadIdx.x < n_stage) {
        const VbPath &p = paths[P0 + threadIdx.x];
        sh_start[threadIdx.x] = __ldg(&p.tiles);
        sh_width[threadIdx.x] = max(__ldg(&p.bbox[2]) - __ldg(&p.bbox[0]), 1u);
    }
    __syncthreads();
    // t's column in its row; w = the row's width, next = the first tile of the next path (t's column is valid until there)
    auto locate = [&](uint32_t t, uint32_t &w, uint32_t &next) -> uint32_t {
        uint32_t lo = 0u, m = n_stage, start; // the path is one of lo .. lo + m - 1 (counted from P0)
        if (staged) {
            while (m > 1u) {
                const uint32_t h = m >> 1;
                const bool le = sh_start[lo + h] <= t;
                lo = le ? lo + h : lo;
                m = le ? m - h : h;
            }
            start = sh_start[lo];
            w = sh_width[lo];
            next = lo + 1u < n_stage ? sh_start[lo + 1u] : 0xffffffffu;
        } else {
            while (m > 1u) {
                const uint32_t h = m >> 1;
                const bool le = __ldg(&paths[P0 + lo + h].tiles) <= t;
                lo = le ? lo + h : lo;
                m = le ? m - h : h;
            }
            const VbPath &p = paths[P0 + lo];
            start = __ldg(&p.tiles);
            w = max(__ldg(&p.bbox[2]) - __ldg(&p.bbox[0]), 1u);
            next = lo + 1u < n_stage ? __ldg(&paths[P0 + lo + 1u].tiles) : 0xffffffffu;
        }
        return (t - start) % w;
    };
    // my tiles [t0, t0 + mine) of the arena: which start a row (bit i), and my aggregate
    int4 *row = sh_tiles + threadIdx.x * BD_ROW4;
    const uint32_t l0 = threadIdx.x * BD_PER_THREAD, mine = n > l0 ? min(n - l0, BD_PER_THREAD) : 0u, t0 = c0 + l0;
    uint32_t starts = 0u, cnt = 0u, sum = 0u;
    if (mine > 0u) {
        uint32_t w, next, x = locate(t0, w, next);
#pragma unroll
        for (uint32_t i = 0; i < BD_PER_THREAD; i++) {
            if (i >= mine) break;
            if (i > 0u) {
                if (t0 + i >= next) x = locate(t0 + i, w, next);
                else x = x + 1u == w ? 0u : x + 1u;
            }
            const int4 q = row[i / 2u];
            if (x == 0u) {
                starts |= 1u << i;
                sum = 0u;
            }
            sum += (uint32_t)(i % 2u ? q.z : q.x);
            cnt += (uint32_t)(i % 2u ? q.w : q.y);
        }
    }
    // the threads' inclusive scan inside the warp (a lower lane is earlier), the warps' in warp 0, the look-back
    uint32_t incl[3] = {cnt, starts != 0u ? 1u : 0u, sum}, before[3];
#pragma unroll
    for (uint32_t o = 1u; o < 32u; o <<= 1) {
        uint32_t u[3];
#pragma unroll
        for (int k = 0; k < 3; k++) u[k] = __shfl_up_sync(VB_FULL, incl[k], o);
        if (lane >= o) BdSegOp::combine(u, incl, incl);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        before[k] = __shfl_up_sync(VB_FULL, incl[k], 1);
        if (lane == 0u) before[k] = 0u;
    }
    if (lane == 31u) {
#pragma unroll
        for (int k = 0; k < 3; k++) sh_pre[warp][k] = incl[k];
    }
    __syncthreads();
    if (warp == 0u) {
        uint32_t wincl[3] = {0u, 0u, 0u}, wbefore[3], agg[3], excl[3];
        if (lane < BD_WARPS) {
#pragma unroll
            for (int k = 0; k < 3; k++) wincl[k] = sh_pre[lane][k];
        }
#pragma unroll
        for (uint32_t o = 1u; o < BD_WARPS; o <<= 1) {
            uint32_t u[3];
#pragma unroll
            for (int k = 0; k < 3; k++) u[k] = __shfl_up_sync(VB_FULL, wincl[k], o);
            if (lane >= o) BdSegOp::combine(u, wincl, wincl);
        }
#pragma unroll
        for (int k = 0; k < 3; k++) agg[k] = __shfl_sync(VB_FULL, wincl[k], BD_WARPS - 1);
        vb_lookback<3, BdSegOp>(lb, part, agg, excl);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            wbefore[k] = __shfl_up_sync(VB_FULL, wincl[k], 1);
            if (lane == 0u) wbefore[k] = 0u;
        }
        BdSegOp::combine(excl, wbefore, wbefore);
        if (lane < BD_WARPS) {
#pragma unroll
            for (int k = 0; k < 3; k++) sh_pre[lane][k] = wbefore[k];
        }
        if (lane == 0u && part == n_chunks - 1u) {
            bump->segments = excl[0] + agg[0];
            reinterpret_cast<uint32_t *>(bump)[VB_CTL_SEG_HOLES] = excl[0] + agg[0]; // coarse subtracts its fills
        }
    }
    __syncthreads();
    // My tiles again, from my exclusive prefix. The carry is the backdrop of the tiles left of t0 in t0's row: the prefix's
    // sum since its last row start, which is t0's own row start whenever t0 does not start a row itself.
    {
        uint32_t pre[3] = {sh_pre[warp][0], sh_pre[warp][1], sh_pre[warp][2]};
        BdSegOp::combine(pre, before, pre);
        uint32_t slice = pre[0], carry = pre[2];
#pragma unroll
        for (uint32_t j = 0; j < BD_PER_THREAD / 2u; j++) {
            if (2u * j >= mine) break;
            const int4 q = row[j];
            int4 out;
            carry = ((starts >> (2u * j)) & 1u ? 0u : carry) + (uint32_t)q.x;
            out.x = (int32_t)carry;
            out.y = (int32_t)~slice;
            slice += (uint32_t)q.y;
            carry = ((starts >> (2u * j + 1u)) & 1u ? 0u : carry) + (uint32_t)q.z;
            out.z = (int32_t)carry;
            out.w = (int32_t)~slice;
            slice += (uint32_t)q.w;
            row[j] = out;
        }
    }
    __syncthreads();
#pragma unroll
    for (uint32_t k = 0; k < BD_PER_THREAD / 2u; k++) {
        const uint32_t g = k * BD_THREADS + threadIdx.x;
        const int4 v = sh_tiles[(g / (BD_PER_THREAD / 2u)) * BD_ROW4 + g % (BD_PER_THREAD / 2u)];
        if (2u * g + 1u < n) reinterpret_cast<int4 *>(tiles + c0)[g] = v;
        else if (2u * g < n) reinterpret_cast<int2 *>(tiles)[c0 + 2u * g] = make_int2(v.x, v.y);
    }
}

extern "C" uint32_t vb_launch_tile_alloc(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (b.parts_tile == 0) return 0;
    k_tile_alloc<<<b.parts_tile, TA_THREADS, 0, st>>>(cfg, b.scene, b.draw_bboxes, b.bump(), b.paths, b.tiles, b.lb_tile, b.parts_tile);
    k_tile_zero<<<(uint32_t)b.sm_count * 4u, 256, 0, st>>>(cfg, b.bump(), b.tiles);
    return 2;
}
extern "C" uint32_t vb_tile_alloc_parts(uint32_t n_draw) { return (n_draw + TA_THREADS - 1) / TA_THREADS; }
// look-back partitions of k_backdrop: the chunks of the tile arena's capacity (CTAs past bump.tile exit at once)
extern "C" uint32_t vb_backdrop_parts(uint32_t tiles_size) {
    const uint32_t n = tiles_size / BD_CHUNK + (tiles_size % BD_CHUNK != 0u ? 1u : 0u);
    return n ? n : 1u;
}
extern "C" uint32_t vb_launch_backdrop(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (cfg.layout.n_draw_objects == 0) return 0;
    k_backdrop<<<b.parts_backdrop, BD_THREADS, 0, st>>>(cfg, b.bump(), b.paths, b.tiles, b.lb_backdrop, b.parts_backdrop);
    return 1;
}
