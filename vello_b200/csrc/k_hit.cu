// k_hit.cu -- hit testing (vb_hit_test): the last draw object in draw order that covers each point of the last frame.
//
// No counterpart in the reference (vello's applications hit-test on the host against their own geometry). The kernel only
// reads what a finished frame left on the device: the bins' draw lists (bin_headers / info_bin_data), the draw tags, draw
// monoids and fill-rule flags, the paths' tile boxes, the tiles after backdrop ({backdrop, ~slice start}) and the segments.
// One warp per point: the lanes walk the point's bin list in draw order, 32 draws at a time, each lane computing the winding
// number of its draw's path at the point by the rule fine samples with (tests/tile_walk_ref.py, "the joint contract"): the
// tile's backdrop, plus the sign of every segment whose left-edge crossing y_edge lies at or above the point, plus the
// segments that cross the point's row left of it (decided by the sign of a cross product: f32 can only err within a rounding
// of the line, where the answer is not promised). A ballot of the results feeds the clip state machine coarse runs per tile
// (k_coarse.cu, clip_zero_depth), here per point: a draw inside a BEGIN_CLIP that does not cover the point is skipped up to
// its END_CLIP. A draw whose tile box misses the point's tile does not cover it (binning and tile_alloc clipped its box to
// its enclosing clips and the frame).
#include "vb_device.cuh"
#include "vb_stages.h"

#define HT_THREADS 256
#define HT_WARPS (HT_THREADS / 32)

// w plus what segment g of a tile contributes to the winding number at (sx, sy), the point relative to the tile's corner: its
// sign when its left-edge crossing y_edge lies at or above the point, and its direction when it crosses the point's row left
// of the point. Both kernels take the winding through this one function, so a map and a hit test agree bit for bit (the
// build does not contract to FMA). The by-value form keeps k_hit_test's code what it was before the function existed.
__device__ __forceinline__ int32_t ht_wind(int32_t w, const VbSegment g, float sx, float sy) {
    if (g.y_edge <= sy) w += (g.p1[0] > g.p0[0]) - (g.p1[0] < g.p0[0]);
    if ((g.p0[1] <= sy) != (g.p1[1] <= sy)) {
        // it crosses the row left of the point: (crossing x - sx) * dy < 0, without a division
        const float dy = g.p1[1] - g.p0[1];
        const float c = (g.p0[0] - sx) * dy + (sy - g.p0[1]) * (g.p1[0] - g.p0[0]);
        if (dy > 0.0f ? c < 0.0f : c > 0.0f) w += dy > 0.0f ? -1 : 1;
    }
    return w;
}

__global__ void __launch_bounds__(HT_THREADS)
k_hit_test(VbConfig cfg, const uint32_t *__restrict__ scene, const VbDrawMonoid *__restrict__ draw_monoids,
           const VbBinHeader *__restrict__ bin_headers, const uint32_t *__restrict__ info_bin_data, const VbPath *__restrict__ paths,
           const VbTile *__restrict__ tiles, const VbSegment *__restrict__ segments, const VbBump *__restrict__ bump,
           const float *__restrict__ xy, uint32_t n, int32_t *__restrict__ out) {
    const uint32_t lane = vb_lane();
    const uint32_t tile_end = min(bump->tile, cfg.tiles_size), seg_end = bump->segments;
    const uint32_t wb = (cfg.width_in_tiles + VB_N_TILE_X - 1u) / VB_N_TILE_X, hb = (cfg.height_in_tiles + VB_N_TILE_Y - 1u) / VB_N_TILE_Y;
    const uint32_t aligned_n_bins = (wb * hb * cfg.n_cells + VB_N_TILE - 1u) & ~(VB_N_TILE - 1u);
    for (uint32_t i = blockIdx.x * HT_WARPS + (threadIdx.x >> 5); i < n; i += gridDim.x * HT_WARPS) {
        const float px = xy[2u * (size_t)i], py = xy[2u * (size_t)i + 1u];
        int32_t best = -1;
        // outside the frame, NaN included (every comparison with NaN is false): no draw
        if (px >= 0.0f && py >= 0.0f && px < (float)cfg.target_width && py < (float)(cfg.n_cells * cfg.target_height)) {
            const uint32_t xi = (uint32_t)px, yi = (uint32_t)py; // floor: both are >= 0
            const uint32_t cell = yi / cfg.target_height, yl = yi - cell * cfg.target_height;
            const uint32_t tx = xi / VB_TILE_WIDTH, ty = yl / VB_TILE_HEIGHT;
            // the point relative to its tile, exactly: the tile's corner is an integer no larger than the coordinate
            const float sx = px - (float)(tx * VB_TILE_WIDTH), sy = (py - (float)(cell * cfg.target_height)) - (float)(ty * VB_TILE_HEIGHT);
            const uint32_t bin_ix = wb * (cell * hb + ty / VB_N_TILE_Y) + tx / VB_N_TILE_X;
            // a batch cell's draws sit in the partitions of its draw range (as in k_coarse)
            uint32_t part = 0u, part_end = (cfg.layout.n_draw_objects + VB_N_TILE - 1u) / VB_N_TILE;
            if (cfg.n_cells > 1u) {
                const uint32_t d0 = __ldg(cfg.cell_draw + cell), d1 = __ldg(cfg.cell_draw + cell + 1u);
                part = d0 / VB_N_TILE;
                part_end = d1 > d0 ? (d1 + VB_N_TILE - 1u) / VB_N_TILE : part;
            }
            uint32_t clip_depth = 0u, clip_zero_depth = 0u;
            for (; part < part_end; part++) {
                const VbBinHeader h = bin_headers[(size_t)part * aligned_n_bins + bin_ix];
                for (uint32_t k0 = 0u; k0 < h.element_count; k0 += 32u) {
                    const uint32_t k = k0 + lane;
                    uint32_t tag = VB_DRAWTAG_NOP, drawobj_ix = 0u;
                    bool covers = false;
                    if (k < h.element_count) {
                        drawobj_ix = info_bin_data[cfg.layout.bin_data_start + h.chunk_offset + k];
                        tag = vb_scene(scene, cfg, cfg.layout.draw_tag_base + drawobj_ix);
                    }
                    if (tag != VB_DRAWTAG_NOP) {
                        const VbDrawMonoid dm = draw_monoids[drawobj_ix];
                        const uint4 pb = *reinterpret_cast<const uint4 *>(&paths[dm.path_ix].bbox[0]); // the path's tile box
                        if (tx >= pb.x && tx < pb.z && ty >= pb.y && ty < pb.w) {
                            const uint32_t tix = paths[dm.path_ix].tiles + (ty - pb.y) * (pb.z - pb.x) + (tx - pb.x);
                            const CoTile t = co_load_tile(tiles, tix, tile_end, seg_end);
                            int32_t w = t.backdrop;
                            for (uint32_t s = t.seg_ix; s < t.seg_ix + t.n_segs; s++) {
                                const VbSegment g = segments[s];
                                w = ht_wind(w, g, sx, sy);
                            }
                            const bool even_odd = (info_bin_data[dm.info_offset] & 1u) != 0u;
                            covers = even_odd ? (w & 1) != 0 : w != 0;
                        }
                    }
                    const uint32_t m_cov = __ballot_sync(VB_FULL, covers);
                    const uint32_t m_begin = __ballot_sync(VB_FULL, tag == VB_DRAWTAG_BEGIN_CLIP);
                    const uint32_t m_end = __ballot_sync(VB_FULL, tag == VB_DRAWTAG_END_CLIP);
                    const uint32_t m_hit = m_cov & ~(m_begin | m_end);
                    int top = -1; // the lane of the last draw of this chunk that is hit
                    if ((m_begin | m_end) == 0u) {
                        if (clip_zero_depth == 0u && m_hit != 0u) top = 31 - __clz((int)m_hit);
                    } else {
                        // coarse's per-tile clip state machine, per point, serial over the chunk in draw order (every lane alike)
                        for (int j = 0; j < 32; j++) {
                            const uint32_t bit = 1u << j;
                            if (clip_zero_depth == 0u) {
                                if (m_begin & bit) {
                                    if (!(m_cov & bit)) clip_zero_depth = clip_depth + 1u;
                                    clip_depth += 1u;
                                } else if (m_end & bit) {
                                    clip_depth -= 1u;
                                } else if (m_hit & bit) {
                                    top = j;
                                }
                            } else if (m_begin & bit) {
                                clip_depth += 1u;
                            } else if (m_end & bit) {
                                if (clip_depth == clip_zero_depth) clip_zero_depth = 0u;
                                clip_depth -= 1u;
                            }
                        }
                    }
                    if (top >= 0) best = (int32_t)__shfl_sync(VB_FULL, drawobj_ix, top); // `top` is the same in every lane
                }
            }
        }
        if (lane == 0u) out[i] = best;
    }
}

extern "C" uint32_t vb_launch_hit_test(const VbConfig &cfg, const VbFrameBufs &b, const float *xy, uint32_t n, int32_t *draw_ix,
                                       cudaStream_t st) {
    if (n == 0u) return 0;
    const uint64_t blocks = ((uint64_t)n + HT_WARPS - 1u) / HT_WARPS, most = (uint64_t)b.sm_count * 8u;
    const uint32_t grid = (uint32_t)(blocks < most ? blocks : most);
    k_hit_test<<<grid, HT_THREADS, 0, st>>>(cfg, b.scene, b.draw_monoids, b.bin_headers, b.info_bin_data, b.paths, b.tiles, b.segments,
                                            b.bump(), xy, n, draw_ix);
    return 1;
}

// ---- hit maps (vb_hit_map) -----------------------------------------------------------------------------------------------
// k_hit_test's answer at every pixel centre of a rectangle. One CTA of 256 threads per 16x16 tile the rectangle touches, one
// thread per pixel centre; the centre's offset within its tile is (lx + 0.5, ly + 0.5), exactly what k_hit_test computes for
// the same centre. The tile's 256 pixels share one bin list, one tile record per draw and one segment slice, so the CTA reads
// each once: per step of 256 list entries (a batch cell's own partitions, as in k_hit_test) it keeps, compacted in draw order,
// the draws whose tile box contains the tile and every BEGIN_CLIP / END_CLIP (a BEGIN_CLIP whose box misses the tile covers
// none of it), with the kept draws' tile records. The kept slices then stream through shared memory HM_SEGS segments at a
// time, while every thread sums its own winding per entry and runs coarse's clip state machine. A tile without segments
// needs only its backdrop: nothing is staged for it.
#define HM_SEGS 512u
#define HM_BEGIN 1u // entry kinds; a draw is neither
#define HM_END 2u
#define HM_IN_BOX 4u // the path's tile box contains the tile (only then can it cover a pixel of it)
#define HM_EVEN_ODD 8u

__global__ void __launch_bounds__(HT_THREADS)
k_hit_map(VbConfig cfg, const uint32_t *__restrict__ scene, const VbDrawMonoid *__restrict__ draw_monoids,
          const VbBinHeader *__restrict__ bin_headers, const uint32_t *__restrict__ info_bin_data, const VbPath *__restrict__ paths,
          const VbTile *__restrict__ tiles, const VbSegment *__restrict__ segments, const VbBump *__restrict__ bump, uint32_t x0,
          uint32_t y0, uint32_t w, uint32_t h, uint32_t tx0, uint32_t tr0, uint32_t n_rows, int32_t *__restrict__ out, size_t pitch) {
    __shared__ VbSegment sh_seg[HM_SEGS];
    // a round of up to 256 partitions: the inclusive prefix of their list lengths, and where entry k of the round lies in
    // info_bin_data past bin_data_start (k + sh_part_base of its partition)
    __shared__ uint32_t sh_part_end[HT_THREADS], sh_part_base[HT_THREADS];
    // a step's kept entries in draw order: draw index, HM_* flags, tile backdrop, the inclusive prefix of their slice lengths,
    // and the segment index of slice position s of entry e (sh_seg_base[e] + s, modulo 2^32)
    __shared__ uint32_t sh_draw[HT_THREADS], sh_flags[HT_THREADS], sh_seg_end[HT_THREADS], sh_seg_base[HT_THREADS];
    __shared__ int32_t sh_backdrop[HT_THREADS];
    __shared__ uint32_t sh_scan[HT_WARPS + 1];
    const uint32_t tid = threadIdx.x, lx = tid % VB_TILE_WIDTH, ly = tid / VB_TILE_WIDTH;
    const float sx = (float)lx + 0.5f, sy = (float)ly + 0.5f;
    const uint32_t tile_end = min(bump->tile, cfg.tiles_size), seg_end = bump->segments;
    const uint32_t wb = (cfg.width_in_tiles + VB_N_TILE_X - 1u) / VB_N_TILE_X, hb = (cfg.height_in_tiles + VB_N_TILE_Y - 1u) / VB_N_TILE_Y;
    const uint32_t aligned_n_bins = (wb * hb * cfg.n_cells + VB_N_TILE - 1u) & ~(VB_N_TILE - 1u);
    const uint32_t tx = tx0 + blockIdx.x;
    for (uint32_t row = blockIdx.y; row < n_rows; row += gridDim.y) {
        // tile row `trow` of the tall tile grid: cell `cell`'s tile row ty
        const uint32_t trow = tr0 + row, cell = trow / cfg.height_in_tiles, ty = trow - cell * cfg.height_in_tiles;
        const uint32_t bin_ix = wb * (cell * hb + ty / VB_N_TILE_Y) + tx / VB_N_TILE_X;
        uint32_t part = 0u, part_end = (cfg.layout.n_draw_objects + VB_N_TILE - 1u) / VB_N_TILE;
        if (cfg.n_cells > 1u) {
            const uint32_t d0 = __ldg(cfg.cell_draw + cell), d1 = __ldg(cfg.cell_draw + cell + 1u);
            part = d0 / VB_N_TILE;
            part_end = d1 > d0 ? (d1 + VB_N_TILE - 1u) / VB_N_TILE : part;
        }
        uint32_t clip_depth = 0u, clip_zero_depth = 0u;
        int32_t best = -1;
        // Every shared array is written only after a block scan, whose barriers every thread reaches only once it is done
        // reading what the previous step or round left there.
        for (; part < part_end; part += HT_THREADS) {
            VbBinHeader hd{0u, 0u};
            if (part + tid < part_end) hd = bin_headers[(size_t)(part + tid) * aligned_n_bins + bin_ix];
            uint32_t n_list;
            const uint32_t at = vb_block_excl_scan(hd.element_count, sh_scan, &n_list);
            sh_part_end[tid] = at + hd.element_count;
            sh_part_base[tid] = hd.chunk_offset - at;
            __syncthreads();
            for (uint32_t k0 = 0u; k0 < n_list; k0 += HT_THREADS) {
                const uint32_t k = k0 + tid;
                uint32_t tag = VB_DRAWTAG_NOP, drawobj_ix = 0u, flags = 0u, seg_ix = 0u, n_segs = 0u;
                int32_t backdrop = 0;
                if (k < n_list) {
                    uint32_t p = 0u; // the first partition whose prefix passes k
#pragma unroll
                    for (uint32_t i = 0u; i < 8u; i++) {
                        const uint32_t probe = p + (128u >> i);
                        if (k >= sh_part_end[probe - 1u]) p = probe;
                    }
                    drawobj_ix = info_bin_data[cfg.layout.bin_data_start + sh_part_base[p] + k];
                    tag = vb_scene(scene, cfg, cfg.layout.draw_tag_base + drawobj_ix);
                }
                bool keep = tag == VB_DRAWTAG_BEGIN_CLIP || tag == VB_DRAWTAG_END_CLIP;
                if (tag != VB_DRAWTAG_NOP && tag != VB_DRAWTAG_END_CLIP) { // an END_CLIP's coverage is never asked
                    const VbDrawMonoid dm = draw_monoids[drawobj_ix];
                    const uint4 pb = *reinterpret_cast<const uint4 *>(&paths[dm.path_ix].bbox[0]); // the path's tile box
                    if (tx >= pb.x && tx < pb.z && ty >= pb.y && ty < pb.w) {
                        const uint32_t tix = paths[dm.path_ix].tiles + (ty - pb.y) * (pb.z - pb.x) + (tx - pb.x);
                        const CoTile t = co_load_tile(tiles, tix, tile_end, seg_end);
                        keep = true;
                        backdrop = t.backdrop;
                        seg_ix = t.seg_ix;
                        n_segs = t.n_segs;
                        flags = HM_IN_BOX | ((info_bin_data[dm.info_offset] & 1u) != 0u ? HM_EVEN_ODD : 0u);
                    }
                }
                flags |= tag == VB_DRAWTAG_BEGIN_CLIP ? HM_BEGIN : tag == VB_DRAWTAG_END_CLIP ? HM_END : 0u;
                uint32_t n_kept, n_seg_total;
                const uint32_t e_at = vb_block_excl_scan(keep ? 1u : 0u, sh_scan, &n_kept);
                const uint32_t s_at = vb_block_excl_scan(n_segs, sh_scan, &n_seg_total);
                if (keep) {
                    sh_draw[e_at] = drawobj_ix;
                    sh_flags[e_at] = flags;
                    sh_backdrop[e_at] = backdrop;
                    sh_seg_end[e_at] = s_at + n_segs;
                    sh_seg_base[e_at] = seg_ix - s_at;
                }
                __syncthreads();
                uint32_t e = 0u; // the entry this thread is summing
                int32_t wind = n_kept > 0u ? sh_backdrop[0] : 0;
                for (uint32_t s0 = 0u;; s0 += HM_SEGS) {
                    const uint32_t s1 = min(s0 + HM_SEGS, n_seg_total);
                    for (uint32_t s = s0 + tid; s < s1; s += HT_THREADS) {
                        uint32_t lo = 0u, hi = n_kept - 1u; // the entry holding slice position s: the first whose end passes s
                        while (lo < hi) {
                            const uint32_t mid = (lo + hi) >> 1;
                            if (sh_seg_end[mid] > s) hi = mid;
                            else lo = mid + 1u;
                        }
                        sh_seg[s - s0] = segments[sh_seg_base[lo] + s];
                    }
                    __syncthreads();
                    uint32_t s = s0;
                    for (; e < n_kept; e++) {
                        const uint32_t end = sh_seg_end[e];
                        for (; s < min(end, s1); s++) wind = ht_wind(wind, sh_seg[s - s0], sx, sy);
                        if (end > s1) break; // the entry's slice goes on in the next window
                        const uint32_t f = sh_flags[e];
                        const bool covers = (f & HM_IN_BOX) != 0u && ((f & HM_EVEN_ODD) != 0u ? (wind & 1) != 0 : wind != 0);
                        // coarse's per-tile clip state machine, per pixel
                        if (clip_zero_depth == 0u) {
                            if (f & HM_BEGIN) {
                                if (!covers) clip_zero_depth = clip_depth + 1u;
                                clip_depth += 1u;
                            } else if (f & HM_END) {
                                clip_depth -= 1u;
                            } else if (covers) {
                                best = (int32_t)sh_draw[e];
                            }
                        } else if (f & HM_BEGIN) {
                            clip_depth += 1u;
                        } else if (f & HM_END) {
                            if (clip_depth == clip_zero_depth) clip_zero_depth = 0u;
                            clip_depth -= 1u;
                        }
                        if (e + 1u < n_kept) wind = sh_backdrop[e + 1u];
                    }
                    if (s1 >= n_seg_total) break;
                    __syncthreads(); // the window is summed by every thread before the next overwrites it
                }
            }
        }
        // threads of pixels outside the rectangle (or past the cell's last row) only helped
        const uint32_t yl = ty * VB_TILE_HEIGHT + ly, px = tx * VB_TILE_WIDTH + lx, py = cell * cfg.target_height + yl;
        if (yl < cfg.target_height && px >= x0 && px - x0 < w && py >= y0 && py - y0 < h)
            *reinterpret_cast<int32_t *>(reinterpret_cast<char *>(out) + (size_t)(py - y0) * pitch + 4u * (size_t)(px - x0)) = best;
    }
}

extern "C" uint32_t vb_launch_hit_map(const VbConfig &cfg, const VbFrameBufs &b, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h,
                                      int32_t *draw_ix, size_t pitch, cudaStream_t st) {
    if (w == 0u || h == 0u) return 0;
    // the tile rows of the tall grid the rectangle's first and last pixel rows fall in (a cell's last tile row may be partial)
    const uint32_t y1 = y0 + (h - 1u), c0 = y0 / cfg.target_height, c1 = y1 / cfg.target_height;
    const uint32_t tr0 = c0 * cfg.height_in_tiles + (y0 - c0 * cfg.target_height) / VB_TILE_HEIGHT;
    const uint32_t tr1 = c1 * cfg.height_in_tiles + (y1 - c1 * cfg.target_height) / VB_TILE_HEIGHT;
    const uint32_t tx0 = x0 / VB_TILE_WIDTH, n_rows = tr1 - tr0 + 1u;
    const dim3 grid((x0 + (w - 1u)) / VB_TILE_WIDTH - tx0 + 1u, n_rows < 65535u ? n_rows : 65535u);
    k_hit_map<<<grid, HT_THREADS, 0, st>>>(cfg, b.scene, b.draw_monoids, b.bin_headers, b.info_bin_data, b.paths, b.tiles, b.segments,
                                           b.bump(), x0, y0, w, h, tx0, tr0, n_rows, draw_ix, pitch);
    return 1;
}
