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
                                if (g.y_edge <= sy) w += (g.p1[0] > g.p0[0]) - (g.p1[0] < g.p0[0]);
                                if ((g.p0[1] <= sy) != (g.p1[1] <= sy)) {
                                    // it crosses the row left of the point: (crossing x - sx) * dy < 0, without a division
                                    const float dy = g.p1[1] - g.p0[1];
                                    const float c = (g.p0[0] - sx) * dy + (sy - g.p0[1]) * (g.p1[0] - g.p0[0]);
                                    if (dy > 0.0f ? c < 0.0f : c > 0.0f) w += dy > 0.0f ? -1 : 1;
                                }
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
