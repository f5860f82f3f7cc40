// k_path_tiling.cu -- clip every (line, tile) crossing to its tile and store the tile-relative segment.
//
// Reference: vello_shaders/shader/path_tiling.wgsl:40-172 (+ path_tiling_setup.wgsl), CPU twin
// cpu/path_tiling.rs. One thread per crossing (SegmentCount record); no indirect dispatch: the grid
// is sized from the arena and strides over bump.seg_counts read on the device.
// Slices: k_backdrop gives every (path, tile) with crossings its slice, so this kernel does not wait for coarse; the
// two run side by side on two streams (vb_frame.cu). Crossings of tiles that coarse emits no CMD_FILL for are still
// written, into slots no command reads (the reference, which allocates in coarse, skips them).
// Algorithmic bytes per crossing: 12 (SegmentCount) + 24 (LineSoup gather) + 32 (Path) + 8 (Tile)
// read, 24 written (scattered into the tile's slice).
#include "vb_device.cuh"
#include "vb_stages.h"

#ifndef PTI_THREADS
#define PTI_THREADS 256
#endif
#ifndef PTI_MINB
#define PTI_MINB 8
#endif
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define TILE_SCALE 0.0625f

__global__ void __launch_bounds__(PTI_THREADS, PTI_MINB)
k_path_tiling(VbConfig cfg, VbBump *bump, const VbSegmentCount *__restrict__ seg_counts,
              const VbLineSoup *__restrict__ lines, const VbPath *__restrict__ paths, const VbTile *__restrict__ tiles,
              VbSegment *segments) {
    // backdrop assigned more segment slots than the arena holds: flagged here (one thread), decided by every CTA alike.
    // Only the stages before coarse abort this kernel: coarse, running beside it, may raise its bit at any time.
    const bool seg_overflow = bump->segments > cfg.segments_size;
    if (seg_overflow && blockIdx.x == 0u && threadIdx.x == 0u) atomicOr(&bump->failed, VB_STAGE_FINE_SEGMENTS);
    if ((bump->failed & VB_STAGES_BEFORE_COARSE) != 0u || seg_overflow) return;
    const uint32_t n_segments = min(bump->seg_counts, cfg.seg_counts_size);
    for (uint32_t g = blockIdx.x * PTI_THREADS + threadIdx.x; g < n_segments; g += gridDim.x * PTI_THREADS) {
        const VbSegmentCount sc = seg_counts[g];
        const uint2 *lp = reinterpret_cast<const uint2 *>(lines + sc.line_ix);
        const uint2 w0 = __ldg(lp), w1 = __ldg(lp + 1), w2 = __ldg(lp + 2);
        const uint32_t path_ix = w0.x;
        const float p0x = __uint_as_float(w1.x), p0y = __uint_as_float(w1.y);
        const float p1x = __uint_as_float(w2.x), p1y = __uint_as_float(w2.y);
        const uint32_t seg_within_slice = sc.seg_within_slice;
        const uint32_t seg_within_line = sc.seg_within_line;
        if (seg_within_slice == VB_SEG_OUTSIDE) continue; // path_count found its tile outside the path's tile box
        const bool is_down = p1y >= p0y;
        float xy0x = is_down ? p0x : p1x, xy0y = is_down ? p0y : p1y;
        float xy1x = is_down ? p1x : p0x, xy1y = is_down ? p1y : p0y;
        const float s0x = xy0x * TILE_SCALE, s0y = xy0y * TILE_SCALE, s1x = xy1x * TILE_SCALE, s1y = xy1y * TILE_SCALE;
        const uint32_t count_x = vb_span(s0x, s1x) - 1u;
        const uint32_t count = count_x + vb_span(s0y, s1y);
        const float dx = fabsf(s1x - s0x);
        const float dy = s1y - s0y;
        const float idxdy = 1.0f / (dx + dy);
        float a = dx * idxdy;
        const bool is_positive_slope = s1x >= s0x;
        const float x_sign = is_positive_slope ? 1.0f : -1.0f;
        const float xt0 = floorf(s0x * x_sign);
        const float c = s0x * x_sign - xt0;
        const float y0i = floorf(s0y);
        const float ytop = (s0y == s1y) ? ceilf(s0y) : y0i + 1.0f;
        const float b = fminf((dy * c + dx * (ytop - s0y)) * idxdy, ONE_MINUS_ULP);
        const float robust_err = floorf(a * ((float)count - 1.0f) + b) - (float)count_x;
        if (robust_err != 0.0f) a -= ROBUST_EPSILON * vb_signf(robust_err);
        const int32_t x0i = vb_f2i_sat(xt0 * x_sign + 0.5f * (x_sign - 1.0f));
        const float z = floorf(a * (float)seg_within_line + b);
        const int32_t x = x0i + vb_f2i_sat(x_sign * z);
        const int32_t y = vb_f2i_sat(y0i + (float)seg_within_line - z);
        const VbPath path = paths[path_ix];
        const int32_t bx0 = (int32_t)path.bbox[0], by0 = (int32_t)path.bbox[1], bx1 = (int32_t)path.bbox[2];
        const int32_t by1 = (int32_t)path.bbox[3];
        // path_count's x is one f32 sum, this one two int parts: past 2^24 tiles they may differ, so bound this one too
        if (x < bx0 || x >= bx1 || y < by0 || y >= by1) continue;
        const int32_t stride = bx1 - bx0;
        const int32_t tile_ix = (int32_t)path.tiles + (y - by0) * stride + x - bx0;
        const uint32_t seg_start = ~tiles[tile_ix].segment_count_or_ix; // every tile has its slice (k_backdrop)
        const float tile_x = (float)x * 16.0f, tile_y = (float)y * 16.0f;
        const float tile_x1 = tile_x + 16.0f, tile_y1 = tile_y + 16.0f;
        if (seg_within_line > 0u) {
            const float z_prev = floorf(a * ((float)seg_within_line - 1.0f) + b);
            if (z == z_prev) {
                float xt = xy0x + (xy1x - xy0x) * (tile_y - xy0y) / (xy1y - xy0y);
                xt = vb_clampf(xt, tile_x + 1e-3f, tile_x1);
                xy0x = xt; xy0y = tile_y;
            } else {
                const float x_clip = is_positive_slope ? tile_x : tile_x1;
                float yt = xy0y + (xy1y - xy0y) * (x_clip - xy0x) / (xy1x - xy0x);
                yt = vb_clampf(yt, tile_y + 1e-3f, tile_y1);
                xy0x = x_clip; xy0y = yt;
            }
        }
        if (seg_within_line < count - 1u) {
            const float z_next = floorf(a * ((float)seg_within_line + 1.0f) + b);
            if (z == z_next) {
                float xt = xy0x + (xy1x - xy0x) * (tile_y1 - xy0y) / (xy1y - xy0y);
                xt = vb_clampf(xt, tile_x + 1e-3f, tile_x1);
                xy1x = xt; xy1y = tile_y1;
            } else {
                const float x_clip = is_positive_slope ? tile_x1 : tile_x;
                float yt = xy0y + (xy1y - xy0y) * (x_clip - xy0x) / (xy1x - xy0x);
                yt = vb_clampf(yt, tile_y + 1e-3f, tile_y1);
                xy1x = x_clip; xy1y = yt;
            }
        }
        float y_edge = 1e9f;
        float q0x = xy0x - tile_x, q0y = xy0y - tile_y, q1x = xy1x - tile_x, q1y = xy1y - tile_y;
        const float EPSILON = 1e-6f;
        if (q0x == 0.0f) {
            if (q1x == 0.0f) {
                q0x = EPSILON;
                if (q0y == 0.0f) {
                    q1x = EPSILON;
                    q1y = 16.0f;
                } else {
                    q1x = 2.0f * EPSILON;
                    q1y = q0y;
                }
            } else if (q0y == 0.0f) {
                q0x = EPSILON;
            } else {
                y_edge = q0y;
            }
        } else if (q1x == 0.0f) {
            if (q1y == 0.0f) q1x = EPSILON;
            else y_edge = q1y;
        }
        if (q0x == floorf(q0x) && q0x != 0.0f) q0x -= EPSILON;
        if (q1x == floorf(q1x) && q1x != 0.0f) q1x -= EPSILON;
        if (!is_down) {
            float t;
            t = q0x; q0x = q1x; q1x = t;
            t = q0y; q0y = q1y; q1y = t;
        }
        const uint32_t out_ix = seg_start + seg_within_slice;
        if (out_ix < cfg.segments_size) {
            uint2 *dst = reinterpret_cast<uint2 *>(segments + out_ix);
            dst[0] = make_uint2(__float_as_uint(q0x), __float_as_uint(q0y));
            dst[1] = make_uint2(__float_as_uint(q1x), __float_as_uint(q1y));
            dst[2] = make_uint2(__float_as_uint(y_edge), 0u);
        }
    }
}

// The grid comes from the seg_counts capacity (at most 16 CTAs per SM); the kernel strides over the count read on the device.
extern "C" uint32_t vb_launch_path_tiling(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const uint64_t blocks = ((uint64_t)cfg.seg_counts_size + 255) / 256, most = (uint64_t)b.sm_count * 16;
    const uint32_t grid = (uint32_t)(blocks < most ? blocks : most);
    if (grid == 0) return 0;
    k_path_tiling<<<grid, PTI_THREADS, 0, st>>>(cfg, b.bump(), b.seg_counts, b.lines, b.paths, b.tiles, b.segments);
    return 1;
}
