// k_path_count.cu -- line -> tile DDA: backdrop deltas, per-tile segment counts, crossing worklist.
//
// Reference: vello_shaders/shader/path_count.wgsl:51-202 (+ path_count_setup.wgsl), CPU twin
// cpu/path_count.rs; the conservative line walk is Appendix C.1 of SURVEY.md. Comparisons follow
// the WGSL where the CPU twin differs (`s1.y <= bbox.y`, `max(s0.x,s1.x) <= bbox.x`); WGSL
// round() is ties-to-even -> rintf.
//
// Design: one thread per line as in the WGSL, but (i) no indirect dispatch -- the grid is
// sized from the arena capacity and reads bump.lines on the device, (ii) the seg_counts
// allocation is aggregated per CTA: one atomicAdd per 256 lines instead of one per line (same-address atomics serialise;
// per-warp aggregation still left ~133 k of them a frame and was slower),
// (iii) backdrop / count updates are fire-and-forget RED operations except the slot fetch.
// Per-tile slot order (seg_within_slice) is atomic-order dependent exactly as in the reference.
#include "vb_device.cuh"
#include "vb_stages.h"

#ifndef PC_THREADS
#define PC_THREADS 256
#endif
#ifndef PC_MINB
#define PC_MINB 8
#endif
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define TILE_SCALE 0.0625f

__global__ void __launch_bounds__(PC_THREADS, PC_MINB)
k_path_count(VbConfig cfg, VbBump *bump, const VbLineSoup *__restrict__ lines, const VbPath *__restrict__ paths, VbTile *tile,
             VbSegmentCount *seg_counts) {
    __shared__ uint32_t sh_scan[PC_THREADS / 32 + 2];
    __shared__ uint32_t sh_base;
    if (bump->failed != 0u) return;
    const uint32_t n_lines = min(bump->lines, cfg.lines_size);
    for (uint32_t line_base = blockIdx.x * PC_THREADS; line_base < n_lines; line_base += gridDim.x * PC_THREADS) {
        const uint32_t line_ix = line_base + threadIdx.x;
        bool active = line_ix < n_lines;
        uint32_t imin = 0u, imax = 0u;
        float a = 0.f, b = 0.f, x0 = 0.f, y0 = 0.f, x_sign = 1.f, s0y = 0.f;
        int32_t bx0 = 0, by0 = 0, bx1 = 0, stride = 0, delta = 0;
        uint32_t path_tiles = 0;
        if (active) {
            const uint2 *lp = reinterpret_cast<const uint2 *>(lines + line_ix);
            uint2 w0 = __ldg(lp), w1 = __ldg(lp + 1), w2 = __ldg(lp + 2);
            const uint32_t path_ix = w0.x;
            const float p0x = __uint_as_float(w1.x), p0y = __uint_as_float(w1.y);
            const float p1x = __uint_as_float(w2.x), p1y = __uint_as_float(w2.y);
            const bool is_down = p1y >= p0y;
            const float xy0x = is_down ? p0x : p1x, xy0y = is_down ? p0y : p1y;
            const float xy1x = is_down ? p1x : p0x, xy1y = is_down ? p1y : p0y;
            const float s0x = xy0x * TILE_SCALE, s1x = xy1x * TILE_SCALE, s1y = xy1y * TILE_SCALE;
            s0y = xy0y * TILE_SCALE;
            const uint32_t count_x = vb_span(s0x, s1x) - 1u;
            const uint32_t count = count_x + vb_span(s0y, s1y);
            const float dx = fabsf(s1x - s0x);
            const float dy = s1y - s0y;
            if (dx + dy == 0.0f) active = false;
            if (dy == 0.0f && floorf(s0y) == s0y) active = false;
            if (active && path_ix >= cfg.layout.n_draw_objects) active = false;
            if (active) {
                const float idxdy = 1.0f / (dx + dy);
                a = dx * idxdy;
                const bool is_positive_slope = s1x >= s0x;
                x_sign = is_positive_slope ? 1.0f : -1.0f;
                const float xt0 = floorf(s0x * x_sign);
                const float c = s0x * x_sign - xt0;
                y0 = floorf(s0y);
                const float ytop = (s0y == s1y) ? ceilf(s0y) : y0 + 1.0f;
                b = fminf((dy * c + dx * (ytop - s0y)) * idxdy, ONE_MINUS_ULP);
                const float robust_err = floorf(a * ((float)count - 1.0f) + b) - (float)count_x;
                if (robust_err != 0.0f) a -= ROBUST_EPSILON * vb_signf(robust_err);
                x0 = xt0 * x_sign + (is_positive_slope ? 0.0f : -1.0f);
                const VbPath path = paths[path_ix];
                bx0 = (int32_t)path.bbox[0]; by0 = (int32_t)path.bbox[1]; bx1 = (int32_t)path.bbox[2];
                const int32_t by1 = (int32_t)path.bbox[3];
                path_tiles = path.tiles;
                const float xmin = fminf(s0x, s1x);
                stride = bx1 - bx0;
                if (s0y >= (float)by1 || s1y <= (float)by0 || xmin >= (float)bx1 || stride == 0) {
                    active = false;
                } else {
                    if (s0y < (float)by0) {
                        float iminf = rintf(((float)by0 - y0 + b - a) / (1.0f - a)) - 1.0f;
                        if (y0 + iminf - floorf(a * iminf + b) < (float)by0) iminf += 1.0f;
                        imin = vb_f2u_sat(iminf);
                    }
                    imax = count;
                    if (s1y > (float)by1) {
                        float imaxf = rintf(((float)by1 - y0 + b - a) / (1.0f - a)) - 1.0f;
                        if (y0 + imaxf - floorf(a * imaxf + b) < (float)by1) imaxf += 1.0f;
                        imax = vb_f2u_sat(imaxf);
                    }
                    delta = is_down ? -1 : 1;
                    int32_t ymin = 0, ymax = 0;
                    if (fmaxf(s0x, s1x) <= (float)bx0) {
                        ymin = vb_f2i_sat(ceilf(s0y));
                        ymax = vb_f2i_sat(ceilf(s1y));
                        imax = imin;
                    } else {
                        const float fudge = is_positive_slope ? 0.0f : 1.0f;
                        if (xmin < (float)bx0) {
                            float f = rintf((x_sign * ((float)bx0 - x0) - b + fudge) / a);
                            if ((x0 + x_sign * floorf(a * f + b) < (float)bx0) == is_positive_slope) f += 1.0f;
                            const int32_t ynext = vb_f2i_sat(y0 + f - floorf(a * f + b) + 1.0f);
                            if (is_positive_slope) {
                                if (vb_f2u_sat(f) > imin) {
                                    ymin = vb_f2i_sat(y0 + ((y0 == s0y) ? 0.0f : 1.0f));
                                    ymax = ynext;
                                    imin = vb_f2u_sat(f);
                                }
                            } else {
                                if (vb_f2u_sat(f) < imax) {
                                    ymin = ynext;
                                    ymax = vb_f2i_sat(ceilf(s1y));
                                    imax = vb_f2u_sat(f);
                                }
                            }
                        }
                        if (fmaxf(s0x, s1x) > (float)bx1) {
                            float f = rintf((x_sign * ((float)bx1 - x0) - b + fudge) / a);
                            if ((x0 + x_sign * floorf(a * f + b) < (float)bx1) == is_positive_slope) f += 1.0f;
                            if (is_positive_slope) imax = min(imax, vb_f2u_sat(f));
                            else imin = max(imin, vb_f2u_sat(f));
                        }
                    }
                    imax = max(imin, imax);
                    ymin = max(ymin, by0);
                    ymax = min(ymax, by1);
                    for (int32_t y = ymin; y < ymax; y++) {
                        const int32_t base = (int32_t)path_tiles + (y - by0) * stride;
                        atomicAdd(&tile[base].backdrop, delta);
                    }
                }
            }
        }
        const uint32_t n = active ? imax - imin : 0u;
        // CTA-aggregated worklist allocation: one same-address atomic per 256 lines
        uint32_t cta_total;
        const uint32_t excl = vb_block_excl_scan(n, sh_scan, &cta_total);
        if (threadIdx.x == 0 && cta_total != 0u) sh_base = atomicAdd(&bump->seg_counts, cta_total);
        __syncthreads();
        const uint32_t cta_base = sh_base;
        if (n != 0u) {
            const uint32_t seg_base = cta_base + excl;
            float last_z = floorf(a * ((float)imin - 1.0f) + b);
            for (uint32_t i = imin; i < imax; i++) {
                const float zf = a * (float)i + b;
                const float z = floorf(zf);
                const int32_t y = vb_f2i_sat(y0 + (float)i - z);
                const int32_t x = vb_f2i_sat(x0 + x_sign * z);
                const int32_t base = (int32_t)path_tiles + (y - by0) * stride - bx0;
                const bool top_edge = (i == 0u) ? (y0 == s0y) : (last_z == z);
                if (top_edge && x + 1 < bx1) {
                    const int32_t x_bump = max(x + 1, bx0);
                    atomicAdd(&tile[base + x_bump].backdrop, delta);
                }
                const uint32_t seg_within_slice = atomicAdd(&tile[base + x].segment_count_or_ix, 1u);
                const uint32_t seg_ix = seg_base + i - imin;
                if (seg_ix < cfg.seg_counts_size) {
                    VbSegmentCount sc = {line_ix, (seg_within_slice << 16) | i};
                    seg_counts[seg_ix] = sc;
                }
                last_z = z;
            }
        }
    }
}

// The seg_counts overflow check (the WGSL does it at the top of coarse) lives at the top of k_backdrop, the next kernel.

// The grid comes from the lines capacity (at most 16 CTAs per SM); the kernel strides over the count read on the device.
extern "C" uint32_t vb_launch_path_count(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const uint64_t blocks = ((uint64_t)cfg.lines_size + 255) / 256, most = (uint64_t)b.sm_count * 16;
    const uint32_t grid = (uint32_t)(blocks < most ? blocks : most);
    if (grid == 0) return 0;
    k_path_count<<<grid, PC_THREADS, 0, st>>>(cfg, b.bump(), b.lines, b.paths, b.tiles, b.seg_counts);
    return 1;
}
