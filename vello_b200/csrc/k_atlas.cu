// k_atlas.cu -- copy images that live in device memory into the image atlas (Renderer::override_image / register_texture,
// vello/src/lib.rs:536-603; the wgpu engine does it with one texture copy per image, Command::WriteImage, wgpu_engine.rs:480-500).
//
// One launch copies N rectangles. The work of rectangle i is h_i rows of `spr_i` units; a unit is one 16-byte-aligned window of
// four texels of the DESTINATION row, so every full window is stored with one 16-byte store whatever the source alignment.
// The rectangles' units are concatenated (unit0 = exclusive prefix, computed on the host) and every CTA takes the same number
// of consecutive units: a 4096x4096 texture and hundreds of 8x8 icons share the grid evenly. A source row is only guaranteed
// 4-byte aligned (the pitch is any multiple of 4, e.g. a column slice of a wider tensor), so a window is loaded with one
// 16-byte load only when it is full and its source texels start on a 16-byte boundary; otherwise texel by texel.
#include "vb_device.cuh"
#include "vb_types.h"
#include "vb_stages.h"

#define AB_THREADS 256u
#define AB_UNITS_PER_THREAD 4u
#define AB_UNITS_PER_CTA (AB_THREADS * AB_UNITS_PER_THREAD)

// the rectangle holding unit u: the last i in [lo, hi] with rects[i].unit0 <= u
__device__ __forceinline__ uint32_t ab_find(const VbBlitRect *__restrict__ rects, uint32_t lo, uint32_t hi, uint64_t u) {
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (rects[mid].unit0 <= u) lo = mid;
        else hi = mid - 1u;
    }
    return lo;
}

__global__ void __launch_bounds__(AB_THREADS)
k_atlas_blit(const VbBlitRect *__restrict__ rects, uint32_t n, uint64_t total_units, uint8_t *__restrict__ atlas, uint32_t atlas_w) {
    const uint64_t c0 = (uint64_t)blockIdx.x * AB_UNITS_PER_CTA;
    const uint64_t c1 = min(c0 + AB_UNITS_PER_CTA, total_units);
    // the CTA's units lie in rectangles first..last (one rectangle for all CTAs inside a large image)
    const uint32_t first = ab_find(rects, 0u, n - 1u, c0), last = ab_find(rects, first, n - 1u, c1 - 1u);
    uint4 v[AB_UNITS_PER_THREAD];
    uint4 *dst[AB_UNITS_PER_THREAD];
    uint32_t mask[AB_UNITS_PER_THREAD]; // texels of the window that belong to the rectangle (bit l: texel l of the window)
#pragma unroll
    for (uint32_t k = 0; k < AB_UNITS_PER_THREAD; k++) {
        mask[k] = 0u;
        dst[k] = nullptr;
        v[k] = make_uint4(0u, 0u, 0u, 0u);
        const uint64_t u = c0 + k * AB_THREADS + threadIdx.x;
        if (u >= c1) continue;
        const VbBlitRect &R = rects[ab_find(rects, first, last, u)];
        const uint32_t local = (uint32_t)(u - R.unit0);
        const uint32_t row = local / R.spr, slot = local - row * R.spr;
        const size_t dst_px = (size_t)(R.dst_y + row) * atlas_w + R.dst_x;
        const uint32_t mis = (uint32_t)(dst_px & 3u);            // texels between the row start and the 16-byte boundary before it
        const int32_t t0 = (int32_t)(slot * 4u) - (int32_t)mis;  // first texel of the window, relative to the row start
        if (t0 >= (int32_t)R.w) continue;                        // spr covers the worst misalignment; this row needs one unit less
        const uint8_t *src = R.src + (size_t)row * R.src_pitch;
        dst[k] = reinterpret_cast<uint4 *>(atlas + (dst_px - mis) * 4u) + slot;
        const bool full = t0 >= 0 && t0 + 4 <= (int32_t)R.w;
        if (full && ((reinterpret_cast<uintptr_t>(src) + (uint32_t)t0 * 4u) & 15u) == 0u) {
            v[k] = __ldg(reinterpret_cast<const uint4 *>(src + (uint32_t)t0 * 4u));
            mask[k] = 0xFu;
            continue;
        }
        uint32_t t[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int l = 0; l < 4; l++) {
            const int32_t x = t0 + l;
            if (x >= 0 && x < (int32_t)R.w) {
                t[l] = __ldg(reinterpret_cast<const uint32_t *>(src) + x);
                mask[k] |= 1u << l;
            }
        }
        v[k] = make_uint4(t[0], t[1], t[2], t[3]);
    }
#pragma unroll
    for (uint32_t k = 0; k < AB_UNITS_PER_THREAD; k++) {
        if (mask[k] == 0xFu) {
            *dst[k] = v[k];
        } else if (mask[k]) {
            uint32_t *d = reinterpret_cast<uint32_t *>(dst[k]);
            if (mask[k] & 1u) d[0] = v[k].x;
            if (mask[k] & 2u) d[1] = v[k].y;
            if (mask[k] & 4u) d[2] = v[k].z;
            if (mask[k] & 8u) d[3] = v[k].w;
        }
    }
}

// Units of a w x h rectangle: every row gets the windows of its worst-case placement, ceil((3 + w) / 4).
extern "C" uint32_t vb_atlas_blit_units_per_row(uint32_t w) { return (w + 6u) / 4u; }

extern "C" uint32_t vb_launch_atlas_blit(const VbBlitRect *rects, uint32_t n, uint64_t total_units, uint8_t *atlas, uint32_t atlas_w,
                                         cudaStream_t st) {
    if (n == 0u || total_units == 0u) return 0u;
    const uint64_t grid = (total_units + AB_UNITS_PER_CTA - 1u) / AB_UNITS_PER_CTA;
    k_atlas_blit<<<(uint32_t)grid, AB_THREADS, 0, st>>>(rects, n, total_units, atlas, atlas_w);
    return 1u;
}
