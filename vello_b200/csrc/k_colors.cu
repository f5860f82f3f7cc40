// k_colors.cu -- bound draw colours (vb_bind_draw_colors): every frame renders draw object k, for k below the bound count, as
// if it had been encoded with Color(row k) of a device array, read when the frame runs.
//
// No pipeline kernel changes for it. The frame's layout.draw_data_base points at a region past the scene's streams (prepare,
// vb_frame.cu), and k_draw_colors writes the whole draw-data stream there at the start of the frame: the scene's words, with
// each bound colour word replaced by its row's conversion. draw, coarse (the colour and its opacity test) and fine then read
// the bound words as they would read an uploaded scene's. Bound gradient stops use the same region for their ramp words
// (k_resolve.cu), so it is written when colours, stops or both are bound. Where the colour words lie is fixed while the rows are bound, since
// every scene installation unbinds: k_draw_color_slots finds them once, at bind time, with a scan of the draw tags (a composed
// or device-resolved scene's tags exist only on the device).
#include "vb_device.cuh"
#include "vb_stages.h"

#define DC_THREADS 256u
#define DC_SLOT_THREADS 1024u

// One CTA walks the first n draw tags a chunk at a time: the exclusive scan of their draw-data sizes (draw.rs's DrawTag, as
// k_draw's monoid has it) gives each draw object's first word, which is its colour for FILL_COLOR and BLURRED_ROUNDED_RECT.
__global__ void __launch_bounds__(DC_SLOT_THREADS) k_draw_color_slots(const uint32_t *__restrict__ tags, uint32_t n, uint32_t *slots,
                                                                      uint32_t n_words) {
    __shared__ uint32_t sh[DC_SLOT_THREADS / 32u + 1u];
    uint32_t base = 0u;
    for (uint32_t c = 0u; c < n; c += DC_SLOT_THREADS) {
        const uint32_t k = c + threadIdx.x;
        const uint32_t tag = k < n ? __ldg(tags + k) : VB_DRAWTAG_NOP;
        uint32_t total;
        const uint32_t off = base + vb_block_excl_scan((tag >> 2) & 7u, sh, &total);
        if ((tag == VB_DRAWTAG_FILL_COLOR || tag == VB_DRAWTAG_BLURRED_ROUNDED_RECT) && off < n_words) slots[off] = k;
        base += total;
    }
}

// One thread per draw-data word u: the scene's word, at a colour slot the converted row, at a bound gradient's ramp word the
// gradient's own ramp row (ramp0 + g) with its extend mode kept. A row with a value that is not finite keeps the scene's word,
// so the frame renders that draw object as encoded.
__global__ void __launch_bounds__(DC_THREADS) k_draw_colors(const uint8_t *__restrict__ rows, uint32_t pitch, const uint32_t *__restrict__ slots,
                                                            const uint32_t *__restrict__ src, uint32_t *dst, uint32_t n_words, uint32_t ramp0) {
    const uint32_t u = blockIdx.x * DC_THREADS + threadIdx.x;
    if (u >= n_words) return;
    uint32_t w = __ldg(src + u);
    const uint32_t k = __ldg(slots + u);
    if (k != VB_COLOR_NONE && (k & VB_GRAD_SLOT)) {
        w = ((ramp0 + (k & ~VB_GRAD_SLOT)) << 2) | (w & 3u);
    } else if (k != VB_COLOR_NONE) {
        const float *row = reinterpret_cast<const float *>(rows + (size_t)k * pitch);
        const float r = __ldg(row), g = __ldg(row + 1), b = __ldg(row + 2), a = __ldg(row + 3);
        if (isfinite(r) && isfinite(g) && isfinite(b) && isfinite(a)) w = dc_premul_rgba8(r, g, b, a);
    }
    dst[u] = w;
}

extern "C" uint32_t vb_launch_draw_color_slots(const uint32_t *tags, uint32_t n, uint32_t *slots, uint32_t n_words, cudaStream_t st) {
    if (n == 0u) return 0u;
    k_draw_color_slots<<<1, DC_SLOT_THREADS, 0, st>>>(tags, n, slots, n_words);
    return 1u;
}

extern "C" uint32_t vb_launch_draw_colors(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (!b.bound.col_slots) return 0u;
    // the region prepare reserved past the scene's streams and the transform regions
    const uint32_t n = b.dd_len;
    if (n == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + cfg.layout.draw_data_base;
    const VbRows &rows = b.bound.rows[VB_BIND_COLORS];
    k_draw_colors<<<(n + DC_THREADS - 1u) / DC_THREADS, DC_THREADS, 0, st>>>(rows.rows, rows.pitch, b.bound.col_slots, b.col_src, dst, n,
                                                                              b.bound.rs_ramp0);
    return 1u;
}
