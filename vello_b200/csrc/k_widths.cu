// k_widths.cu -- bound stroke widths (vb_bind_stroke_widths): every frame strokes draw object k, for k below the bound count,
// with the width in row k of a device array, read when the frame runs.
//
// A row plays the part of the stroke's encoded width word (its style's second word): flatten's plan_tag offsets the stroke's
// centreline by half of it and grows its cull hull by it, and nothing else in the pipeline reads a width. Joins, caps, miter
// limit and dashes keep their encoded values. Hit tests and hit maps answer from the frame's lines, so they follow.
//
// The caller's rows are read once per frame, here, at the start of flatten's stage, into a renderer-owned snapshot
// (VbConfig::widths). Flatten and damage tracking read only the snapshot: k_flatten_lean counts a partition's lines and
// k_flatten_emit plans the same tags again to write them at the counted offsets, so both must see the same width even when the
// caller writes its rows while the frame runs.
#include "vb_device.cuh"
#include "vb_stages.h"

#define WD_THREADS 256u

// One thread per snapshot entry k: row k when draw object k is a stroke, k < n and the row is finite and > 0; else 0, which
// keeps the encoded width. A stroke is a draw object that is no layer's BEGIN_CLIP or END_CLIP (an END_CLIP's empty path
// inherits the style before it, and a layer's clip may be stroked), and whose path's style (the one in effect at its end tag,
// pathtag's path_draw) has the stroke bit.
__global__ void __launch_bounds__(WD_THREADS) k_stroke_widths(const uint8_t *__restrict__ rows, uint32_t pitch, uint32_t n,
                                                              const uint32_t *__restrict__ draw_tags, const uint2 *__restrict__ path_draw,
                                                              uint32_t n_paths, const uint32_t *__restrict__ styles, uint32_t n_style,
                                                              float *widths, uint32_t n_entries) {
    const uint32_t k = blockIdx.x * WD_THREADS + threadIdx.x;
    if (k >= n_entries) return;
    float w = 0.f;
    if (k < n && k < n_paths) {
        const uint32_t tag = __ldg(draw_tags + k), s = __ldg(&path_draw[k].x);
        const bool stroke = tag != VB_DRAWTAG_BEGIN_CLIP && tag != VB_DRAWTAG_END_CLIP && s < n_style &&
                            (__ldg(styles + s) & STYLE_FLAGS_STYLE) != 0u;
        const float row = __ldg(reinterpret_cast<const float *>(rows + (size_t)k * pitch));
        if (stroke && row > 0.f && row <= 3.402823466e38f) w = row; // NaN and +inf fail
    }
    widths[k] = w;
}

extern "C" uint32_t vb_launch_stroke_widths(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (!cfg.widths) return 0u;
    const uint32_t n_entries = vb_width_entries(cfg.layout);
    if (n_entries == 0u) return 0u;
    const VbRows &rows = b.bound.rows[VB_BIND_WIDTHS];
    const VbLayout &L = cfg.layout;
    const uint32_t n_style = cfg.scene_words > L.style_base ? cfg.scene_words - L.style_base : 0u;
    // the bind checked that the draw tags of the n rows lie inside the scene's words
    k_stroke_widths<<<(n_entries + WD_THREADS - 1u) / WD_THREADS, WD_THREADS, 0, st>>>(
        rows.rows, rows.pitch, rows.n, b.scene + L.draw_tag_base, b.path_draw, L.n_paths, b.scene + L.style_base, n_style,
        const_cast<float *>(cfg.widths), n_entries);
    return 1u;
}
