// k_opacity.cu -- bound opacity (vb_bind_draw_opacity): every frame draws layer or image k, for k below the bound count, with
// the alpha in row k of a device array, read when the frame runs.
//
// No pipeline kernel changes for it. A layer's alpha and blend word and an image's sample word are draw-data words, and
// draw, coarse and fine read draw data only through layout.draw_data_base. While opacity is bound the frame reads the draw
// data from the region past the scene's streams that bound colours and stops use (k_colors.cu): k_draw_colors copies the
// scene's words there at the start of the frame, and k_draw_opacity then patches the bound words:
//   - a layer's BEGIN_CLIP (blend, luminance-mask or clip layer): its alpha word becomes the row, clamped to [0, 1] as both
//     encoders' push_layer clamp it. An END_CLIP reads its BEGIN_CLIP's draw data (clip_leaf gives it that draw monoid offset),
//     so the pair agrees, and an END_CLIP's own row is never read.
//   - a clip layer (blend word CLIP_BLEND_MODE, 0x8003) with a row below 1: its blend word also becomes Normal / SrcOver (3),
//     so the frame renders push_layer(Mix::Normal, Compose::SrcOver, row) in its place. Coarse sets a layer's blend flag from
//     this word: a 0x8003 layer emits no BEGIN_CLIP / END_CLIP in tiles wholly inside its clip, and an alpha alone would only
//     fade its edge tiles. With a row of 1 it stays as encoded.
//   - an image (FILL_IMAGE): the low byte of its sample word becomes int(row * 255 + 0.5), the encoders' conversion of the
//     image alpha times the brush alpha, with the product and the sum each rounded on their own (no FMA).
// Every other draw object ignores its row, and a row that is not finite keeps the encoded words for that frame. Where the
// bound words lie is fixed while the rows are bound, since every scene installation unbinds: k_draw_opacity_slots finds them
// once, at bind time, with a scan of the draw tags (a composed or device-resolved scene's tags exist only on the device).
#include "vb_device.cuh"
#include "vb_stages.h"

#define OP_THREADS 256u
#define OP_SLOT_THREADS 1024u
#define OP_NORMAL_SRC_OVER 3u   // (Mix::Normal << 8) | Compose::SrcOver
#define OP_CLIP_BLEND 0x8003u   // (Mix::Clip << 8) | Compose::SrcOver: push_clip_layer's blend word

// The encoders' image alpha byte of a row already clamped to [0, 1]: int(f32(a) * 255 + 0.5), each step rounded on its own
// (encoding.py's encode_brush, vb_scene.cpp's encode_brush, with a brush alpha of 1).
__device__ __forceinline__ uint32_t op_alpha_byte(float a) { return (uint32_t)__fadd_rn(__fmul_rn(a, 255.0f), 0.5f); }

// One CTA walks the first n draw tags a chunk at a time: the exclusive scan of their draw-data sizes gives each draw object's
// first word. Entry k of `table` is VB_OP_ENTRY(w, kind) for the word w it patches (relative to the draw data): a BEGIN_CLIP's
// alpha word (its second), kind VB_OP_CLIP when its blend word (its first, in the scene's draw data `dd`) is the clip
// layer's, else VB_OP_LAYER; an image's sample word (its third), VB_OP_IMAGE; VB_COLOR_NONE for every other draw object.
__global__ void __launch_bounds__(OP_SLOT_THREADS) k_draw_opacity_slots(const uint32_t *__restrict__ tags, const uint32_t *__restrict__ dd,
                                                                        uint32_t n, uint32_t n_words, uint32_t *table) {
    __shared__ uint32_t sh[OP_SLOT_THREADS / 32u + 1u];
    uint32_t base = 0u;
    for (uint32_t c = 0u; c < n; c += OP_SLOT_THREADS) {
        const uint32_t k = c + threadIdx.x;
        const uint32_t tag = k < n ? __ldg(tags + k) : VB_DRAWTAG_NOP;
        uint32_t total;
        const uint32_t off = base + vb_block_excl_scan((tag >> 2) & 7u, sh, &total);
        uint32_t e = VB_COLOR_NONE;
        if (tag == VB_DRAWTAG_BEGIN_CLIP && off + 1u < n_words)
            e = VB_OP_ENTRY(off + 1u, __ldg(dd + off) == OP_CLIP_BLEND ? VB_OP_CLIP : VB_OP_LAYER);
        else if (tag == VB_DRAWTAG_FILL_IMAGE && off + 2u < n_words)
            e = VB_OP_ENTRY(off + 2u, VB_OP_IMAGE);
        if (k < n) table[k] = e;
        base += total;
    }
}

// One thread per bound draw object k: its row, when finite and the draw object has a bound word, clamped and written over
// the word k_draw_colors copied into the frame's draw data `dst`.
__global__ void __launch_bounds__(OP_THREADS) k_draw_opacity(const uint8_t *__restrict__ rows, uint32_t pitch, const uint32_t *__restrict__ table,
                                                             uint32_t n, uint32_t *dst) {
    const uint32_t k = blockIdx.x * OP_THREADS + threadIdx.x;
    if (k >= n) return;
    const uint32_t e = __ldg(table + k);
    if (e == VB_COLOR_NONE) return;
    const float row = __ldg(reinterpret_cast<const float *>(rows + (size_t)k * pitch));
    if (!isfinite(row)) return;
    const float a = row < 0.0f ? 0.0f : (row > 1.0f ? 1.0f : row); // as the encoders clamp: -0.0 stays -0.0
    const uint32_t w = e >> 2, kind = e & 3u;
    if (kind == VB_OP_IMAGE) {
        dst[w] = (dst[w] & ~0xFFu) | op_alpha_byte(a);
    } else if (kind == VB_OP_LAYER || a < 1.0f) {
        dst[w] = __float_as_uint(a);
        if (kind == VB_OP_CLIP) dst[w - 1u] = OP_NORMAL_SRC_OVER;
    }
}

extern "C" uint32_t vb_launch_draw_opacity_slots(const uint32_t *tags, const uint32_t *dd, uint32_t n, uint32_t n_words, uint32_t *table,
                                                 cudaStream_t st) {
    if (n == 0u) return 0u;
    k_draw_opacity_slots<<<1, OP_SLOT_THREADS, 0, st>>>(tags, dd, n, n_words, table);
    return 1u;
}

extern "C" uint32_t vb_launch_draw_opacity(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbRows &rows = b.bound.rows[VB_BIND_OPACITY];
    if (!b.bound.op_slots || rows.n == 0u || b.dd_len == 0u) return 0u;
    // the region prepare reserved past the scene's streams, which k_draw_colors has just written
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + cfg.layout.draw_data_base;
    k_draw_opacity<<<(rows.n + OP_THREADS - 1u) / OP_THREADS, OP_THREADS, 0, st>>>(rows.rows, rows.pitch, b.bound.op_slots, rows.n, dst);
    return 1u;
}
