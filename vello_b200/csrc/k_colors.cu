// k_colors.cu -- the bound draw data: every frame renders the scene's draw data with the words that bound colours
// (vb_bind_draw_colors), bound gradient stops (vb_bind_gradient_stops) and bound opacity (vb_bind_draw_opacity) make from
// device rows, read when the frame runs.
//
// No pipeline kernel changes for them. The frame's layout.draw_data_base points at a region past the scene's streams (prepare,
// vb_frame.cu), and k_draw_data writes the whole draw-data stream there at the start of the frame, each word once: the scene's
// word, or the word its binding makes from its row. draw, coarse and fine then read the bound words as they would read an
// uploaded scene's. Where the bound words lie is fixed while the rows are bound, since every scene installation unbinds:
// k_draw_data_slots finds them once, at bind time, with one scan of the draw tags (a composed or device-resolved scene's tags
// exist only on the device), into one table with a word per draw-data word: the draw object k it belongs to, or VB_COLOR_NONE.
// The word's role follows from k's tag:
//   - a colour (FILL_COLOR, BLURRED_ROUNDED_RECT; its first word, for k below the bound colours): the premultiplied RGBA8
//     word of row k, the encoder's premultiply().to_rgba8().
//   - a gradient's ramp word (its first) while stops are bound: bound gradient g = rs_draw[k] takes ramp row ramp0 + g, a
//     row of its own (k_resolve.cu), with its extend mode kept. A gradient that is not bound keeps its word.
//   - a layer's BEGIN_CLIP (blend, luminance-mask or clip layer; for k below the bound opacity rows): its alpha word (its
//     second) becomes the row, clamped to [0, 1] as both encoders' push_layer clamp it. An END_CLIP reads its BEGIN_CLIP's
//     draw data (clip_leaf gives it that draw monoid offset), so the pair agrees, and an END_CLIP's own row is never read.
//   - a clip layer's blend word (its first, when the scene's is CLIP_BLEND_MODE, 0x8003: the word whose successor holds the
//     same k): with a row below 1 it becomes Normal / SrcOver (3), and its alpha word the row, so the frame renders
//     push_layer(Mix::Normal, Compose::SrcOver, row) in its place. Coarse sets a layer's blend flag from this word: a 0x8003
//     layer emits no BEGIN_CLIP / END_CLIP in tiles wholly inside its clip, and an alpha alone would only fade its edge tiles.
//     With a row of 1 both words stay as encoded.
//   - an image's sample word (FILL_IMAGE; its third, for k below the bound opacity rows): its low byte becomes
//     int(row * 255 + 0.5), the encoders' conversion of the image alpha times the brush alpha, with the product and the sum
//     each rounded on their own (no FMA).
// Every other draw object's row is never read, and a row with a value that is not finite keeps the encoded words for that
// frame.
#include "vb_device.cuh"
#include "vb_stages.h"

#define DD_THREADS 256u
#define DD_SLOT_THREADS 1024u
#define DD_NORMAL_SRC_OVER 3u // (Mix::Normal << 8) | Compose::SrcOver
#define DD_CLIP_BLEND 0x8003u // (Mix::Clip << 8) | Compose::SrcOver: push_clip_layer's blend word

__device__ __forceinline__ bool dd_gradient(uint32_t tag) {
    return tag == VB_DRAWTAG_FILL_LIN_GRADIENT || tag == VB_DRAWTAG_FILL_RAD_GRADIENT || tag == VB_DRAWTAG_FILL_SWEEP_GRADIENT;
}

// The encoders' image alpha byte of a row already clamped to [0, 1]: int(f32(a) * 255 + 0.5), each step rounded on its own
// (encoding.py's encode_brush, vb_scene.cpp's encode_brush, with a brush alpha of 1).
__device__ __forceinline__ uint32_t dd_alpha_byte(float a) { return (uint32_t)__fadd_rn(__fmul_rn(a, 255.0f), 0.5f); }

// One CTA walks the first n draw tags a chunk at a time: the exclusive scan of their draw-data sizes (draw.rs's DrawTag, as
// k_draw's monoid has it) gives each draw object's first word, and the words of the draw objects the bindings reach (n_col
// colours, n_op layers and images, every gradient while n_grads > 0) get their draw object. Then each bound gradient g whose
// ramp word (grad_dd[g], relative to the draw data) is a gradient's first word gives that draw object k draw_grad[k] = g. The
// caller sets both tables to VB_COLOR_NONE first.
__global__ void __launch_bounds__(DD_SLOT_THREADS) k_draw_data_slots(const uint32_t *__restrict__ tags, const uint32_t *__restrict__ dd,
                                                                     uint32_t n_words, uint32_t n, uint32_t n_col, uint32_t n_op,
                                                                     const uint32_t *__restrict__ grad_dd, uint32_t n_grads,
                                                                     uint32_t *slots, uint32_t *draw_grad) {
    __shared__ uint32_t sh[DD_SLOT_THREADS / 32u + 1u];
    uint32_t base = 0u;
    for (uint32_t c = 0u; c < n; c += DD_SLOT_THREADS) {
        const uint32_t k = c + threadIdx.x;
        const uint32_t tag = k < n ? __ldg(tags + k) : VB_DRAWTAG_NOP;
        uint32_t total;
        const uint32_t off = base + vb_block_excl_scan((tag >> 2) & 7u, sh, &total);
        if ((tag == VB_DRAWTAG_FILL_COLOR || tag == VB_DRAWTAG_BLURRED_ROUNDED_RECT) && k < n_col && off < n_words) {
            slots[off] = k;
        } else if (dd_gradient(tag) && n_grads && off < n_words) {
            slots[off] = k;
        } else if (tag == VB_DRAWTAG_BEGIN_CLIP && k < n_op && off + 1u < n_words) {
            slots[off + 1u] = k;
            if (__ldg(dd + off) == DD_CLIP_BLEND) slots[off] = k;
        } else if (tag == VB_DRAWTAG_FILL_IMAGE && k < n_op && off + 2u < n_words) {
            slots[off + 2u] = k;
        }
        base += total;
    }
    __syncthreads();
    for (uint32_t g = threadIdx.x; g < n_grads; g += DD_SLOT_THREADS) {
        const uint32_t w = __ldg(grad_dd + g);
        const uint32_t k = w < n_words ? slots[w] : VB_COLOR_NONE;
        if (k != VB_COLOR_NONE && dd_gradient(__ldg(tags + k))) draw_grad[k] = g;
    }
}

// One thread per draw-data word u: the scene's word `src[u]`, or the word its slot's binding makes from its row (the rules
// above), into the frame's draw data `dst`.
__global__ void __launch_bounds__(DD_THREADS) k_draw_data(const uint32_t *__restrict__ slots, const uint32_t *__restrict__ tags,
                                                          const uint32_t *__restrict__ src, uint32_t *dst, uint32_t n_words,
                                                          const uint8_t *__restrict__ col_rows, uint32_t col_pitch,
                                                          const uint8_t *__restrict__ op_rows, uint32_t op_pitch,
                                                          const uint32_t *__restrict__ draw_grad, uint32_t ramp0) {
    const uint32_t u = blockIdx.x * DD_THREADS + threadIdx.x;
    if (u >= n_words) return;
    uint32_t w = __ldg(src + u);
    const uint32_t k = __ldg(slots + u);
    if (k != VB_COLOR_NONE) {
        const uint32_t tag = __ldg(tags + k);
        if (tag == VB_DRAWTAG_BEGIN_CLIP || tag == VB_DRAWTAG_FILL_IMAGE) {
            const float row = __ldg(reinterpret_cast<const float *>(op_rows + (size_t)k * op_pitch));
            if (isfinite(row)) {
                const float a = row < 0.0f ? 0.0f : (row > 1.0f ? 1.0f : row); // as the encoders clamp: -0.0 stays -0.0
                if (tag == VB_DRAWTAG_FILL_IMAGE)
                    w = (w & ~0xFFu) | dd_alpha_byte(a);
                else if (u + 1u < n_words && __ldg(slots + u + 1u) == k) // a clip layer's blend word
                    w = a < 1.0f ? DD_NORMAL_SRC_OVER : w;
                else if (a < 1.0f || __ldg(slots + u - 1u) != k) // an alpha word (so u > 0): a clip layer's only below 1
                    w = __float_as_uint(a);
            }
        } else if (dd_gradient(tag)) {
            const uint32_t g = __ldg(draw_grad + k);
            if (g != VB_COLOR_NONE) w = ((ramp0 + g) << 2) | (w & 3u);
        } else {
            const float *row = reinterpret_cast<const float *>(col_rows + (size_t)k * col_pitch);
            const float r = __ldg(row), g = __ldg(row + 1), b = __ldg(row + 2), a = __ldg(row + 3);
            if (isfinite(r) && isfinite(g) && isfinite(b) && isfinite(a)) w = dc_premul_rgba8(r, g, b, a);
        }
    }
    dst[u] = w;
}

extern "C" uint32_t vb_launch_draw_data_slots(const VbBound &b, const uint32_t *tags, const uint32_t *dd, uint32_t n_words, uint32_t n_draw,
                                              const uint32_t *grad_dd, uint32_t *slots, cudaStream_t st) {
    const uint32_t n_col = b.rows[VB_BIND_COLORS].n, n_op = b.rows[VB_BIND_OPACITY].n;
    const uint32_t n = max(max(n_col, n_op), b.rs_grads_n ? n_draw : 0u);
    if (n == 0u) return 0u;
    k_draw_data_slots<<<1, DD_SLOT_THREADS, 0, st>>>(tags, dd, n_words, n, n_col, n_op, grad_dd, b.rs_grads_n, slots,
                                                     const_cast<uint32_t *>(b.rs_draw));
    return 1u;
}

extern "C" uint32_t vb_launch_draw_data(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (!b.bound.dd_slots) return 0u;
    // the region prepare reserved past the scene's streams and the transform regions
    const uint32_t n = b.dd_len;
    if (n == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + cfg.layout.draw_data_base;
    const VbRows &col = b.bound.rows[VB_BIND_COLORS], &op = b.bound.rows[VB_BIND_OPACITY];
    k_draw_data<<<(n + DD_THREADS - 1u) / DD_THREADS, DD_THREADS, 0, st>>>(b.bound.dd_slots, b.scene + cfg.layout.draw_tag_base, b.dd_src, dst, n,
                                                                           col.rows, col.pitch, op.rows, op.pitch, b.bound.rs_draw,
                                                                           b.bound.rs_ramp0);
    return 1u;
}
