// k_visibility.cu -- bound visibility (vb_bind_draw_visibility): every frame shows draw object k, for k below the bound count,
// only when byte k of a device array is nonzero, read when the frame runs.
//
// Hiding is culling in flatten: plan_tag skips every tag of a hidden path (path p is draw object p), so the path's box stays
// empty, binning gives it no bins, tile_alloc no tiles, and coarse, fine, hit tests and hit maps never see it. A hidden
// BEGIN_CLIP's clip box is empty, so everything up to its END_CLIP, and the layer's blend, draws nothing: the frame is what
// the scene re-encoded without the hidden draw objects renders.
//
// The caller's bytes are read once per frame, here, at the start of flatten's stage, and packed into a renderer-owned bit mask
// (VbConfig::vis). Flatten and damage tracking read only the mask. k_flatten_lean counts a partition's lines and
// k_flatten_emit plans the same tags again to write them at the counted offsets, so both must see the same flags even when the
// caller writes its rows while the frame runs.
#include "vb_device.cuh"
#include "vb_stages.h"

#define VIS_THREADS 256u

// One thread per bit of the mask: bit k is row k's byte normalised to 0 / 1 below n, and 1 from n on.
__global__ void __launch_bounds__(VIS_THREADS) k_draw_visibility(const uint8_t *__restrict__ rows, uint32_t pitch, uint32_t n, uint32_t *mask,
                                                                 uint32_t n_words) {
    const uint32_t k = blockIdx.x * VIS_THREADS + threadIdx.x;
    if ((k >> 5) >= n_words) return; // whole warps: n_words * 32 bits
    const bool shown = k >= n || __ldg(rows + (size_t)k * pitch) != 0u;
    const uint32_t word = __ballot_sync(0xffffffffu, shown);
    if ((k & 31u) == 0u) mask[k >> 5] = word;
}

extern "C" uint32_t vb_launch_draw_visibility(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (!cfg.vis) return 0u;
    const uint32_t n_words = vb_vis_words(cfg.layout);
    if (n_words == 0u) return 0u;
    const uint32_t n_bits = n_words * 32u;
    const VbRows &rows = b.bound.rows[VB_BIND_VISIBILITY];
    k_draw_visibility<<<(n_bits + VIS_THREADS - 1u) / VIS_THREADS, VIS_THREADS, 0, st>>>(rows.rows, rows.pitch, rows.n,
                                                                                        const_cast<uint32_t *>(cfg.vis), n_words);
    return 1u;
}
