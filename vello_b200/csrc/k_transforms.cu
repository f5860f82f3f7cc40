// k_transforms.cu -- bound transforms (vb_bind_transforms): every frame reads transform-stream entry k of the scene, for k below
// the bound count, from row k of a device array, read when the frame runs.
//
// No pipeline kernel changes for it. Transforms are read through the frame's layout.transform_base, by flatten (a segment's
// transform) and draw (a path's brush transform). prepare (vb_frame.cu) points that at the bound region past the scene's
// streams, the one bound instance transforms write, and k_bound_transforms writes it at the start of flatten's stage: each
// entry's row bits, or its source when the row is unbound or not finite. The source is the scene's own transforms, or with
// bound instance transforms the region itself, after k_instance_transforms wrote it. A view then applies on top
// (k_view_transforms reads the bound region). The tags never change while rows are bound (every scene installation unbinds),
// so each path's transform range, which damage tracking reads, is found once at bind time by k_path_point_slots (k_points.cu).
#include "vb_device.cuh"
#include "vb_stages.h"

#define BT_THREADS 256u

// One thread per transform entry u: below n the row's six words when none has an all-ones exponent (an infinity or a NaN),
// else the source's words; with no source (in place) the entry keeps what the region holds. Bits are copied, never
// converted or multiplied: a bound frame reads exactly the words a host-patched upload holds.
__global__ void __launch_bounds__(BT_THREADS) k_bound_transforms(const uint8_t *__restrict__ rows, uint32_t pitch, uint32_t n, const uint32_t *src,
                                                                 uint32_t *dst, uint32_t n_transforms) {
    const uint32_t u = blockIdx.x * BT_THREADS + threadIdx.x;
    if (u >= n_transforms) return;
    if (u < n) {
        const uint32_t *row = reinterpret_cast<const uint32_t *>(rows + (size_t)u * pitch);
        uint32_t w[6];
        bool finite = true;
#pragma unroll
        for (int i = 0; i < 6; i++) {
            w[i] = __ldg(row + i);
            finite = finite && (w[i] & 0x7f800000u) != 0x7f800000u;
        }
        if (finite) {
#pragma unroll
            for (int i = 0; i < 6; i++) dst[6u * u + i] = w[i];
            return;
        }
    }
    if (!src) return;
#pragma unroll
    for (int i = 0; i < 6; i++) dst[6u * u + i] = __ldg(src + 6u * u + i);
}

extern "C" uint32_t vb_launch_bound_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbRows &rows = b.bound.rows[VB_BIND_TRANSFORMS];
    if (!rows.rows) return 0u;
    // the bound region prepare reserved (vb_launch_instance_transforms): at transform_base, or with a view at the view's source
    const uint32_t n = b.xf_len;
    if (n == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + (b.view ? cfg.view_src : cfg.layout.transform_base);
    const uint32_t *src = b.bound.rows[VB_BIND_INSTANCES].rows ? nullptr : b.xf_src;
    k_bound_transforms<<<(n + BT_THREADS - 1u) / BT_THREADS, BT_THREADS, 0, st>>>(rows.rows, rows.pitch, rows.n, src, dst, n);
    return 1u;
}
