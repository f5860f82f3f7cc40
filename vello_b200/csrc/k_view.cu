// k_view.cu -- views of a resident scene (vb_set_view): every draw rendered as Scene::new().append(&scene, Some(view)) would
// render it (vello_encoding/src/encoding.rs:94-174), without touching the uploaded bytes.
//
// The view V lives in device memory, written in stream order by k_view_set, so that frames enqueued before a change keep
// the view they were enqueued with and a captured frame replays under a new view. k_view_transforms, the first kernel of a
// viewed frame, writes V * T for every transform T of the scene into a region past the scene's streams; the frame's
// layout.transform_base points there (prepare, vb_frame.cu). The scene's own transforms are never modified, so a re-run after
// an arena overflow, a graph replay or the next frame compose the view once.
#include "vb_device.cuh"
#include "vb_stages.h"

struct ViewCoeffs {
    float m[6];
};

__global__ void k_view_set(ViewCoeffs v, float *dst) {
    if (threadIdx.x < 6u) dst[threadIdx.x] = v.m[threadIdx.x];
}

// V * T with Encoding::append's arithmetic (vb_affine_mul), so the viewed transforms are the bits a host-side append produces.
__global__ void __launch_bounds__(256) k_view_transforms(const float *__restrict__ view, const uint32_t *__restrict__ src, uint32_t *dst,
                                                         uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float a[6], b[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
        a[k] = __ldg(view + k);
        b[k] = __uint_as_float(__ldg(src + 6u * i + k));
    }
    float r[6];
    vb_affine_mul(a, b, r);
#pragma unroll
    for (int k = 0; k < 6; k++) dst[6u * i + k] = __float_as_uint(r[k]);
}

extern "C" void vb_launch_view_set(float *dst, const float m[6], cudaStream_t st) {
    ViewCoeffs v;
    for (int k = 0; k < 6; k++) v.m[k] = m[k];
    k_view_set<<<1, 32, 0, st>>>(v, dst);
}

extern "C" uint32_t vb_launch_view_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    // exactly the region prepare reserved and sized the allocation for: n transforms at transform_base, past the uploaded
    // streams. It is empty for a layout whose transforms do not lie inside the uploaded words, so such a layout launches
    // nothing, and the source transforms [view_src, view_src + 6 n) lie inside the scene whenever n > 0.
    const uint32_t n = b.xf_len;
    if (n == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + cfg.layout.transform_base;
    k_view_transforms<<<(n + 255u) / 256u, 256, 0, st>>>(b.view, b.scene + cfg.view_src, dst, n);
    return 1u;
}
