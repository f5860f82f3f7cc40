// k_resolve.cu -- the device half of Resolver::resolve (vello_encoding/src/resolve.rs:183-399, ramp_cache.rs:119-155).
//
// vb_scene_upload_streams (vb_upload.cu) copies the six encoding streams straight to their Layout offsets inside the packed scene
// buffer on the device; what is left of `resolve` runs here: the zero padding of the tag stream and the trailing PATH tags /
// END_CLIP draw tags of unclosed clips (resolve.rs:127-141), the late-bound patches (gradient ramp id | extend, atlas x | y:
// resolve.rs:268-330) and the gradient ramps themselves (512 premultiplied RGBA8 texels per unique gradient). The ramps of
// bound gradient stops (vb_bind_gradient_stops) are made here too, every frame, by the same walk.
// Arithmetic of the ramps is the host statement's (vb_scene.cpp make_ramp), float for float; the TU is built with -fmad=false.
#include "vb_device.cuh"
#include "vb_stages.h"

#define RS_TAG_PATH 0x10u
#define RS_DRAWTAG_END_CLIP 0x21u
#define RS_SAMPLES 512u

__global__ void k_resolve_finish(uint32_t *scene, uint32_t n_tag_bytes, uint32_t n_open_clips, uint32_t padded_tag_bytes, uint32_t end_clip_word0,
                                 const RsPatch *patches, uint32_t n_patches) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    uint8_t *tags = reinterpret_cast<uint8_t *>(scene);
    for (uint32_t b = n_tag_bytes + i; b < padded_tag_bytes; b += stride) tags[b] = b < n_tag_bytes + n_open_clips ? (uint8_t)RS_TAG_PATH : (uint8_t)0;
    for (uint32_t k = i; k < n_open_clips; k += stride) scene[end_clip_word0 + k] = RS_DRAWTAG_END_CLIP;
    for (uint32_t k = i; k < n_patches; k += stride) scene[patches[k].word] = patches[k].value;
}

__device__ __forceinline__ uint32_t rs_premul_rgba8(float r, float g, float b, float a) { // draw.rs:76-84
    const float comps[4] = {r * a, g * a, b * a, a};
    uint32_t out = 0u;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float v = floorf(comps[i] * 255.0f + 0.5f);
        if (!(v > 0.0f)) v = 0.0f; // also NaN
        if (v > 255.0f) v = 255.0f;
        out |= (uint32_t)v << (8 * i);
    }
    return out;
}

// Texel i of a ramp of n_stops stops, stop j read as stop(j): make_ramp's walk and conversion (vb_scene.cpp), which every
// ramp on the device runs. Each product and sum is rounded on its own (the TU is built with -fmad=false), as on the host. The
// host loop advances its stop cursor monotonically with u; starting from the initial state for every texel reaches the same
// cursor (every advance made for a smaller u is also made for this one).
template <class StopAt>
__device__ __forceinline__ uint32_t rs_ramp_texel(uint32_t i, uint32_t n_stops, uint32_t premul, StopAt stop) {
    const float u = (float)i / (float)(RS_SAMPLES - 1u);
    float last_u = 0.0f, this_u = 0.0f;
    const RsStop s0 = stop(0u);
    float lr = s0.r, lg = s0.g, lb = s0.b, la = s0.a;
    float tr = lr, tg = lg, tb = lb, ta = la;
    uint32_t j = 0u;
    while (u > this_u) {
        last_u = this_u;
        lr = tr; lg = tg; lb = tb; la = ta;
        if (j + 1u < n_stops) {
            const RsStop sj = stop(j + 1u);
            this_u = sj.offset;
            tr = sj.r; tg = sj.g; tb = sj.b; ta = sj.a;
            j += 1u;
        } else {
            break;
        }
    }
    const float du = this_u - last_u;
    float cr, cg, cb, ca;
    if (du < 1e-9f) {
        cr = tr; cg = tg; cb = tb; ca = ta;
    } else {
        const float t = (u - last_u) / du;
        if (premul != 0u) { // AlphaColor::lerp: premultiply, lerp_rect, un-premultiply (color crate)
            const float pa[4] = {lr * la, lg * la, lb * la, la};
            const float pb[4] = {tr * ta, tg * ta, tb * ta, ta};
            float pc[4];
#pragma unroll
            for (int k = 0; k < 4; k++) pc[k] = pa[k] + (pb[k] - pa[k]) * t;
            if (pc[3] == 0.0f || pc[3] == 1.0f) {
                cr = pc[0]; cg = pc[1]; cb = pc[2]; ca = pc[3];
            } else {
                const float inv = 1.0f / pc[3];
                cr = pc[0] * inv; cg = pc[1] * inv; cb = pc[2] * inv; ca = pc[3];
            }
        } else {
            cr = lr + (tr - lr) * t; cg = lg + (tg - lg) * t; cb = lb + (tb - lb) * t; ca = la + (ta - la) * t;
        }
    }
    return rs_premul_rgba8(cr, cg, cb, ca);
}

// one CTA per ramp, one thread per texel
__global__ void __launch_bounds__(RS_SAMPLES)
k_make_ramps(const RsRamp *ramps, const RsStop *stops, uint32_t *out) {
    const RsRamp rp = ramps[blockIdx.x];
    const RsStop *st = stops + rp.first_stop;
    const uint32_t i = threadIdx.x;
    out[(size_t)blockIdx.x * RS_SAMPLES + i] = rs_ramp_texel(i, rp.n_stops, rp.premul, [&](uint32_t j) { return st[j]; });
}

// ---- bound gradient stops (vb_bind_gradient_stops) ------------------------------------------------------------------------------
// A bound gradient renders from a ramp row of its own: resolves share one row between gradients whose stops are equal, and
// bound rows may part them. The binding gives bound gradient g row ramp0 + g of a renderer-owned copy of the scene's ramps,
// and k_draw_data (k_colors.cu) writes that row into the gradient's ramp word in the frame's draw data. No pipeline kernel
// changes: fine reads the row as any other, bounded by cfg.n_ramps.

// One CTA per bound gradient, one thread per texel: its ramp row from its stops, stop k (global over the scene's ramp patches)
// read from the caller's row when k < n_rows and all five values are finite, else as encoded.
__global__ void __launch_bounds__(RS_SAMPLES) k_bound_ramps(const RsRamp *__restrict__ grads, const RsStop *__restrict__ enc,
                                                            const uint8_t *__restrict__ rows, uint32_t n_rows, uint32_t pitch, uint32_t *out) {
    const RsRamp rp = grads[blockIdx.x];
    const uint32_t i = threadIdx.x;
    auto stop = [&](uint32_t j) {
        const uint32_t k = rp.first_stop + j;
        RsStop s = enc[k];
        if (k < n_rows) {
            const float *row = reinterpret_cast<const float *>(rows + (size_t)k * pitch);
            const RsStop t = {__ldg(row), __ldg(row + 1), __ldg(row + 2), __ldg(row + 3), __ldg(row + 4)};
            if (isfinite(t.offset) && isfinite(t.r) && isfinite(t.g) && isfinite(t.b) && isfinite(t.a)) s = t;
        }
        return s;
    };
    out[(size_t)blockIdx.x * RS_SAMPLES + i] = rs_ramp_texel(i, rp.n_stops, rp.premul, stop);
}

extern "C" void vb_launch_resolve_finish(uint32_t *scene, uint32_t n_tag_bytes, uint32_t n_open_clips, uint32_t padded_tag_bytes,
                                         uint32_t end_clip_word0, const RsPatch *patches, uint32_t n_patches, cudaStream_t st) {
    const uint32_t work = max(max(padded_tag_bytes - n_tag_bytes, n_open_clips), n_patches);
    if (work == 0u) return;
    const uint32_t grid = min((work + 255u) / 256u, 592u);
    k_resolve_finish<<<grid, 256, 0, st>>>(scene, n_tag_bytes, n_open_clips, padded_tag_bytes, end_clip_word0, patches, n_patches);
}
extern "C" void vb_launch_make_ramps(const RsRamp *ramps, const RsStop *stops, uint32_t n_ramps, uint32_t *out, cudaStream_t st) {
    if (n_ramps) k_make_ramps<<<n_ramps, RS_SAMPLES, 0, st>>>(ramps, stops, out);
}
extern "C" uint32_t vb_launch_bound_ramps(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbRows &rows = b.bound.rows[VB_BIND_STOPS];
    if (!rows.rows || b.bound.rs_grads_n == 0u) return 0u;
    uint32_t *out = const_cast<uint32_t *>(b.ramps) + (size_t)b.bound.rs_ramp0 * RS_SAMPLES;
    k_bound_ramps<<<b.bound.rs_grads_n, RS_SAMPLES, 0, st>>>(b.bound.rs_grads, b.bound.rs_stops, rows.rows, rows.n, rows.pitch, out);
    return 1u;
}
