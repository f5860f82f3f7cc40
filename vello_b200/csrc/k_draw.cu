// k_draw.cu -- draw-object monoid scan + per-draw info records + clip inputs
// (replaces draw_reduce + draw_leaf).
//
// Reference: vello_shaders/shader/draw_reduce.wgsl:22-55, draw_leaf.wgsl:53-303,
// shared/drawtag.wgsl:47-54, shared/transform.wgsl; CPU twins cpu/draw_reduce.rs, cpu/draw_leaf.rs.
//
// Design: one pass, decoupled look-back over the 4-field monoid (the WGSL strides <= 256
// workgroups over the tags and rescans the reduced prefix in every workgroup).
#include "vb_device.cuh"
#include "vb_stages.h"

#define DR_THREADS 256

struct DXform { float m0, m1, m2, m3, tx, ty; };
__device__ __forceinline__ DXform dx_read(const VbConfig &cfg, const uint32_t *__restrict__ scene, uint32_t ix) {
    uint32_t b = cfg.layout.transform_base + ix * 6u;
    DXform t;
    t.m0 = __uint_as_float(vb_scene(scene, cfg, b));
    t.m1 = __uint_as_float(vb_scene(scene, cfg, b + 1));
    t.m2 = __uint_as_float(vb_scene(scene, cfg, b + 2));
    t.m3 = __uint_as_float(vb_scene(scene, cfg, b + 3));
    t.tx = __uint_as_float(vb_scene(scene, cfg, b + 4));
    t.ty = __uint_as_float(vb_scene(scene, cfg, b + 5));
    return t;
}
__device__ __forceinline__ void dx_apply(const DXform &t, float px, float py, float &ox, float &oy) { // transform.wgsl:12-14
    ox = t.m0 * px + t.m2 * py + t.tx;
    oy = t.m1 * px + t.m3 * py + t.ty;
}
__device__ __forceinline__ DXform dx_inverse(const DXform &t) { // transform.wgsl:16-21
    float inv_det = 1.0f / (t.m0 * t.m3 - t.m1 * t.m2);
    DXform r;
    r.m0 = inv_det * t.m3;
    r.m1 = inv_det * -t.m1;
    r.m2 = inv_det * -t.m2;
    r.m3 = inv_det * t.m0;
    r.tx = r.m0 * -t.tx + r.m2 * -t.ty;
    r.ty = r.m1 * -t.tx + r.m3 * -t.ty;
    return r;
}
__device__ __forceinline__ DXform dx_mul(const DXform &a, const DXform &b) { // transform.wgsl:23-28
    DXform r;
    r.m0 = a.m0 * b.m0 + a.m2 * b.m1;
    r.m1 = a.m1 * b.m0 + a.m3 * b.m1;
    r.m2 = a.m0 * b.m2 + a.m2 * b.m3;
    r.m3 = a.m1 * b.m2 + a.m3 * b.m3;
    r.tx = a.m0 * b.tx + a.m2 * b.ty + a.tx;
    r.ty = a.m1 * b.tx + a.m3 * b.ty + a.ty;
    return r;
}
__device__ __forceinline__ DXform from_poly2(float p0x, float p0y, float p1x, float p1y) { // draw_leaf.wgsl:298-303
    DXform r = {p1y - p0y, p0x - p1x, p1x - p0x, p1y - p0y, p0x, p0y};
    return r;
}
__device__ __forceinline__ DXform two_point_to_unit_line(float p0x, float p0y, float p1x, float p1y) {
    DXform tmp1 = from_poly2(p0x, p0y, p1x, p1y);
    DXform inv = dx_inverse(tmp1);
    DXform tmp2 = from_poly2(0.f, 0.f, 1.f, 0.f);
    return dx_mul(tmp2, inv);
}
__device__ __forceinline__ void put_xform(uint32_t *info, const DXform &x) {
    info[0] = __float_as_uint(x.m0); info[1] = __float_as_uint(x.m1); info[2] = __float_as_uint(x.m2);
    info[3] = __float_as_uint(x.m3); info[4] = __float_as_uint(x.tx); info[5] = __float_as_uint(x.ty);
}

__global__ void __launch_bounds__(DR_THREADS)
k_draw(VbConfig cfg, const uint32_t *__restrict__ scene, const uint2 *__restrict__ path_draw, VbDrawMonoid *draw_monoid,
       uint32_t *info, VbClipInp *clip_inp, uint32_t *lb_mem, uint32_t n_parts) {
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_warp[4][DR_THREADS / 32];
    __shared__ uint32_t sh_prefix[4];
    VbLookback lb = vb_lookback_view(lb_mem, n_parts, 4);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t ix = part * DR_THREADS + threadIdx.x;
    const uint32_t n = cfg.layout.n_draw_objects;
    const uint32_t tag_word = ix < n ? vb_scene(scene, cfg, cfg.layout.draw_tag_base + ix) : VB_DRAWTAG_NOP;
    uint32_t v[4] = {(uint32_t)(tag_word != VB_DRAWTAG_NOP), tag_word & 1u, (tag_word >> 2) & 7u, (tag_word >> 6) & 0xfu};
    uint32_t incl[4];
#pragma unroll
    for (int k = 0; k < 4; k++) incl[k] = vb_warp_incl_scan(v[k]);
    const uint32_t warp = threadIdx.x >> 5, lane = vb_lane();
    if (lane == 31) {
#pragma unroll
        for (int k = 0; k < 4; k++) sh_warp[k][warp] = incl[k];
    }
    __syncthreads();
    uint32_t woff[4], agg[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint32_t o = 0, t = 0;
#pragma unroll
        for (int w = 0; w < DR_THREADS / 32; w++) {
            uint32_t x = sh_warp[k][w];
            if ((uint32_t)w < warp) o += x;
            t += x;
        }
        woff[k] = o;
        agg[k] = t;
    }
    if (warp == 0) {
        uint32_t excl[4];
        vb_lookback<4>(lb, part, agg, excl);
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 4; k++) sh_prefix[k] = excl[k];
        }
    }
    __syncthreads();
    VbDrawMonoid m;
    m.path_ix = sh_prefix[0] + woff[0] + incl[0] - v[0];
    m.clip_ix = sh_prefix[1] + woff[1] + incl[1] - v[1];
    m.scene_offset = sh_prefix[2] + woff[2] + incl[2] - v[2];
    m.info_offset = sh_prefix[3] + woff[3] + incl[3] - v[3];
    if (ix >= n) return;
    draw_monoid[ix] = m;
    const uint32_t dd = cfg.layout.draw_data_base + m.scene_offset;
    const uint32_t di = m.info_offset;
    if (tag_word == VB_DRAWTAG_FILL_COLOR || tag_word == VB_DRAWTAG_FILL_LIN_GRADIENT || tag_word == VB_DRAWTAG_FILL_RAD_GRADIENT ||
        tag_word == VB_DRAWTAG_FILL_SWEEP_GRADIENT || tag_word == VB_DRAWTAG_FILL_IMAGE || tag_word == VB_DRAWTAG_BEGIN_CLIP ||
        tag_word == VB_DRAWTAG_BLURRED_ROUNDED_RECT) {
        const uint2 pd = path_draw[m.path_ix]; // {style_ix, trans_ix}: the draw flags are the style's fill rule (fl_open_path)
        info[di] = (vb_scene(scene, cfg, cfg.layout.style_base + pd.x) & STYLE_FLAGS_FILL) == 0u ? 0u : 1u;
        if (tag_word != VB_DRAWTAG_FILL_COLOR && tag_word != VB_DRAWTAG_BEGIN_CLIP) {
            DXform transform = dx_read(cfg, scene, pd.y);
            switch (tag_word) {
            case VB_DRAWTAG_FILL_LIN_GRADIENT: {
                float p0x, p0y, p1x, p1y;
                dx_apply(transform, __uint_as_float(vb_scene(scene, cfg, dd + 1)), __uint_as_float(vb_scene(scene, cfg, dd + 2)), p0x, p0y);
                dx_apply(transform, __uint_as_float(vb_scene(scene, cfg, dd + 3)), __uint_as_float(vb_scene(scene, cfg, dd + 4)), p1x, p1y);
                float dx = p1x - p0x, dy = p1y - p0y;
                float scale = 1.0f / (dx * dx + dy * dy);
                float lx = dx * scale, ly = dy * scale;
                float line_c = -(p0x * lx + p0y * ly);
                info[di + 1] = __float_as_uint(lx);
                info[di + 2] = __float_as_uint(ly);
                info[di + 3] = __float_as_uint(line_c);
                break;
            }
            case VB_DRAWTAG_FILL_RAD_GRADIENT: {
                const float GRADIENT_EPSILON = 1.0f / (float)(1u << 12);
                float p0x = __uint_as_float(vb_scene(scene, cfg, dd + 1)), p0y = __uint_as_float(vb_scene(scene, cfg, dd + 2));
                float p1x = __uint_as_float(vb_scene(scene, cfg, dd + 3)), p1y = __uint_as_float(vb_scene(scene, cfg, dd + 4));
                float r0 = __uint_as_float(vb_scene(scene, cfg, dd + 5));
                float r1 = __uint_as_float(vb_scene(scene, cfg, dd + 6));
                DXform user_to_gradient = dx_inverse(transform);
                DXform xform = {0, 0, 0, 0, 0, 0};
                float focal_x = 0.0f, radius = 0.0f;
                uint32_t kind = 0u, flags = 0u;
                if (fabsf(r0 - r1) <= GRADIENT_EPSILON) {
                    kind = 2u;
                    float ddx = p0x - p1x, ddy = p0y - p1y;
                    float scaled = r0 / sqrtf(ddx * ddx + ddy * ddy);
                    xform = dx_mul(two_point_to_unit_line(p0x, p0y, p1x, p1y), user_to_gradient);
                    radius = scaled * scaled;
                } else {
                    kind = 4u;
                    if (p0x == p1x && p0y == p1y) {
                        kind = 1u;
                        p0x += GRADIENT_EPSILON;
                        p0y += GRADIENT_EPSILON;
                    }
                    if (r1 == 0.0f) {
                        flags |= 1u;
                        float t;
                        t = p0x; p0x = p1x; p1x = t;
                        t = p0y; p0y = p1y; p1y = t;
                        t = r0; r0 = r1; r1 = t;
                    }
                    focal_x = r0 / (r0 - r1);
                    float cfx = (1.0f - focal_x) * p0x + focal_x * p1x, cfy = (1.0f - focal_x) * p0y + focal_x * p1y;
                    float ex = cfx - p1x, ey = cfy - p1y;
                    radius = r1 / sqrtf(ex * ex + ey * ey);
                    DXform user_to_unit_line = dx_mul(two_point_to_unit_line(cfx, cfy, p1x, p1y), user_to_gradient);
                    DXform user_to_scaled;
                    if (fabsf(radius - 1.0f) <= GRADIENT_EPSILON) {
                        kind = 3u;
                        float scale = 0.5f * fabsf(1.0f - focal_x);
                        DXform s = {scale, 0.f, 0.f, scale, 0.f, 0.f};
                        user_to_scaled = dx_mul(s, user_to_unit_line);
                    } else {
                        float a = radius * radius - 1.0f;
                        float scale_ratio = fabsf(1.0f - focal_x) / a;
                        float scale_x = radius * scale_ratio;
                        float scale_y = sqrtf(fabsf(a)) * scale_ratio;
                        DXform s = {scale_x, 0.f, 0.f, scale_y, 0.f, 0.f};
                        user_to_scaled = dx_mul(s, user_to_unit_line);
                    }
                    xform = user_to_scaled;
                }
                put_xform(info + di + 1, xform);
                info[di + 7] = __float_as_uint(focal_x);
                info[di + 8] = __float_as_uint(radius);
                info[di + 9] = (flags << 3) | kind;
                break;
            }
            case VB_DRAWTAG_FILL_SWEEP_GRADIENT: {
                DXform tr = {1.f, 0.f, 0.f, 1.f, __uint_as_float(vb_scene(scene, cfg, dd + 1)), __uint_as_float(vb_scene(scene, cfg, dd + 2))};
                DXform inv = dx_inverse(dx_mul(transform, tr));
                put_xform(info + di + 1, inv);
                info[di + 7] = vb_scene(scene, cfg, dd + 3);
                info[di + 8] = vb_scene(scene, cfg, dd + 4);
                break;
            }
            case VB_DRAWTAG_FILL_IMAGE: {
                DXform inv = dx_inverse(transform);
                put_xform(info + di + 1, inv);
                info[di + 7] = vb_scene(scene, cfg, dd);
                info[di + 8] = vb_scene(scene, cfg, dd + 1);
                info[di + 9] = vb_scene(scene, cfg, dd + 2);
                break;
            }
            case VB_DRAWTAG_BLURRED_ROUNDED_RECT: {
                DXform inv = dx_inverse(transform);
                put_xform(info + di + 1, inv);
                info[di + 7] = vb_scene(scene, cfg, dd + 1);
                info[di + 8] = vb_scene(scene, cfg, dd + 2);
                info[di + 9] = vb_scene(scene, cfg, dd + 3);
                info[di + 10] = vb_scene(scene, cfg, dd + 4);
                break;
            }
            default: break;
            }
        }
    }
    if (tag_word == VB_DRAWTAG_BEGIN_CLIP || tag_word == VB_DRAWTAG_END_CLIP) {
        uint32_t path_ix = tag_word == VB_DRAWTAG_BEGIN_CLIP ? m.path_ix : ~ix;
        if (m.clip_ix < cfg.layout.n_clips) {
            VbClipInp ci;
            ci.ix = ix;
            ci.path_ix = (int32_t)path_ix;
            clip_inp[m.clip_ix] = ci;
        }
    }
}

extern "C" uint32_t vb_launch_draw(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (b.parts_draw == 0) return 0;
    k_draw<<<b.parts_draw, DR_THREADS, 0, st>>>(cfg, b.scene, b.path_draw, b.draw_monoids, b.info_bin_data, b.clip_inp, b.lb_draw, b.parts_draw);
    return 1;
}
extern "C" uint32_t vb_draw_parts(uint32_t n_draw) { return (n_draw + DR_THREADS - 1) / DR_THREADS; }
