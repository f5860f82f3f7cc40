/* vbo_fine.c -- CPU ORACLE, fine rasterisation.  TEST INFRASTRUCTURE ONLY (see vbo.h).
 *
 * Restated from vello_shaders/shader/fine.wgsl (area: :1005-1059, msaa: :146-709, PTCL
 * interpreter: :1064-1398) and shader/shared/blend.wgsl. One "workgroup" = one 16x16 tile;
 * a WGSL thread owns 4 horizontally adjacent pixels and several expressions are evaluated
 * relative to the thread's first pixel (e.g. `d + line_x * f32(i)`), which is reproduced here
 * so that float results are bit-identical to a faithful GPU execution of the same arithmetic.
 *
 * Conventions fixed where WGSL leaves latitude (same choices in the CUDA kernels):
 *   unpack4x8unorm: byte / 255.0f;  pack4x8unorm and the rgba8unorm store: floor(0.5 + 255 x);
 *   round(): ties to even (rintf);   mix(a, b, t) = a * (1 - t) + b * t;   pow(x, 2.0) = x * x.
 */
#include <pthread.h>

#include "vbo_internal.h"

enum { CMD_END = 0, CMD_FILL = 1, CMD_SOLID = 3, CMD_COLOR = 5, CMD_LIN_GRAD = 6, CMD_RAD_GRAD = 7, CMD_SWEEP_GRAD = 8,
       CMD_IMAGE = 9, CMD_BEGIN_CLIP = 10, CMD_END_CLIP = 11, CMD_JUMP = 12, CMD_BLUR_RECT = 13 };
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define GRADIENT_WIDTH 512

typedef struct { float r, g, b, a; } rgba_t;
static inline rgba_t RG(float r, float g, float b, float a) { rgba_t c = {r, g, b, a}; return c; }
static inline rgba_t rg_scale(rgba_t c, float s) { return RG(c.r * s, c.g * s, c.b * s, c.a * s); }
static inline rgba_t unpack4x8unorm(uint32_t u) {
    return RG((float)(u & 0xffu) / 255.0f, (float)((u >> 8) & 0xffu) / 255.0f, (float)((u >> 16) & 0xffu) / 255.0f,
              (float)(u >> 24) / 255.0f);
}
static inline uint32_t unorm8(float x) { return (uint32_t)floorf(0.5f + 255.0f * fminf(1.0f, fmaxf(0.0f, x))); }
static inline uint32_t pack4x8unorm(rgba_t c) {
    return unorm8(c.r) | (unorm8(c.g) << 8) | (unorm8(c.b) << 16) | (unorm8(c.a) << 24);
}
/* rgba = rgba * (1 - fg.a) + fg  (fine.wgsl:1117), evaluated as a fused multiply-add: WGSL lets the implementation
 * contract a*b+c, and GPU back ends do; this is one of the conventions shared with the CUDA kernel. */
static inline rgba_t over(rgba_t bg, rgba_t fg) {
    float k = 1.0f - fg.a;
    return RG(fmaf(bg.r, k, fg.r), fmaf(bg.g, k, fg.g), fmaf(bg.b, k, fg.b), fmaf(bg.a, k, fg.a));
}

/* Sizes of every buffer the interpreter reads or writes: fine may be replayed on buffers another implementation wrote
 * (vbo_set_buffer), so each access is checked and a reference outside a buffer fails the run instead of reading or
 * writing past it. */
typedef struct {
    const vbo_ctx *c;
    const uint32_t *ptcl, *info;
    const Segment *segments;
    uint32_t *blend_spill;
    size_t n_ptcl, n_info, n_segments, n_spill;
    int *error;
} FineIn;

static void fine_fail(const FineIn *in) { __atomic_store_n(in->error, 1, __ATOMIC_RELAXED); }
static uint32_t cmd_words(uint32_t tag) {
    switch (tag) {
    case CMD_FILL: return 4u;
    case CMD_COLOR: case CMD_IMAGE: case CMD_JUMP: return 2u;
    case CMD_LIN_GRAD: case CMD_RAD_GRAD: case CMD_SWEEP_GRAD: case CMD_END_CLIP: case CMD_BLUR_RECT: return 3u;
    default: return 1u;
    }
}
static int in_range(size_t start, size_t n, size_t size) { return start <= size && n <= size - start; }

/* ---------------- area coverage: fine.wgsl:1005-1059 ---------------- */
static void fill_path_area(const FineIn *in, uint32_t size_and_rule, uint32_t seg_data, int32_t backdrop, float *area) {
    uint32_t n_segs = size_and_rule >> 1;
    int even_odd = (size_and_rule & 1u) != 0u;
    float backdrop_f = (float)backdrop;
    for (int i = 0; i < 256; i++) area[i] = backdrop_f;
    for (uint32_t s = 0; s < n_segs; s++) {
        Segment seg = in->segments[seg_data + s];
        float deltax = seg.p1[0] - seg.p0[0], deltay = seg.p1[1] - seg.p0[1];
        for (int ly = 0; ly < 16; ly++) {
            float xyy = (float)ly;
            float y = seg.p0[1] - xyy;
            float y0 = clampf(y, 0.0f, 1.0f);
            float y1 = clampf(y + deltay, 0.0f, 1.0f);
            float dy = y0 - y1;
            float y_edge = signf(deltax) * clampf(xyy - seg.y_edge + 1.0f, 0.0f, 1.0f);
            for (int gx = 0; gx < 4; gx++) {
                float xyx = (float)(gx * 4);
                float *ar = area + ly * 16 + gx * 4;
                if (dy != 0.0f) {
                    float vec_y_recip = 1.0f / deltay;
                    float t0 = (y0 - y) * vec_y_recip;
                    float t1 = (y1 - y) * vec_y_recip;
                    float startx = seg.p0[0] - xyx;
                    float x0 = startx + t0 * deltax;
                    float x1 = startx + t1 * deltax;
                    float xmin0 = fminf(x0, x1);
                    float xmax0 = fmaxf(x0, x1);
                    for (int i = 0; i < 4; i++) {
                        float i_f = (float)i;
                        float xmin = fminf(xmin0 - i_f, 1.0f) - 1.0e-6f;
                        float xmax = xmax0 - i_f;
                        float b = fminf(xmax, 1.0f);
                        float cc = fmaxf(b, 0.0f);
                        float d = fmaxf(xmin, 0.0f);
                        float a = (b + 0.5f * (d * d - cc * cc) - xmin) / (xmax - xmin);
                        ar[i] += a * dy;
                    }
                }
                for (int i = 0; i < 4; i++) ar[i] += y_edge;
            }
        }
    }
    if (even_odd) {
        for (int i = 0; i < 256; i++) {
            float a = area[i];
            area[i] = fabsf(a - 2.0f * rintf(0.5f * a));
        }
    } else {
        for (int i = 0; i < 256; i++) area[i] = fminf(fabsf(area[i]), 1.0f);
    }
}

/* ---------------- MSAA coverage: fine.wgsl:146-709 ----------------
 * The shared-memory SWAR state is reproduced word for word; the atomics commute, so segments and
 * their pixel touches are visited serially here. */
typedef struct {
    uint32_t sh_winding_y[4], sh_winding_y_prefix[4], sh_winding[64], sh_samples[1024];
} MsState;

static void fill_path_ms(const FineIn *in, const uint32_t *mask_lut, int msaa16, uint32_t size_and_rule, uint32_t seg_data,
                         int32_t backdrop, float *area) {
    MsState st;
    uint32_t n_segs = size_and_rule >> 1;
    int even_odd = (size_and_rule & 1u) != 0u;
    const uint32_t MASK_WIDTH = msaa16 ? 64u : 32u, MASK_HEIGHT = MASK_WIDTH;
    const uint32_t WPP = msaa16 ? 4u : 2u; /* SAMPLE_WORDS_PER_PIXEL */
    if (even_odd) {
        st.sh_winding_y[0] = 0u;
        for (int i = 0; i < 16; i++) st.sh_winding[i] = 0u;
        for (int i = 0; i < 256; i++) st.sh_samples[i] = 0u;
    } else {
        for (int i = 0; i < 4; i++) st.sh_winding_y[i] = 0x80808080u;
        for (int i = 0; i < 64; i++) st.sh_winding[i] = 0x80808080u;
        for (uint32_t i = 0; i < 256u * WPP; i++) st.sh_samples[i] = 0x80808080u;
    }
    for (uint32_t s = 0; s < n_segs; s++) {
        Segment seg = in->segments[seg_data + s];
        v2 p0 = V2(seg.p0[0], seg.p0[1]), p1 = V2(seg.p1[0], seg.p1[1]);
        uint32_t count = 0u;
        {
            float y_edge_f = 16.0f;
            int32_t delta = (p1.x <= p0.x) ? 1 : -1;
            if (p0.x == 0.0f) y_edge_f = p0.y;
            else if (p1.x == 0.0f) y_edge_f = p1.y;
            if (!(p0.y == p1.y && p0.y == floorf(p0.y))) count = span_u(p0.x, p1.x) + span_u(p0.y, p1.y) - 1u;
            uint32_t y_edge = f2u_sat(ceilf(y_edge_f));
            if (y_edge < 16u) {
                if (even_odd) st.sh_winding_y[0] ^= 1u << y_edge;
                else st.sh_winding_y[y_edge >> 2] += ((uint32_t)delta) << ((y_edge & 3u) << 3);
            }
        }
        if (count == 0u) continue;
        int is_down = p1.y >= p0.y;
        v2 xy0 = is_down ? p0 : p1;
        v2 xy1 = is_down ? p1 : p0;
        float dx = fabsf(xy1.x - xy0.x);
        float dy = xy1.y - xy0.y;
        float idxdy = 1.0f / (dx + dy);
        float a = dx * idxdy;
        int is_positive_slope = xy1.x >= xy0.x;
        float x_sign = is_positive_slope ? 1.0f : -1.0f;
        float xt0 = floorf(xy0.x * x_sign);
        float cc = xy0.x * x_sign - xt0;
        float y0i = floorf(xy0.y);
        float ytop = y0i + 1.0f;
        float b = fminf((dy * cc + dx * (ytop - xy0.y)) * idxdy, ONE_MINUS_ULP);
        uint32_t count_x = span_u(xy0.x, xy1.x) - 1u;
        uint32_t count_full = count_x + span_u(xy0.y, xy1.y);
        float robust_err = floorf(a * ((float)count_full - 1.0f) + b) - (float)count_x;
        if (robust_err != 0.0f) a -= ROBUST_EPSILON * signf(robust_err);
        int32_t x0i = f2i_sat(xt0 * x_sign + 0.5f * (x_sign - 1.0f));
        for (uint32_t sub_ix = 0; sub_ix < count; sub_ix++) {
            int last_pixel = sub_ix + 1u == count;
            float zf = a * (float)sub_ix + b;
            float z = floorf(zf);
            int32_t x = x0i + f2i_sat(x_sign * z);
            int32_t y = f2i_sat(y0i) + (int32_t)sub_ix - f2i_sat(z);
            int is_delta, is_bump = 0;
            if (sub_ix == 0u) {
                is_delta = y0i == xy0.y;
                is_bump = even_odd ? (xy0.x == 0.0f) : (xy0.x == 0.0f && y0i != xy0.y);
            } else {
                float zp = floorf(a * (float)(sub_ix - 1u) + b);
                is_delta = z == zp;
                is_bump = is_positive_slope && !is_delta;
            }
            uint32_t pix_ix = (uint32_t)y * 16u + (uint32_t)x;
            if ((uint32_t)x < 15u && (uint32_t)y < 16u) {
                if (is_delta) {
                    if (even_odd) {
                        st.sh_winding[y] ^= 2u << (uint32_t)x;
                    } else {
                        uint32_t delta_pix = pix_ix + 1u;
                        uint32_t d = (is_down ? 1u : 0xffffffffu) << ((delta_pix & 3u) << 3);
                        st.sh_winding[delta_pix >> 2] += d;
                    }
                }
            }
            uint32_t mask_block = (uint32_t)is_positive_slope * (MASK_WIDTH * MASK_HEIGHT / 2u);
            float half_height = (float)(MASK_HEIGHT / 2u);
            float mask_row = floorf(fminf(a * half_height, half_height - 1.0f)) * (float)MASK_WIDTH;
            float mask_col = floorf((zf - z) * (float)MASK_WIDTH);
            uint32_t mask_ix = mask_block + f2u_sat(mask_row + mask_col);
            if (pix_ix >= 256u) continue; /* out-of-tile touches write nowhere meaningful */
            if (!msaa16) {
                uint32_t mask = (mask_lut[(mask_ix / 4u) & 255u] >> ((mask_ix % 4u) * 8u)) & 0xffu;
                if (sub_ix == 0u && !is_bump) {
                    uint32_t sh = f2u_sat(rintf(8.0f * (xy0.y - (float)y)));
                    mask &= sh < 32u ? (0xffu << sh) : 0u;
                }
                if (last_pixel && xy1.x != 0.0f) {
                    uint32_t sh = f2u_sat(rintf(8.0f * (xy1.y - (float)y)));
                    mask &= ~(sh < 32u ? (0xffu << sh) : 0u);
                }
                if (even_odd) {
                    if (is_bump) mask ^= 0xffu;
                    st.sh_samples[pix_ix] ^= mask;
                } else {
                    uint32_t mask_a = mask ^ (mask << 7);
                    uint32_t mask_b = mask_a ^ (mask_a << 14);
                    uint32_t m0 = mask_b & 0x1010101u, m1 = (mask_b >> 4) & 0x1010101u;
                    uint32_t m0s = is_down ? (uint32_t)(-(int32_t)m0) : m0;
                    uint32_t m1s = is_down ? (uint32_t)(-(int32_t)m1) : m1;
                    if (is_bump) {
                        uint32_t bd = is_down ? 0x1010101u : (uint32_t)(-(int32_t)0x1010101);
                        m0s += bd; m1s += bd;
                    }
                    st.sh_samples[pix_ix * 2u] += m0s;
                    st.sh_samples[pix_ix * 2u + 1u] += m1s;
                }
            } else {
                uint32_t mask = (mask_lut[(mask_ix / 2u) & 2047u] >> ((mask_ix % 2u) * 16u)) & 0xffffu;
                if (sub_ix == 0u && !is_bump) {
                    uint32_t sh = f2u_sat(rintf(16.0f * (xy0.y - (float)y)));
                    mask &= sh < 32u ? (0xffffu << sh) : 0u;
                }
                if (last_pixel && xy1.x != 0.0f) {
                    uint32_t sh = f2u_sat(rintf(16.0f * (xy1.y - (float)y)));
                    mask &= ~(sh < 32u ? (0xffffu << sh) : 0u);
                }
                if (even_odd) {
                    if (is_bump) mask ^= 0xffffu;
                    st.sh_samples[pix_ix] ^= mask;
                } else {
                    uint32_t mask0 = mask & 0xffu;
                    uint32_t mask0_a = mask0 ^ (mask0 << 7);
                    uint32_t mask0_b = mask0_a ^ (mask0_a << 14);
                    uint32_t e0 = mask0_b & 0x1010101u, e1 = (mask0_b >> 4) & 0x1010101u;
                    uint32_t mask1 = (mask >> 8) & 0xffu;
                    uint32_t mask1_a = mask1 ^ (mask1 << 7);
                    uint32_t mask1_b = mask1_a ^ (mask1_a << 14);
                    uint32_t e2 = mask1_b & 0x1010101u, e3 = (mask1_b >> 4) & 0x1010101u;
                    uint32_t s0 = is_down ? (uint32_t)(-(int32_t)e0) : e0;
                    uint32_t s1 = is_down ? (uint32_t)(-(int32_t)e1) : e1;
                    uint32_t s2 = is_down ? (uint32_t)(-(int32_t)e2) : e2;
                    uint32_t s3 = is_down ? (uint32_t)(-(int32_t)e3) : e3;
                    if (is_bump) {
                        uint32_t bd = is_down ? 0x1010101u : (uint32_t)(-(int32_t)0x1010101);
                        s0 += bd; s1 += bd; s2 += bd; s3 += bd;
                    }
                    st.sh_samples[pix_ix * 4u] += s0;
                    st.sh_samples[pix_ix * 4u + 1u] += s1;
                    st.sh_samples[pix_ix * 4u + 2u] += s2;
                    st.sh_samples[pix_ix * 4u + 3u] += s3;
                }
            }
        }
    }
    /* resolve */
    if (even_odd) {
        for (uint32_t ly = 0; ly < 16; ly++) {
            uint32_t scan_x = st.sh_winding[ly];
            scan_x ^= scan_x << 1; scan_x ^= scan_x << 2; scan_x ^= scan_x << 4; scan_x ^= scan_x << 8;
            uint32_t scan_y = st.sh_winding_y[0];
            scan_y ^= scan_y << 1; scan_y ^= scan_y << 2; scan_y ^= scan_y << 4; scan_y ^= scan_y << 8;
            uint32_t row_parity = (scan_y >> ly) ^ (uint32_t)backdrop;
            for (uint32_t lx = 0; lx < 16; lx++) {
                uint32_t pix_ix = ly * 16u + lx;
                uint32_t samples = st.sh_samples[pix_ix];
                uint32_t pix_parity = row_parity ^ (scan_x >> (pix_ix % 16u));
                uint32_t pix_mask = (uint32_t)(-(int32_t)(pix_parity & 1u));
                if (msaa16) area[pix_ix] = (float)__builtin_popcount((samples ^ pix_mask) & 0xffffu) * 0.0625f;
                else area[pix_ix] = (float)__builtin_popcount((samples ^ pix_mask) & 0xffu) * 0.125f;
            }
        }
        return;
    }
    uint32_t packed_w_arr[64], wind_y_arr[64];
    uint32_t new_winding[64];
    for (uint32_t th = 0; th < 64; th++) {
        uint32_t lx = th & 3u, ly = th >> 2;
        uint32_t major = th;
        uint32_t packed_w = st.sh_winding[major];
        packed_w += (packed_w - 0x808080u) << 8;
        packed_w += (packed_w - 0x8080u) << 16;
        uint32_t packed_y = st.sh_winding_y[ly >> 2];
        packed_y += (packed_y - 0x808080u) << 8;
        packed_y += (packed_y - 0x8080u) << 16;
        uint32_t wind_y = (packed_y >> ((ly & 3u) << 3)) - 0x80u;
        if ((ly & 3u) == 3u && lx == 0u) st.sh_winding_y_prefix[ly >> 2] = wind_y;
        uint32_t prefix_x = ((packed_w >> 24) - 0x80u) * 0x1010101u;
        new_winding[major] = prefix_x;
        packed_w_arr[th] = packed_w;
        wind_y_arr[th] = wind_y;
    }
    for (uint32_t th = 0; th < 64; th++) {
        uint32_t ly = th >> 2;
        uint32_t major = th;
        uint32_t packed_w = packed_w_arr[th];
        for (uint32_t i = (major & ~3u); i < major; i++) packed_w += new_winding[i];
        uint32_t wind_y = wind_y_arr[th];
        for (uint32_t i = 0; i < (ly >> 2); i++) wind_y += st.sh_winding_y_prefix[i];
        for (uint32_t i = 0; i < 4; i++) {
            uint32_t pix_ix = th * 4u + i;
            uint32_t expected_zero = (((packed_w >> (i * 8u)) + wind_y) & 0xffu) - (uint32_t)backdrop;
            if (expected_zero >= 256u) {
                area[pix_ix] = 1.0f;
            } else if (!msaa16) {
                uint32_t samples0 = st.sh_samples[pix_ix * 2u], samples1 = st.sh_samples[pix_ix * 2u + 1u];
                uint32_t xored0 = (expected_zero * 0x1010101u) ^ samples0;
                uint32_t xored0_2 = xored0 | (xored0 * 2u);
                uint32_t xored1 = (expected_zero * 0x1010101u) ^ samples1;
                uint32_t xored1_2 = xored1 | (xored1 >> 1);
                uint32_t xored2 = (xored0_2 & 0xAAAAAAAAu) | (xored1_2 & 0x55555555u);
                uint32_t xored4 = xored2 | (xored2 * 4u);
                uint32_t xored8 = xored4 | (xored4 * 16u);
                area[pix_ix] = (float)__builtin_popcount(xored8 & 0xC0C0C0C0u) * 0.125f;
            } else {
                uint32_t sm0 = st.sh_samples[pix_ix * 4u], sm1 = st.sh_samples[pix_ix * 4u + 1u];
                uint32_t sm2 = st.sh_samples[pix_ix * 4u + 2u], sm3 = st.sh_samples[pix_ix * 4u + 3u];
                uint32_t ez = expected_zero * 0x1010101u;
                uint32_t xored0 = ez ^ sm0;
                uint32_t xored0_2 = xored0 | (xored0 * 2u);
                uint32_t xored1 = ez ^ sm1;
                uint32_t xored1_2 = xored1 | (xored1 >> 1);
                uint32_t xored01 = (xored0_2 & 0xAAAAAAAAu) | (xored1_2 & 0x55555555u);
                uint32_t xored01_4 = xored01 | (xored01 * 4u);
                uint32_t xored2 = ez ^ sm2;
                uint32_t xored2_2 = xored2 | (xored2 * 2u);
                uint32_t xored3 = ez ^ sm3;
                uint32_t xored3_2 = xored3 | (xored3 >> 1);
                uint32_t xored23 = (xored2_2 & 0xAAAAAAAAu) | (xored3_2 & 0x55555555u);
                uint32_t xored23_4 = xored23 | (xored23 >> 2);
                uint32_t xored4 = (xored01_4 & 0xCCCCCCCCu) | (xored23_4 & 0x33333333u);
                uint32_t xored8 = xored4 | (xored4 * 16u);
                area[pix_ix] = (float)__builtin_popcount(xored8 & 0xF0F0F0F0u) * 0.0625f;
            }
        }
    }
}

/* ---------------- blend.wgsl ---------------- */
typedef struct { float x, y, z; } v3;
static inline v3 V3(float x, float y, float z) { v3 r = {x, y, z}; return r; }
static float color_dodge(float cb, float cs) {
    if (cb == 0.0f) return 0.0f;
    if (cs == 1.0f) return 1.0f;
    return fminf(1.0f, cb / (1.0f - cs));
}
static float color_burn(float cb, float cs) {
    if (cb == 1.0f) return 1.0f;
    if (cs == 0.0f) return 0.0f;
    return 1.0f - fminf(1.0f, (1.0f - cb) / cs);
}
static float screen1(float cb, float cs) { return cb + cs - (cb * cs); }
static float hard_light1(float cb, float cs) { return cs <= 0.5f ? cb * 2.0f * cs : screen1(cb, 2.0f * cs - 1.0f); }
static float soft_light1(float cb, float cs) {
    float d = cb <= 0.25f ? ((16.0f * cb - 12.0f) * cb + 4.0f) * cb : sqrtf(cb);
    return cs <= 0.5f ? cb - (1.0f - 2.0f * cs) * cb * (1.0f - cb) : cb + (2.0f * cs - 1.0f) * (d - cb);
}
static float sat3(v3 c) { return fmaxf(c.x, fmaxf(c.y, c.z)) - fminf(c.x, fminf(c.y, c.z)); }
static float dot3(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static float lum(v3 c) { return dot3(c, V3(0.3f, 0.59f, 0.11f)); }
static float svg_lum(v3 c) { return dot3(c, V3(0.2125f, 0.7154f, 0.0721f)); }
static v3 clip_color(v3 c) {
    float l = lum(c);
    float n = fminf(c.x, fminf(c.y, c.z));
    float x = fmaxf(c.x, fmaxf(c.y, c.z));
    if (n < 0.0f) c = V3(l + (((c.x - l) * l) / (l - n)), l + (((c.y - l) * l) / (l - n)), l + (((c.z - l) * l) / (l - n)));
    if (x > 1.0f)
        c = V3(l + (((c.x - l) * (1.0f - l)) / (x - l)), l + (((c.y - l) * (1.0f - l)) / (x - l)),
               l + (((c.z - l) * (1.0f - l)) / (x - l)));
    return c;
}
static v3 set_lum(v3 c, float l) {
    float d = l - lum(c);
    return clip_color(V3(c.x + d, c.y + d, c.z + d));
}
static void set_sat_inner(float *cmin, float *cmid, float *cmax, float s) {
    if (*cmax > *cmin) {
        *cmid = ((*cmid - *cmin) * s) / (*cmax - *cmin);
        *cmax = s;
    } else {
        *cmid = 0.0f;
        *cmax = 0.0f;
    }
    *cmin = 0.0f;
}
static v3 set_sat(v3 c, float s) {
    float r = c.x, g = c.y, b = c.z;
    if (r <= g) {
        if (g <= b) set_sat_inner(&r, &g, &b, s);
        else if (r <= b) set_sat_inner(&r, &b, &g, s);
        else set_sat_inner(&b, &r, &g, s);
    } else {
        if (r <= b) set_sat_inner(&g, &r, &b, s);
        else if (g <= b) set_sat_inner(&g, &b, &r, s);
        else set_sat_inner(&b, &g, &r, s);
    }
    return V3(r, g, b);
}
static v3 blend_mix(v3 cb, v3 cs, uint32_t mode) {
    switch (mode) {
    case 1: return V3(cb.x * cs.x, cb.y * cs.y, cb.z * cs.z);
    case 2: return V3(screen1(cb.x, cs.x), screen1(cb.y, cs.y), screen1(cb.z, cs.z));
    case 3: return V3(hard_light1(cs.x, cb.x), hard_light1(cs.y, cb.y), hard_light1(cs.z, cb.z));
    case 4: return V3(fminf(cb.x, cs.x), fminf(cb.y, cs.y), fminf(cb.z, cs.z));
    case 5: return V3(fmaxf(cb.x, cs.x), fmaxf(cb.y, cs.y), fmaxf(cb.z, cs.z));
    case 6: return V3(color_dodge(cb.x, cs.x), color_dodge(cb.y, cs.y), color_dodge(cb.z, cs.z));
    case 7: return V3(color_burn(cb.x, cs.x), color_burn(cb.y, cs.y), color_burn(cb.z, cs.z));
    case 8: return V3(hard_light1(cb.x, cs.x), hard_light1(cb.y, cs.y), hard_light1(cb.z, cs.z));
    case 9: return V3(soft_light1(cb.x, cs.x), soft_light1(cb.y, cs.y), soft_light1(cb.z, cs.z));
    case 10: return V3(fabsf(cb.x - cs.x), fabsf(cb.y - cs.y), fabsf(cb.z - cs.z));
    case 11: return V3(cb.x + cs.x - 2.0f * cb.x * cs.x, cb.y + cs.y - 2.0f * cb.y * cs.y, cb.z + cs.z - 2.0f * cb.z * cs.z);
    case 12: return set_lum(set_sat(cs, sat3(cb)), lum(cb));
    case 13: return set_lum(set_sat(cb, sat3(cs)), lum(cb));
    case 14: return set_lum(cs, lum(cb));
    case 15: return set_lum(cb, lum(cs));
    default: return cs;
    }
}
static rgba_t blend_compose(v3 cb, v3 cs, float ab, float as_, uint32_t mode) {
    float fa = 0.0f, fb = 0.0f;
    switch (mode) {
    case 1: fa = 1.0f; fb = 0.0f; break;
    case 2: fa = 0.0f; fb = 1.0f; break;
    case 3: fa = 1.0f; fb = 1.0f - as_; break;
    case 4: fa = 1.0f - ab; fb = 1.0f; break;
    case 5: fa = ab; fb = 0.0f; break;
    case 6: fa = 0.0f; fb = as_; break;
    case 7: fa = 1.0f - ab; fb = 0.0f; break;
    case 8: fa = 0.0f; fb = 1.0f - as_; break;
    case 9: fa = ab; fb = 1.0f - as_; break;
    case 10: fa = 1.0f - ab; fb = as_; break;
    case 11: fa = 1.0f - ab; fb = 1.0f - as_; break;
    case 12: fa = 1.0f; fb = 1.0f; break;
    case 13:
        return RG(fminf(1.0f, as_ * cs.x + ab * cb.x), fminf(1.0f, as_ * cs.y + ab * cb.y), fminf(1.0f, as_ * cs.z + ab * cb.z),
                  fminf(1.0f, as_ + ab));
    default: break;
    }
    float as_fa = as_ * fa, ab_fb = ab * fb;
    return RG(as_fa * cs.x + ab_fb * cb.x, as_fa * cs.y + ab_fb * cb.y, as_fa * cs.z + ab_fb * cb.z, fminf(as_fa + ab_fb, 1.0f));
}
static v3 unpremultiply(rgba_t c) {
    float inv = 1.0f / fmaxf(c.a, 1e-15f);
    return V3(c.r * inv, c.g * inv, c.b * inv);
}
static inline float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; }
static rgba_t blend_mix_compose(rgba_t backdrop, rgba_t src, uint32_t mode) {
    if ((mode & 0x7fffu) == 3u) return over(backdrop, src);
    v3 cs = unpremultiply(src);
    v3 cb = unpremultiply(backdrop);
    v3 mixed = blend_mix(cb, cs, mode >> 8);
    cs = V3(mixf(cs.x, mixed.x, backdrop.a), mixf(cs.y, mixed.y, backdrop.a), mixf(cs.z, mixed.z, backdrop.a));
    uint32_t compose_mode = mode & 0xffu;
    if (compose_mode == 3u) {
        return RG(mixf(backdrop.r, cs.x, src.a), mixf(backdrop.g, cs.y, src.a), mixf(backdrop.b, cs.z, src.a),
                  src.a + backdrop.a * (1.0f - src.a));
    }
    return blend_compose(cb, cs, backdrop.a, src.a, compose_mode);
}

/* ---------------- gradients / images ---------------- */
static float extend_mode_normalized(float t, uint32_t mode) {
    if (mode == 0u) return clampf(t, 0.0f, 1.0f);
    if (mode == 1u) return t - floorf(t);
    return fabsf(t - 2.0f * rintf(0.5f * t));
}
static float extend_mode(float t, uint32_t mode, float max) {
    if (mode == 0u) return clampf(t, 0.0f, max);
    return extend_mode_normalized(t / max, mode) * max;
}
static rgba_t ramp_load(const vbo_ctx *c, int32_t x, uint32_t index) {
    if (index >= c->n_ramps || x < 0 || x >= GRADIENT_WIDTH) return RG(0, 0, 0, 0);
    return unpack4x8unorm(c->ramps[(size_t)index * GRADIENT_WIDTH + (uint32_t)x]);
}
static rgba_t atlas_load(const vbo_ctx *c, float fx, float fy) {
    int32_t x = f2i_sat(fx), y = f2i_sat(fy);
    if (x < 0 || y < 0 || (uint32_t)x >= c->atlas_w || (uint32_t)y >= c->atlas_h) return RG(0, 0, 0, 0);
    const uint8_t *p = c->atlas + ((size_t)y * c->atlas_w + (uint32_t)x) * 4u;
    return RG((float)p[0] / 255.0f, (float)p[1] / 255.0f, (float)p[2] / 255.0f, (float)p[3] / 255.0f);
}
static rgba_t maybe_premul(rgba_t p, uint32_t alpha_type) {
    if (alpha_type == 1u) return p;
    return RG(p.r * p.a, p.g * p.a, p.b * p.a, p.a);
}
static rgba_t pixel_format(rgba_t p, uint32_t format) { return format == 1u ? RG(p.b, p.g, p.r, p.a) : p; }
static float erf7(float x) {
    float y = clampf(x * 1.1283791671f, -100.0f, 100.0f);
    float yy = y * y;
    float z = y + (0.24295f + (0.03395f + 0.0104f * yy) * yy) * (y * yy);
    return z / sqrtf(1.0f + z * z);
}
static float hypot_w(float a, float b) { return sqrtf(a * a + b * b); }

static float single_weight(float t, float a, float b, float c, float d) { return t * (t * (t * d + c) + b) + a; }
static void cubic_weights(float fr, float w[4]) {
    static const float MF[4][4] = {
        {(1.0f / 6.0f) / 3.0f, -(3.0f / 6.0f) / 3.0f - 1.0f / 3.0f, (3.0f / 6.0f) / 3.0f + 2.0f * 1.0f / 3.0f,
         -(1.0f / 6.0f) / 3.0f - 1.0f / 3.0f},
        {1.0f - (2.0f / 6.0f) / 3.0f, 0.0f, -3.0f + (12.0f / 6.0f) / 3.0f + 1.0f / 3.0f, 2.0f - (9.0f / 6.0f) / 3.0f - 1.0f / 3.0f},
        {(1.0f / 6.0f) / 3.0f, (3.0f / 6.0f) / 3.0f + 1.0f / 3.0f, 3.0f - (15.0f / 6.0f) / 3.0f - 2.0f * 1.0f / 3.0f,
         -2.0f + (9.0f / 6.0f) / 3.0f + 1.0f / 3.0f},
        {0.0f, 0.0f, -1.0f / 3.0f, (1.0f / 6.0f) / 3.0f + 1.0f / 3.0f}};
    for (int i = 0; i < 4; i++) w[i] = single_weight(fr, MF[i][0], MF[i][1], MF[i][2], MF[i][3]);
}
static rgba_t bicubic_sample(const vbo_ctx *c, float cx, float cy, float ox, float oy, float mx, float my, uint32_t alpha_type) {
    float fxx = (cx + 0.5f) - floorf(cx + 0.5f), fyy = (cy + 0.5f) - floorf(cy + 0.5f);
    float wx[4], wy[4];
    cubic_weights(fxx, wx);
    cubic_weights(fyy, wy);
    static const float offs[4] = {-1.5f, -0.5f, 0.5f, 1.5f};
    rgba_t rows[4];
    for (int j = 0; j < 4; j++) {
        rgba_t acc = RG(0, 0, 0, 0);
        for (int i = 0; i < 4; i++) {
            rgba_t s = maybe_premul(atlas_load(c, clampf(cx + offs[i], ox, mx), clampf(cy + offs[j], oy, my)), alpha_type);
            if (i == 0) acc = rg_scale(s, wx[0]);
            else acc = RG(acc.r + wx[i] * s.r, acc.g + wx[i] * s.g, acc.b + wx[i] * s.b, acc.a + wx[i] * s.a);
        }
        rows[j] = acc;
    }
    rgba_t r = rg_scale(rows[0], wy[0]);
    for (int j = 1; j < 4; j++)
        r = RG(r.r + wy[j] * rows[j].r, r.g + wy[j] * rows[j].g, r.b + wy[j] * rows[j].b, r.a + wy[j] * rows[j].a);
    float a = clampf(r.a, 0.0f, 1.0f);
    return RG(clampf(r.r, 0.0f, a), clampf(r.g, 0.0f, a), clampf(r.b, 0.0f, a), a);
}

/* ---------------- the per-tile PTCL interpreter: fine.wgsl:1064-1398 ---------------- */
static void fine_tile(const FineIn *in, const uint32_t *mask_lut, uint32_t tile_x, uint32_t tile_y, uint8_t *out) {
    const vbo_ctx *c = in->c;
    const Config *cfg = &c->cfg;
    const uint32_t *ptcl = in->ptcl;
    const uint32_t *info = in->info;
    uint32_t aa = c->params.aa;
    uint32_t tile_ix = tile_y * cfg->width_in_tiles + tile_x;
    rgba_t rgba[256];
    float area[256];
    rgba_t base = unpack4x8unorm(cfg->base_color);
    for (int i = 0; i < 256; i++) { rgba[i] = base; area[i] = 0.0f; }
    uint32_t *stack = NULL; /* packed blend stack, [depth][256] */
    uint32_t stack_cap = 0;
    uint32_t clip_depth = 0u;
    uint32_t cmd_ix = tile_ix * 64u;
    uint32_t blend_offset = in_range(cmd_ix, 1, in->n_ptcl) ? ptcl[cmd_ix] : 0u;
    cmd_ix += 1u;
    for (;;) {
        if (!in_range(cmd_ix, 1, in->n_ptcl) || !in_range(cmd_ix, cmd_words(ptcl[cmd_ix]), in->n_ptcl)) {
            fine_fail(in);
            break;
        }
        uint32_t tag = ptcl[cmd_ix];
        if (tag == CMD_END) break;
        /* brushes that read draw info: the words they read must lie in info_bin_data */
        uint32_t info_n = tag == CMD_LIN_GRAD ? 3u : tag == CMD_RAD_GRAD ? 9u : tag == CMD_SWEEP_GRAD ? 8u : tag == CMD_IMAGE ? 9u
                          : tag == CMD_BLUR_RECT ? 10u : 0u;
        if (info_n && !in_range(ptcl[cmd_ix + (tag == CMD_IMAGE || tag == CMD_BLUR_RECT ? 1u : 2u)], info_n, in->n_info)) {
            fine_fail(in);
            break;
        }
        switch (tag) {
        case CMD_FILL: {
            uint32_t sr = ptcl[cmd_ix + 1], sd = ptcl[cmd_ix + 2];
            int32_t bd = (int32_t)ptcl[cmd_ix + 3];
            if (!in_range(sd, sr >> 1, in->n_segments)) {
                fine_fail(in);
                goto done;
            }
            if (aa == 0u) fill_path_area(in, sr, sd, bd, area);
            else fill_path_ms(in, mask_lut, aa == 2u, sr, sd, bd, area);
            cmd_ix += 4u;
            break;
        }
        case CMD_SOLID:
            for (int i = 0; i < 256; i++) area[i] = 1.0f;
            cmd_ix += 1u;
            break;
        case CMD_COLOR: {
            rgba_t fg = unpack4x8unorm(ptcl[cmd_ix + 1]);
            for (int i = 0; i < 256; i++) rgba[i] = over(rgba[i], rg_scale(fg, area[i]));
            cmd_ix += 2u;
            break;
        }
        case CMD_BEGIN_CLIP: {
            if (clip_depth >= stack_cap) {
                stack_cap = stack_cap ? stack_cap * 2u : 8u;
                stack = realloc(stack, (size_t)stack_cap * 256u * 4u);
            }
            /* mirror the spill buffer traffic (fine.wgsl:1126-1133) at the tile's blend offset */
            int spill = clip_depth >= 4u && in->blend_spill;
            if (spill && !in_range((size_t)blend_offset + (clip_depth - 4u) * 256u, 256, in->n_spill)) {
                fine_fail(in);
                goto done;
            }
            for (int i = 0; i < 256; i++) {
                uint32_t packed = pack4x8unorm(rgba[i]);
                stack[clip_depth * 256u + (uint32_t)i] = packed;
                if (spill) in->blend_spill[blend_offset + (clip_depth - 4u) * 256u + (uint32_t)i] = packed;
                rgba[i] = RG(0, 0, 0, 0);
            }
            clip_depth += 1u;
            cmd_ix += 1u;
            break;
        }
        case CMD_END_CLIP: {
            uint32_t blend = ptcl[cmd_ix + 1];
            float alpha = u2f_bits(ptcl[cmd_ix + 2]);
            if (clip_depth == 0u) {
                fine_fail(in);
                goto done;
            }
            clip_depth -= 1u;
            for (int i = 0; i < 256; i++) {
                rgba_t bg = unpack4x8unorm(stack[clip_depth * 256u + (uint32_t)i]);
                rgba_t fg = rg_scale(rg_scale(rgba[i], area[i]), alpha);
                if (blend == 0x10000u) {
                    if (area[i] == 0.0f) { rgba[i] = bg; continue; }
                    float luminance = clampf(svg_lum(unpremultiply(fg)) * fg.a, 0.0f, 1.0f);
                    rgba[i] = rg_scale(bg, luminance);
                } else {
                    rgba[i] = blend_mix_compose(bg, fg, blend);
                }
            }
            cmd_ix += 3u;
            break;
        }
        case CMD_JUMP:
            cmd_ix = ptcl[cmd_ix + 1];
            break;
        case CMD_BLUR_RECT: {
            uint32_t io = ptcl[cmd_ix + 1];
            rgba_t blur_rgba = unpack4x8unorm(ptcl[cmd_ix + 2]);
            float m0 = u2f_bits(info[io]), m1 = u2f_bits(info[io + 1]), m2 = u2f_bits(info[io + 2]), m3 = u2f_bits(info[io + 3]);
            float tx = u2f_bits(info[io + 4]), ty = u2f_bits(info[io + 5]);
            float bw = u2f_bits(info[io + 6]), bh = u2f_bits(info[io + 7]), bradius = u2f_bits(info[io + 8]);
            float std_dev = fmaxf(u2f_bits(info[io + 9]), 1e-5f);
            float inv_std_dev = 1.0f / std_dev;
            float min_edge = fminf(bw, bh);
            float radius_max = 0.5f * min_edge;
            float r0 = fminf(hypot_w(bradius, std_dev * 1.15f), radius_max);
            float r1 = fminf(hypot_w(bradius, std_dev * 2.0f), radius_max);
            float exponent = 2.0f * r1 / r0;
            float inv_exponent = 1.0f / exponent;
            float ew = 0.5f * inv_std_dev * bw, eh = 0.5f * inv_std_dev * bh;
            float delta = 1.25f * std_dev * (M_EXPF(-(ew * ew)) - M_EXPF(-(eh * eh)));
            float width = bw + fminf(delta, 0.0f);
            float height = bh - fmaxf(delta, 0.0f);
            float scale = 0.5f * erf7(inv_std_dev * 0.5f * (fmaxf(width, height) - 0.5f * bradius));
            for (int i = 0; i < 256; i++) {
                uint32_t lx = (uint32_t)i & 15u, ly = (uint32_t)i >> 4;
                float gx = (float)(tile_x * 16u + (lx & ~3u)) + (float)(lx & 3u);
                float gy = (float)(tile_y * 16u + ly);
                float x = (m0 * gx + m2 * gy) + tx;
                float y = (m1 * gx + m3 * gy) + ty;
                float y0 = fabsf(y) - (height * 0.5f - r1);
                float y1 = fmaxf(y0, 0.0f);
                float x0 = fabsf(x) - (width * 0.5f - r1);
                float x1 = fmaxf(x0, 0.0f);
                float d_pos = M_POWF(M_POWF(x1, exponent) + M_POWF(y1, exponent), inv_exponent);
                float d_neg = fminf(fmaxf(x0, y0), 0.0f);
                float d = d_pos + d_neg - r1;
                float alpha = scale * (erf7(inv_std_dev * (min_edge + d)) - erf7(inv_std_dev * d));
                rgba[i] = over(rgba[i], rg_scale(rg_scale(blur_rgba, alpha), area[i]));
            }
            cmd_ix += 3u;
            break;
        }
        case CMD_LIN_GRAD: {
            uint32_t index_mode = ptcl[cmd_ix + 1], io = ptcl[cmd_ix + 2];
            uint32_t index = index_mode >> 2, ext = index_mode & 3u;
            float line_x = u2f_bits(info[io]), line_y = u2f_bits(info[io + 1]), line_c = u2f_bits(info[io + 2]);
            for (int i = 0; i < 256; i++) {
                uint32_t lx = (uint32_t)i & 15u, ly = (uint32_t)i >> 4;
                float xyx = (float)(tile_x * 16u + (lx & ~3u)), xyy = (float)(tile_y * 16u + ly);
                float d = (line_x * xyx + line_y * xyy) + line_c;
                float my_d = d + line_x * (float)(lx & 3u);
                int32_t x = f2i_sat(rintf(extend_mode_normalized(my_d, ext) * (float)(GRADIENT_WIDTH - 1)));
                rgba[i] = over(rgba[i], rg_scale(ramp_load(c, x, index), area[i]));
            }
            cmd_ix += 3u;
            break;
        }
        case CMD_RAD_GRAD: {
            uint32_t index_mode = ptcl[cmd_ix + 1], io = ptcl[cmd_ix + 2];
            uint32_t index = index_mode >> 2, ext = index_mode & 3u;
            float m0 = u2f_bits(info[io]), m1 = u2f_bits(info[io + 1]), m2 = u2f_bits(info[io + 2]), m3 = u2f_bits(info[io + 3]);
            float tx = u2f_bits(info[io + 4]), ty = u2f_bits(info[io + 5]);
            float focal_x = u2f_bits(info[io + 6]), radius = u2f_bits(info[io + 7]);
            uint32_t flags_kind = info[io + 8];
            uint32_t flags = flags_kind >> 3, kind = flags_kind & 7u;
            int is_strip = kind == 2u, is_circular = kind == 1u, is_focal_on_circle = kind == 3u;
            int is_swapped = (flags & 1u) != 0u;
            float r1_recip = is_circular ? 0.0f : 1.0f / radius;
            float less_scale = (is_swapped || (1.0f - focal_x) < 0.0f) ? -1.0f : 1.0f;
            float t_sign = signf(1.0f - focal_x);
            for (int i = 0; i < 256; i++) {
                uint32_t lx = (uint32_t)i & 15u, ly = (uint32_t)i >> 4;
                float gx = (float)(tile_x * 16u + (lx & ~3u)) + (float)(lx & 3u);
                float gy = (float)(tile_y * 16u + ly);
                float x = (m0 * gx + m2 * gy) + tx;
                float y = (m1 * gx + m3 * gy) + ty;
                float xx = x * x, yy = y * y;
                float t = 0.0f;
                int is_valid = 1;
                if (is_strip) {
                    float a = radius - yy;
                    t = sqrtf(a) + x;
                    is_valid = a >= 0.0f;
                } else if (is_focal_on_circle) {
                    t = (xx + yy) / x;
                    is_valid = t >= 0.0f && x != 0.0f;
                } else if (radius > 1.0f) {
                    t = sqrtf(xx + yy) - x * r1_recip;
                } else {
                    float a = xx - yy;
                    t = less_scale * sqrtf(a) - x * r1_recip;
                    is_valid = a >= 0.0f && t >= 0.0f;
                }
                if (is_valid) {
                    t = extend_mode_normalized(focal_x + t_sign * t, ext);
                    if (is_swapped) t = 1.0f - t;
                    int32_t rx = f2i_sat(rintf(t * (float)(GRADIENT_WIDTH - 1)));
                    rgba[i] = over(rgba[i], rg_scale(ramp_load(c, rx, index), area[i]));
                }
            }
            cmd_ix += 3u;
            break;
        }
        case CMD_SWEEP_GRAD: {
            uint32_t index_mode = ptcl[cmd_ix + 1], io = ptcl[cmd_ix + 2];
            uint32_t index = index_mode >> 2, ext = index_mode & 3u;
            float m0 = u2f_bits(info[io]), m1 = u2f_bits(info[io + 1]), m2 = u2f_bits(info[io + 2]), m3 = u2f_bits(info[io + 3]);
            float tx = u2f_bits(info[io + 4]), ty = u2f_bits(info[io + 5]);
            float t0 = u2f_bits(info[io + 6]), t1 = u2f_bits(info[io + 7]);
            float scale = 1.0f / (t1 - t0);
            for (int i = 0; i < 256; i++) {
                uint32_t lx = (uint32_t)i & 15u, ly = (uint32_t)i >> 4;
                float gx = (float)(tile_x * 16u + (lx & ~3u)) + (float)(lx & 3u);
                float gy = (float)(tile_y * 16u + ly);
                float x = (m0 * gx + m2 * gy) + tx;
                float y = (m1 * gx + m3 * gy) + ty;
                float xabs = fabsf(x), yabs = fabsf(y);
                float slope = fminf(xabs, yabs) / fmaxf(xabs, yabs);
                float s = slope * slope;
                float phi = slope * (0.15912117063999176025390625f +
                                     s * (-5.185396969318389892578125e-2f +
                                          s * (2.476101927459239959716796875e-2f + s * (-7.0547382347285747528076171875e-3f))));
                if (xabs < yabs) phi = 1.0f / 4.0f - phi;
                if (x < 0.0f) phi = 1.0f / 2.0f - phi;
                if (y < 0.0f) phi = 1.0f - phi;
                if (phi != phi) phi = 0.0f;
                phi = (phi - t0) * scale;
                float t = extend_mode_normalized(phi, ext);
                int32_t rx = f2i_sat(rintf(t * (float)(GRADIENT_WIDTH - 1)));
                rgba[i] = over(rgba[i], rg_scale(ramp_load(c, rx, index), area[i]));
            }
            cmd_ix += 3u;
            break;
        }
        case CMD_IMAGE: {
            uint32_t io = ptcl[cmd_ix + 1];
            float m0 = u2f_bits(info[io]), m1 = u2f_bits(info[io + 1]), m2 = u2f_bits(info[io + 2]), m3 = u2f_bits(info[io + 3]);
            float tx = u2f_bits(info[io + 4]), ty = u2f_bits(info[io + 5]);
            uint32_t xy = info[io + 6], wh = info[io + 7], sa = info[io + 8];
            float alpha = (float)(sa & 0xFFu) / 255.0f;
            uint32_t format = sa >> 15, alpha_type = (sa >> 14) & 1u, quality = (sa >> 12) & 3u;
            uint32_t x_ext = (sa >> 10) & 3u, y_ext = (sa >> 8) & 3u;
            float ox = (float)(xy >> 16), oy = (float)(xy & 0xffffu);
            float ew = (float)(wh >> 16), eh = (float)(wh & 0xffffu);
            float mx = ox + ew - 1.0f, my = oy + eh - 1.0f;
            for (int i = 0; i < 256; i++) {
                if (area[i] == 0.0f) continue;
                uint32_t lx = (uint32_t)i & 15u, ly = (uint32_t)i >> 4;
                float gx = ((float)(tile_x * 16u + (lx & ~3u)) + (float)(lx & 3u)) + 0.5f;
                float gy = (float)(tile_y * 16u + ly) + 0.5f;
                float u = (m0 * gx + m2 * gy) + tx;
                float v = (m1 * gx + m3 * gy) + ty;
                u = extend_mode(u, x_ext, ew);
                v = extend_mode(v, y_ext, eh);
                rgba_t fg;
                if (quality == 0u) {
                    u = u + ox; v = v + oy;
                    fg = maybe_premul(atlas_load(c, clampf(u, ox, mx), clampf(v, oy, my)), alpha_type);
                } else if (quality == 2u) {
                    u = u + ox; v = v + oy;
                    fg = bicubic_sample(c, u, v, ox, oy, mx, my, alpha_type);
                } else {
                    u = (u + ox) - 0.5f; v = (v + oy) - 0.5f;
                    float uc = clampf(u, ox, mx), vc = clampf(v, oy, my);
                    float qx0 = floorf(uc), qy0 = floorf(vc), qx1 = ceilf(uc), qy1 = ceilf(vc);
                    float fu = u - floorf(u), fv = v - floorf(v);
                    rgba_t a = maybe_premul(atlas_load(c, qx0, qy0), alpha_type);
                    rgba_t b = maybe_premul(atlas_load(c, qx0, qy1), alpha_type);
                    rgba_t cc = maybe_premul(atlas_load(c, qx1, qy0), alpha_type);
                    rgba_t d = maybe_premul(atlas_load(c, qx1, qy1), alpha_type);
                    rgba_t ab = RG(mixf(a.r, b.r, fv), mixf(a.g, b.g, fv), mixf(a.b, b.b, fv), mixf(a.a, b.a, fv));
                    rgba_t cd = RG(mixf(cc.r, d.r, fv), mixf(cc.g, d.g, fv), mixf(cc.b, d.b, fv), mixf(cc.a, d.a, fv));
                    fg = RG(mixf(ab.r, cd.r, fu), mixf(ab.g, cd.g, fu), mixf(ab.b, cd.b, fu), mixf(ab.a, cd.a, fu));
                }
                rgba_t fg_i = pixel_format(rg_scale(rg_scale(fg, area[i]), alpha), format);
                rgba[i] = over(rgba[i], fg_i);
            }
            cmd_ix += 2u;
            break;
        }
        default:
            cmd_ix += 1u; /* unknown command: WGSL `default: {}` would spin; skip a word */
            break;
        }
    }
done:
    free(stack);
    for (int i = 0; i < 256; i++) {
        uint32_t px = tile_x * 16u + ((uint32_t)i & 15u), py = tile_y * 16u + ((uint32_t)i >> 4);
        if (px < cfg->target_width && py < cfg->target_height) {
            rgba_t fg = rgba[i];
            float a_inv = 1.0f / fmaxf(fg.a, 1e-6f);
            uint8_t *o = out + ((size_t)py * cfg->target_width + px) * 4u;
            o[0] = (uint8_t)unorm8(fg.r * a_inv);
            o[1] = (uint8_t)unorm8(fg.g * a_inv);
            o[2] = (uint8_t)unorm8(fg.b * a_inv);
            o[3] = (uint8_t)unorm8(fg.a);
        }
    }
}

/* mask LUTs: vello_encoding/src/mask.rs:10-98 (f64 maths, as the reference) */
static uint32_t one_mask(double slope, double translation, int is_pos, const uint8_t *pattern, int n) {
    if (is_pos) translation = 1. - translation;
    uint32_t result = 0;
    for (int i = 0; i < n; i++) {
        double y = (i + 0.5) * (1.0 / n);
        double x = (pattern[i] + 0.5) * (1.0 / n);
        if (!is_pos) y = 1. - y;
        if ((x - (1.0 - translation)) * (1. - slope) - (y - translation) * slope >= 0.) result |= 1u << i;
    }
    return result;
}
static void make_mask_luts(uint32_t *lut8 /*256*/, uint32_t *lut16 /*2048*/) {
    static const uint8_t P8[8] = {0, 5, 3, 7, 1, 4, 6, 2};
    static const uint8_t P16[16] = {1, 8, 4, 11, 15, 7, 3, 12, 0, 9, 5, 13, 2, 10, 6, 14};
    memset(lut8, 0, 256 * 4);
    memset(lut16, 0, 2048 * 4);
    for (int i = 0; i < 32 * 32; i++) {
        int u = i % 32, v = i / 32;
        int is_pos = v >= 16;
        double y = ((v % 16) + 0.5) * (1.0 / 16);
        double x = (u + 0.5) * (1.0 / 32);
        lut8[i / 4] |= one_mask(y, x, is_pos, P8, 8) << ((i % 4) * 8);
    }
    for (int i = 0; i < 64 * 64; i++) {
        int u = i % 64, v = i / 64;
        int is_pos = v >= 32;
        double y = ((v % 32) + 0.5) * (1.0 / 32);
        double x = (u + 0.5) * (1.0 / 64);
        lut16[i / 2] |= one_mask(y, x, is_pos, P16, 16) << ((i % 2) * 16);
    }
}

typedef struct {
    const FineIn *in;
    const uint32_t *lut;
    uint8_t *out;
    uint32_t ty0, ty1, wt;
    int tid, nthreads;
} Job;
static void *fine_worker(void *arg) {
    Job *j = arg;
    for (uint32_t ty = j->ty0 + (uint32_t)j->tid; ty < j->ty1; ty += (uint32_t)j->nthreads)
        for (uint32_t tx = 0; tx < j->wt; tx++) fine_tile(j->in, j->lut, tx, ty, j->out);
    return NULL;
}

int vbo_fine(vbo_ctx *c, uint8_t *out) {
    static uint32_t lut8[256], lut16[2048];
    static int luts_ready = 0;
    if (!luts_ready) { make_mask_luts(lut8, lut16); luts_ready = 1; }
    uint32_t *spill = vec_resize(&c->blend_spill, c->bump.blend ? c->bump.blend : 1);
    int error = 0;
    FineIn in = {c, c->ptcl.p, c->info_bin_data.p, c->segments.p, spill,
                 c->ptcl.n, c->info_bin_data.n, c->segments.n, c->bump.blend, &error};
    const uint32_t *lut = c->params.aa == 2u ? lut16 : lut8;
    int nt = c->threads;
    if (nt <= 1) {
        Job j = {&in, lut, out, c->win_ty0, c->win_ty1, c->cfg.width_in_tiles, 0, 1};
        fine_worker(&j);
        return error ? -3 : 0;
    }
    enum { MAX_THREADS = 1024 };
    static pthread_t th[MAX_THREADS]; /* vbo_fine is not re-entrant (one context renders at a time) */
    static Job jobs[MAX_THREADS];
    if (nt > MAX_THREADS) nt = MAX_THREADS;
    if ((uint32_t)nt > c->win_ty1 - c->win_ty0) nt = (int)(c->win_ty1 - c->win_ty0); /* a thread per tile row at most */
    if (nt < 1) nt = 1;
    for (int t = 0; t < nt; t++) {
        Job j = {&in, lut, out, c->win_ty0, c->win_ty1, c->cfg.width_in_tiles, t, nt};
        jobs[t] = j;
        pthread_create(&th[t], NULL, fine_worker, &jobs[t]);
    }
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    return error ? -3 : 0;
}
