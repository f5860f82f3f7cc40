/* vbo_stages.c -- CPU ORACLE, stages pathtag .. path_tiling.  TEST INFRASTRUCTURE ONLY (see vbo.h).
 *
 * Serial restatement of vello_shaders/src/cpu/ (the .rs twins; the code `RendererOptions::use_cpu` runs),
 * with the WGSL's arithmetic where the two differ (listed in oracle/README.md). Buffers grow on
 * demand, so there is no bump overflow in the oracle.
 */
#include "vbo_internal.h"

#include <stdio.h>

/* ------------------------------------------------------------------------------------------
 * 1. path tag monoid: shared/pathtag.wgsl:58-71, vello_encoding/src/path.rs:334-364
 * ---------------------------------------------------------------------------------------- */
static TagMonoid reduce_tag(uint32_t tag_word) {
    TagMonoid c;
    uint32_t point_count = tag_word & 0x3030303u;
    c.pathseg_ix = (uint32_t)__builtin_popcount((point_count * 7u) & 0x4040404u);
    c.trans_ix = (uint32_t)__builtin_popcount(tag_word & (0x20u * 0x1010101u));
    uint32_t n_points = point_count + ((tag_word >> 2) & 0x1010101u);
    uint32_t a = n_points + (n_points & (((tag_word >> 3) & 0x1010101u) * 15u));
    a += a >> 8;
    a += a >> 16;
    c.pathseg_offset = a & 0xffu;
    c.path_ix = (uint32_t)__builtin_popcount(tag_word & (0x10u * 0x1010101u));
    c.style_ix = (uint32_t)__builtin_popcount(tag_word & (0x40u * 0x1010101u)) * 2u;
    return c;
}
static TagMonoid tm_combine(TagMonoid a, TagMonoid b) {
    TagMonoid c = {a.trans_ix + b.trans_ix, a.pathseg_ix + b.pathseg_ix, a.pathseg_offset + b.pathseg_offset,
                   a.style_ix + b.style_ix, a.path_ix + b.path_ix};
    return c;
}

static inline uint32_t scene_rd(const vbo_ctx *c, uint32_t ix) { return ix < c->scene_words ? c->scene[ix] : 0u; }

/* cpu/pathtag_reduce.rs + cpu/pathtag_scan.rs collapsed into one exclusive scan over tag words */
static void stage_pathtag(vbo_ctx *c) {
    uint32_t n_words = (c->cfg.layout.path_data_base - c->cfg.layout.path_tag_base);
    TagMonoid *tm = vec_resize(&c->tag_monoids, n_words);
    TagMonoid m = {0, 0, 0, 0, 0};
    for (uint32_t i = 0; i < n_words; i++) {
        tm[i] = m;
        m = tm_combine(m, reduce_tag(scene_rd(c, c->cfg.layout.path_tag_base + i)));
    }
}

/* ------------------------------------------------------------------------------------------
 * 2. flatten: cpu/flatten.rs, cpu/euler.rs, shader/flatten.wgsl
 * ---------------------------------------------------------------------------------------- */
typedef struct { float m[4]; float t[2]; } Xform; /* column-major 2x2 + translation */

static Xform xf_identity(void) { Xform t = {{1.f, 0.f, 0.f, 1.f}, {0.f, 0.f}}; return t; }
static Xform xf_read(const vbo_ctx *c, uint32_t base, uint32_t ix) {
    Xform t;
    uint32_t b = base + ix * 6u;
    for (int i = 0; i < 4; i++) t.m[i] = u2f_bits(scene_rd(c, b + i));
    t.t[0] = u2f_bits(scene_rd(c, b + 4));
    t.t[1] = u2f_bits(scene_rd(c, b + 5));
    return t;
}
/* flatten.wgsl:668-672: explicit fma */
static v2 xf_apply_fma(const Xform *t, v2 p) {
    return V2(fmaf(t->m[0], p.x, fmaf(t->m[2], p.y, t->t[0])), fmaf(t->m[1], p.x, fmaf(t->m[3], p.y, t->t[1])));
}

typedef struct {
    vbo_ctx *c;
    float bbox[4];
} FlatCtx;

static void write_line(FlatCtx *f, uint32_t path_ix, v2 p0, v2 p1) { /* flatten.wgsl:770-775 */
    f->bbox[0] = fminf(f->bbox[0], fminf(p0.x, p1.x));
    f->bbox[1] = fminf(f->bbox[1], fminf(p0.y, p1.y));
    f->bbox[2] = fmaxf(f->bbox[2], fmaxf(p0.x, p1.x));
    f->bbox[3] = fmaxf(f->bbox[3], fmaxf(p0.y, p1.y));
    Vec *v = &f->c->lines;
    LineSoup *l = vec_reserve(v, v->n + 1);
    l[v->n].path_ix = path_ix;
    l[v->n]._pad = 0;
    l[v->n].p0[0] = p0.x; l[v->n].p0[1] = p0.y;
    l[v->n].p1[0] = p1.x; l[v->n].p1[1] = p1.y;
    v->n++;
}
static void output_line_xf(FlatCtx *f, uint32_t path_ix, v2 p0, v2 p1, const Xform *t) {
    write_line(f, path_ix, xf_apply_fma(t, p0), xf_apply_fma(t, p1));
}

#define DERIV_THRESH 1e-6f
#define DERIV_THRESH_SQUARED (DERIV_THRESH * DERIV_THRESH)
#define DERIV_EPS 1e-6f
#define SUBDIV_LIMIT (1.0f / 65536.0f)
#define K1_THRESH 1e-3f
#define DIST_THRESH 1e-3f
#define TANGENT_THRESH 1e-6f

typedef struct { float th0, th1, chord_len, err; } CubicParams;
typedef struct { float th0, k0, k1, ch; } EulerParams;

/* flatten.wgsl:94-133 (association of the error terms follows the WGSL, not euler.rs:133) */
static CubicParams cubic_from_points_derivs(v2 p0, v2 p1, v2 q0, v2 q1, float dt) {
    CubicParams r;
    v2 chord = v2sub(p1, p0);
    float chord_squared = v2dot(chord, chord);
    float chord_len = sqrtf(chord_squared);
    if (chord_squared < DERIV_THRESH_SQUARED) {
        float chord_err = sqrtf((9.f / 32.0f) * (v2dot(q0, q0) + v2dot(q1, q1))) * dt;
        r.th0 = 0.f; r.th1 = 0.f; r.chord_len = DERIV_THRESH; r.err = chord_err;
        return r;
    }
    float scale = dt / chord_squared;
    v2 h0 = V2(q0.x * chord.x + q0.y * chord.y, q0.y * chord.x - q0.x * chord.y);
    float th0 = M_ATAN2F(h0.y, h0.x);
    float d0 = v2len(h0) * scale;
    v2 h1 = V2(q1.x * chord.x + q1.y * chord.y, q1.x * chord.y - q1.y * chord.x);
    float th1 = M_ATAN2F(h1.y, h1.x);
    float d1 = v2len(h1) * scale;
    float cth0 = M_COSF(th0);
    float cth1 = M_COSF(th1);
    float err = 2.0f;
    if (cth0 * cth1 >= 0.0f) {
        float e0 = (2.f / 3.f) / fmaxf(1.0f + cth0, 1e-9f);
        float e1 = (2.f / 3.f) / fmaxf(1.0f + cth1, 1e-9f);
        float s0 = M_SINF(th0);
        float s1 = M_SINF(th1);
        float s01 = cth0 * s1 + cth1 * s0;
        float amin = 0.15f * (2.f * e0 * s0 + 2.f * e1 * s1 - e0 * e1 * s01);
        float a = 0.15f * (2.f * d0 * s0 + 2.f * d1 * s1 - d0 * d1 * s01);
        float aerr = fabsf(a - amin);
        float symm = fabsf(th0 + th1);
        float asymm = fabsf(th0 - th1);
        float dist = v2len(V2(d0 - e0, d1 - e1));
        float symm2 = symm * symm;
        float ctr = (4.625e-6f * symm * symm2 + 7.5e-3f * asymm) * symm2;
        float halo = (5e-3f * symm + 7e-2f * asymm) * dist;
        err = ctr + 1.55f * aerr + halo;
    }
    err *= chord_len;
    r.th0 = th0; r.th1 = th1; r.chord_len = chord_len; r.err = err;
    return r;
}

/* flatten.wgsl:135-161, euler.rs:166-190 */
static EulerParams es_params_from_angles(float th0, float th1) {
    float k0 = th0 + th1;
    float dth = th1 - th0;
    float d2 = dth * dth;
    float k2 = k0 * k0;
    float a = 6.0f;
    a -= d2 * (1.f / 70.f);
    a -= (d2 * d2) * (1.f / 10780.f);
    a += (d2 * d2 * d2) * 2.769178184818219e-07f;
    float b = -0.1f + d2 * (1.f / 4200.f) + d2 * d2 * 1.6959677820260655e-05f;
    float cc = -1.f / 1400.f + d2 * 6.84915970574303e-05f - k2 * 7.936475029053326e-06f;
    a += (b + cc * k2) * k2;
    float k1 = dth * a;
    float ch = 1.0f;
    ch -= d2 * (1.f / 40.f);
    ch += (d2 * d2) * 0.00034226190482569864f;
    ch -= (d2 * d2 * d2) * 1.9349474568904524e-06f;
    float b_ = -1.f / 24.f + d2 * 0.0024702380951963226f - d2 * d2 * 3.7297408997537985e-05f;
    float c_ = 1.f / 1920.f - d2 * 4.87350869747975e-05f - k2 * 3.1001936068463107e-06f;
    ch += (b_ + c_ * k2) * k2;
    EulerParams r = {th0, k0, k1, ch};
    return r;
}
static float es_eval_th(const EulerParams *p, float t) { return (p->k0 + 0.5f * p->k1 * (t - 1.0f)) * t - p->th0; }

/* flatten.wgsl:168-202, euler.rs:260-294 */
static v2 integ_euler_10(float k0, float k1) {
    float t1_1 = k0;
    float t1_2 = 0.5f * k1;
    float t2_2 = t1_1 * t1_1;
    float t2_3 = 2.f * (t1_1 * t1_2);
    float t2_4 = t1_2 * t1_2;
    float t3_4 = t2_2 * t1_2 + t2_3 * t1_1;
    float t3_6 = t2_4 * t1_2;
    float t4_4 = t2_2 * t2_2;
    float t4_5 = 2.f * (t2_2 * t2_3);
    float t4_6 = 2.f * (t2_2 * t2_4) + t2_3 * t2_3;
    float t4_7 = 2.f * (t2_3 * t2_4);
    float t4_8 = t2_4 * t2_4;
    float t5_6 = t4_4 * t1_2 + t4_5 * t1_1;
    float t5_8 = t4_6 * t1_2 + t4_7 * t1_1;
    float t6_6 = t4_4 * t2_2;
    float t6_7 = t4_4 * t2_3 + t4_5 * t2_2;
    float t6_8 = t4_4 * t2_4 + t4_5 * t2_3 + t4_6 * t2_2;
    float t7_8 = t6_6 * t1_2 + t6_7 * t1_1;
    float t8_8 = t6_6 * t2_2;
    float u = 1.f;
    u -= (1.f / 24.f) * t2_2 + (1.f / 160.f) * t2_4;
    u += (1.f / 1920.f) * t4_4 + (1.f / 10752.f) * t4_6 + (1.f / 55296.f) * t4_8;
    u -= (1.f / 322560.f) * t6_6 + (1.f / 1658880.f) * t6_8;
    u += (1.f / 92897280.f) * t8_8;
    float v = (1.f / 12.f) * t1_2;
    v -= (1.f / 480.f) * t3_4 + (1.f / 2688.f) * t3_6;
    v += (1.f / 53760.f) * t5_6 + (1.f / 276480.f) * t5_8;
    v -= (1.f / 11612160.f) * t7_8;
    return V2(u, v);
}
/* flatten.wgsl:204-215 */
static v2 es_params_eval(const EulerParams *p, float t) {
    float thm = es_eval_th(p, t * 0.5f);
    float k0 = p->k0, k1 = p->k1;
    v2 uv = integ_euler_10((k0 + k1 * (0.5f * t - 0.5f)) * t, k1 * t * t);
    float scale = t / p->ch;
    float s = scale * M_SINF(thm);
    float c = scale * M_COSF(thm);
    return V2(uv.x * c - uv.y * s, -uv.y * c - uv.x * s);
}
static v2 es_params_eval_with_offset(const EulerParams *p, float t, float offset) {
    float th = es_eval_th(p, t);
    v2 v = V2(offset * M_SINF(th), offset * M_COSF(th));
    return v2add(es_params_eval(p, t), v);
}
static v2 es_seg_eval_with_offset(v2 p0, v2 p1, const EulerParams *p, float t, float normalized_offset) {
    v2 chord = v2sub(p1, p0);
    v2 xy = es_params_eval_with_offset(p, t, normalized_offset);
    return V2(p0.x + (chord.x * xy.x - chord.y * xy.y), p0.y + (chord.x * xy.y + chord.y * xy.x));
}
static float pow_1_5_signed(float x) { return x * sqrtf(fabsf(x)); }

#define BREAK1 0.8f
#define BREAK2 1.25f
#define BREAK3 2.1f
#define SIN_SCALE 1.0976991822760038f
#define QUAD_A1 0.6406f
#define QUAD_B1 (-0.81f)
#define QUAD_C1 0.9148117935952064f
#define QUAD_A2 0.5f
#define QUAD_B2 (-0.156f)
#define QUAD_C2 0.16145779359520596f
#define FRAC_PI_4 0.7853981633974483f
#define CBRT_9_8 1.040041911525952f

/* flatten.wgsl:246-259 */
static float espc_int_approx(float x) {
    float y = fabsf(x);
    float a;
    if (y < BREAK1) {
        a = M_SINF(SIN_SCALE * y) * (1.0f / SIN_SCALE);
    } else if (y < BREAK2) {
        a = (sqrtf(8.0f) / 3.0f) * pow_1_5_signed(y - 1.0f) + FRAC_PI_4;
    } else {
        float qa = y < BREAK3 ? QUAD_A1 : QUAD_A2;
        float qb = y < BREAK3 ? QUAD_B1 : QUAD_B2;
        float qc = y < BREAK3 ? QUAD_C1 : QUAD_C2;
        a = (qa * y + qb) * y + qc;
    }
    return a * signf(x);
}
/* flatten.wgsl:261-275 */
static float espc_int_inv_approx(float x) {
    float y = fabsf(x);
    float a;
    if (y < 0.7010707591262915f) {
        a = M_ASINF(y * SIN_SCALE) * (1.0f / SIN_SCALE);
    } else if (y < 0.903249293595206f) {
        float b = y - FRAC_PI_4;
        float u = M_POW23(fabsf(b)) * signf(b);
        a = u * CBRT_9_8 + 1.0f;
    } else {
        const float W1 = 0.5f * QUAD_B1 / QUAD_A1, V1 = 1.0f / QUAD_A1, U1 = W1 * W1 - QUAD_C1 / QUAD_A1;
        const float W2 = 0.5f * QUAD_B2 / QUAD_A2, V2_ = 1.0f / QUAD_A2, U2 = W2 * W2 - QUAD_C2 / QUAD_A2;
        int first = y < 2.038857793595206f;
        float u = first ? U1 : U2, v = first ? V1 : V2_, w = first ? W1 : W2;
        a = sqrtf(u + v * y) - w;
    }
    return a * signf(x);
}

typedef struct { v2 p, q; } PointDeriv;
static PointDeriv eval_cubic_and_deriv(v2 p0, v2 p1, v2 p2, v2 p3, float t) { /* flatten.wgsl:282-290 */
    float m = 1.0f - t;
    float mm = m * m;
    float mt = m * t;
    float tt = t * t;
    PointDeriv r;
    /* p0 * (mm*m) + (p1*(3mm) + p2*(3mt) + p3*tt) * t */
    float a = mm * m, b = 3.0f * mm, c = 3.0f * mt;
    r.p.x = p0.x * a + ((p1.x * b + p2.x * c) + p3.x * tt) * t;
    r.p.y = p0.y * a + ((p1.y * b + p2.y * c) + p3.y * tt) * t;
    float d = 2.0f * mt;
    r.q.x = ((p1.x - p0.x) * mm + (p2.x - p1.x) * d) + (p3.x - p2.x) * tt;
    r.q.y = ((p1.y - p0.y) * mm + (p2.y - p1.y) * d) + (p3.y - p2.y) * tt;
    return r;
}
static v2 cubic_start_tangent(v2 p0, v2 p1, v2 p2, v2 p3) { /* flatten.wgsl:292-298 (EPS 1e-12) */
    const float EPS = 1e-12f;
    v2 d01 = v2sub(p1, p0), d02 = v2sub(p2, p0), d03 = v2sub(p3, p0);
    if (v2dot(d01, d01) > EPS) return d01;
    if (v2dot(d02, d02) > EPS) return d02;
    return d03;
}
static v2 cubic_end_tangent(v2 p0, v2 p1, v2 p2, v2 p3) { /* flatten.wgsl:300-306 */
    const float EPS = 1e-12f;
    v2 d23 = v2sub(p3, p2), d13 = v2sub(p3, p1), d03 = v2sub(p3, p0);
    if (v2dot(d23, d23) > EPS) return d23;
    if (v2dot(d13, d13) > EPS) return d13;
    return d03;
}

typedef struct { v2 p0, p1, p2, p3; } CubicPoints;

/* flatten.wgsl:326-481 */
static void flatten_euler(FlatCtx *f, const CubicPoints *cubic, uint32_t path_ix, const Xform *local_to_device,
                          float offset, v2 start_p, v2 end_p) {
    v2 p0, p1, p2, p3;
    float scale;
    Xform transform;
    v2 t_start = start_p, t_end = end_p;
    if (offset == 0.f) {
        p0 = xf_apply_fma(local_to_device, cubic->p0);
        p1 = xf_apply_fma(local_to_device, cubic->p1);
        p2 = xf_apply_fma(local_to_device, cubic->p2);
        p3 = xf_apply_fma(local_to_device, cubic->p3);
        scale = 1.f;
        transform = xf_identity();
        t_start = p0;
        t_end = p3;
    } else {
        p0 = cubic->p0; p1 = cubic->p1; p2 = cubic->p2; p3 = cubic->p3;
        transform = *local_to_device;
        const float *m = transform.m;
        scale = 0.5f * (v2len(V2(m[0] + m[3], m[1] - m[2])) + v2len(V2(m[0] - m[3], m[1] + m[2])));
    }
    if (v2eq(p0, p1) && v2eq(p0, p2) && v2eq(p0, p3)) return;

    const float tol = 0.25f;
    uint32_t t0_u = 0u;
    float dt = 1.0f;
    v2 last_p = p0;
    v2 last_q = v2sub(p1, p0);
    if (v2dot(last_q, last_q) < DERIV_THRESH_SQUARED) last_q = eval_cubic_and_deriv(p0, p1, p2, p3, DERIV_EPS).q;
    float last_t = 0.0f;
    v2 lp0 = t_start;
    for (;;) {
        float t0 = (float)t0_u * dt;
        if (t0 == 1.0f) break;
        float t1 = t0 + dt;
        v2 this_p0 = last_p;
        v2 this_q0 = last_q;
        PointDeriv this_pq1 = eval_cubic_and_deriv(p0, p1, p2, p3, t1);
        if (v2dot(this_pq1.q, this_pq1.q) < DERIV_THRESH_SQUARED) {
            PointDeriv new_pq1 = eval_cubic_and_deriv(p0, p1, p2, p3, t1 - DERIV_EPS);
            this_pq1.q = new_pq1.q;
            if (t1 < 1.0f) {
                this_pq1.p = new_pq1.p;
                t1 = t1 - DERIV_EPS;
            }
        }
        float actual_dt = t1 - last_t;
        CubicParams cp = cubic_from_points_derivs(this_p0, this_pq1.p, this_q0, this_pq1.q, actual_dt);
        if (cp.err * scale <= tol || dt <= SUBDIV_LIMIT) {
            EulerParams ep = es_params_from_angles(cp.th0, cp.th1);
            v2 es_p0 = this_p0, es_p1 = this_pq1.p;
            float k0 = ep.k0 - 0.5f * ep.k1;
            float k1 = ep.k1;
            float normalized_offset = offset / cp.chord_len;
            float dist_scaled = normalized_offset * ep.ch;
            float scale_multiplier = sqrtf(0.125f * scale * cp.chord_len / (ep.ch * tol));
            float a = 0.0f, b = 0.0f, integral = 0.0f, int0 = 0.0f, n_frac;
            int robust = 0; /* 0 normal, 1 low k1, 2 low dist */
            if (fabsf(k1) < K1_THRESH) {
                float k = ep.k0;
                n_frac = sqrtf(fabsf(k * (k * dist_scaled + 1.0f)));
                robust = 1;
            } else if (fabsf(dist_scaled) < DIST_THRESH) {
                a = k1;
                b = k0;
                int0 = pow_1_5_signed(b);
                float int1 = pow_1_5_signed(a + b);
                integral = int1 - int0;
                n_frac = (2.f / 3.f) * integral / a;
                robust = 2;
            } else {
                a = -2.0f * dist_scaled * k1;
                b = -1.0f - 2.0f * dist_scaled * k0;
                int0 = espc_int_approx(b);
                float int1 = espc_int_approx(a + b);
                integral = int1 - int0;
                float k_peak = k0 - k1 * b / a;
                float integrand_peak = sqrtf(fabsf(k_peak * (k_peak * dist_scaled + 1.0f)));
                n_frac = integral * integrand_peak / a;
            }
            float n = clampf(ceilf(n_frac * scale_multiplier), 1.0f, 100.0f);
            uint32_t n_u = f2u_sat(n);
            for (uint32_t i = 0u; i < n_u; i++) {
                v2 lp1;
                if (i + 1u == n_u && t1 == 1.0f) {
                    lp1 = t_end;
                } else {
                    float t = (float)(i + 1u) / n;
                    float s = t;
                    if (robust != 1) {
                        float u = integral * t + int0;
                        float inv;
                        if (robust == 2) {
                            inv = M_POW23(fabsf(u)) * signf(u);
                        } else {
                            inv = espc_int_inv_approx(u);
                        }
                        s = (inv - b) / a;
                    }
                    lp1 = es_seg_eval_with_offset(es_p0, es_p1, &ep, s, normalized_offset);
                }
                v2 l0 = offset >= 0.f ? lp0 : lp1;
                v2 l1 = offset >= 0.f ? lp1 : lp0;
                output_line_xf(f, path_ix, l0, l1, &transform);
                lp0 = lp1;
            }
            last_p = this_pq1.p;
            last_q = this_pq1.q;
            last_t = t1;
            t0_u += 1u;
            uint32_t shift = (uint32_t)__builtin_ctz(t0_u);
            t0_u >>= shift;
            dt *= (float)(1u << shift);
        } else {
            t0_u = t0_u * 2u;
            dt *= 0.5f;
        }
    }
}

/* flatten.wgsl:494-519 */
static void flatten_arc(FlatCtx *f, uint32_t path_ix, v2 begin, v2 end, v2 center, float angle, const Xform *t) {
    v2 p0 = xf_apply_fma(t, begin);
    v2 r = v2sub(begin, center);
    const float MIN_THETA = 0.0001f;
    const float tol = 0.25f;
    float radius = fmaxf(tol, v2len(v2sub(p0, xf_apply_fma(t, center))));
    float theta = fmaxf(MIN_THETA, 2.f * M_ACOSF(1.f - tol / radius));
    uint32_t n_lines = f2u_sat(ceilf(angle / theta));
    if (n_lines < 1u) n_lines = 1u;
    float c = M_COSF(theta);
    float s = M_SINF(theta);
    /* rot = mat2x2(c, -s, s, c) (columns); rot * r = (c, -s) * r.x + (s, c) * r.y */
    for (uint32_t i = 0u; i + 1u < n_lines; i++) {
        r = V2(c * r.x + s * r.y, -s * r.x + c * r.y);
        v2 p1 = xf_apply_fma(t, v2add(center, r));
        write_line(f, path_ix, p0, p1);
        p0 = p1;
    }
    v2 p1 = xf_apply_fma(t, end);
    write_line(f, path_ix, p0, p1);
}

#define STYLE_FLAGS_STYLE 0x80000000u
#define STYLE_FLAGS_FILL 0x40000000u
#define STYLE_MITER_LIMIT_MASK 0xFFFFu
#define STYLE_FLAGS_START_CAP_MASK 0x0C000000u
#define STYLE_FLAGS_END_CAP_MASK 0x03000000u
#define STYLE_FLAGS_CAP_SQUARE 0x01000000u
#define STYLE_FLAGS_CAP_ROUND 0x02000000u
#define STYLE_FLAGS_JOIN_MASK 0x30000000u
#define STYLE_FLAGS_JOIN_BEVEL 0u
#define STYLE_FLAGS_JOIN_MITER 0x10000000u
#define STYLE_FLAGS_JOIN_ROUND 0x20000000u

/* flatten.wgsl:521-545. The WGSL allocates line slots up front and writes the (square cap)
 * closing line into the FIRST slot; the serial CPU twin (flatten.rs:362-390) appends it last.
 * Slot order inside one tag's allocation follows the WGSL here. */
static void draw_cap(FlatCtx *f, uint32_t path_ix, uint32_t cap_style, v2 point, v2 cap0, v2 cap1, v2 offset_tangent,
                     const Xform *t) {
    if (cap_style == STYLE_FLAGS_CAP_ROUND) {
        flatten_arc(f, path_ix, cap0, cap1, point, 3.1415927f, t);
        return;
    }
    v2 start = cap0, end = cap1;
    if (cap_style == STYLE_FLAGS_CAP_SQUARE) {
        v2 v = offset_tangent;
        v2 p0 = v2add(start, v);
        v2 p1 = v2add(end, v);
        output_line_xf(f, path_ix, p0, p1, t); /* slot line_ix */
        output_line_xf(f, path_ix, start, p0, t); /* slot line_ix + 1 */
        output_line_xf(f, path_ix, p1, end, t);   /* slot line_ix + 2 */
        return;
    }
    output_line_xf(f, path_ix, start, end, t);
}

static float f16_bits_to_f32(uint32_t h) { /* unpack2x16float(x)[0]; math.rs:133-154 */
    uint32_t bits = h & 0xffffu;
    uint32_t o = (bits & 0x7fffu) << 13;
    uint32_t exp = 0x0f800000u & o; /* 0x7c00 << 13 */
    o += (127u - 15u) << 23;
    if (exp == 0x0f800000u) {
        o += (128u - 16u) << 23;
    } else if (exp == 0u) {
        o += 1u << 23;
        o = f2u_bits(u2f_bits(o) - u2f_bits(113u << 23));
    }
    return u2f_bits(o | ((bits & 0x8000u) << 16));
}

/* flatten.wgsl:547-631 */
static void draw_join(FlatCtx *f, uint32_t path_ix, uint32_t style_flags, v2 p0, v2 tan_prev, v2 tan_next, v2 n_prev,
                      v2 n_next, const Xform *t) {
    v2 front0 = v2add(p0, n_prev);
    v2 front1 = v2add(p0, n_next);
    v2 back0 = v2sub(p0, n_next);
    v2 back1 = v2sub(p0, n_prev);
    float cr = tan_prev.x * tan_next.y - tan_prev.y * tan_next.x;
    float d = v2dot(tan_prev, tan_next);
    switch (style_flags & STYLE_FLAGS_JOIN_MASK) {
    case STYLE_FLAGS_JOIN_BEVEL:
        output_line_xf(f, path_ix, front0, front1, t);
        output_line_xf(f, path_ix, back0, back1, t);
        break;
    case STYLE_FLAGS_JOIN_MITER: {
        float hyp = v2len(V2(cr, d));
        float miter_limit = f16_bits_to_f32(style_flags & STYLE_MITER_LIMIT_MASK);
        if (2.f * hyp < (hyp + d) * miter_limit * miter_limit && fabsf(cr) > TANGENT_THRESH * TANGENT_THRESH) {
            int is_backside = cr > 0.f;
            v2 fp_last = is_backside ? back1 : front0;
            v2 fp_this = is_backside ? back0 : front1;
            v2 p = is_backside ? back0 : front0;
            v2 v = v2sub(fp_this, fp_last);
            float h = (tan_prev.x * v.y - tan_prev.y * v.x) / cr;
            v2 miter_pt = v2sub(fp_this, v2scale(tan_next, h));
            output_line_xf(f, path_ix, p, miter_pt, t);
            if (is_backside) back0 = miter_pt; else front0 = miter_pt;
        }
        output_line_xf(f, path_ix, front0, front1, t);
        output_line_xf(f, path_ix, back0, back1, t);
        break;
    }
    case STYLE_FLAGS_JOIN_ROUND: {
        v2 arc0, arc1, other0, other1;
        if (cr > 0.f) { arc0 = back0; arc1 = back1; other0 = front0; other1 = front1; }
        else { arc0 = front0; arc1 = front1; other0 = back0; other1 = back1; }
        flatten_arc(f, path_ix, arc0, arc1, p0, fabsf(M_ATAN2F(cr, d)), t);
        output_line_xf(f, path_ix, other0, other1, t);
        break;
    }
    default: break;
    }
}

typedef struct { uint32_t tag_byte; TagMonoid monoid; } PathTagData;

static PathTagData compute_tag_monoid(const vbo_ctx *c, uint32_t ix) { /* flatten.wgsl:683-699 */
    uint32_t n_words = (uint32_t)c->tag_monoids.n;
    uint32_t tag_word = scene_rd(c, c->cfg.layout.path_tag_base + (ix >> 2));
    uint32_t shift = (ix & 3u) * 8u;
    TagMonoid tm = reduce_tag(tag_word & ((1u << shift) - 1u));
    TagMonoid base = {0, 0, 0, 0, 0};
    if ((ix >> 2) < n_words) base = ((const TagMonoid *)c->tag_monoids.p)[ix >> 2];
    else if (n_words) { /* reading one past the padded stream: behaves as a zero word after the last */
        base = ((const TagMonoid *)c->tag_monoids.p)[n_words - 1];
        base = tm_combine(base, reduce_tag(scene_rd(c, c->cfg.layout.path_tag_base + n_words - 1)));
        tag_word = 0;
        tm = reduce_tag(0);
    }
    tm = tm_combine(base, tm);
    PathTagData r;
    r.tag_byte = (tag_word >> shift) & 0xffu;
    tm.trans_ix -= 1u;
    tm.style_ix -= 2u;
    r.monoid = tm;
    return r;
}

static v2 read_f32_point(const vbo_ctx *c, uint32_t ix) {
    uint32_t b = c->cfg.layout.path_data_base + ix;
    return V2(u2f_bits(scene_rd(c, b)), u2f_bits(scene_rd(c, b + 1)));
}
static v2 read_i16_point(const vbo_ctx *c, uint32_t ix) {
    uint32_t raw = scene_rd(c, c->cfg.layout.path_data_base + ix);
    float x = (float)(((int32_t)(raw << 16)) >> 16);
    float y = (float)(((int32_t)raw) >> 16);
    return V2(x, y);
}

/* flatten.wgsl:708-766 */
static CubicPoints read_path_segment(const vbo_ctx *c, const PathTagData *tag, int is_stroke) {
    v2 p0, p1, p2 = V2(0, 0), p3 = V2(0, 0);
    uint32_t seg_type = tag->tag_byte & 3u;
    uint32_t off = tag->monoid.pathseg_offset;
    int is_stroke_cap_marker = is_stroke && (tag->tag_byte & 4u) != 0u;
    int is_open = seg_type == 2u;
    if (tag->tag_byte & 8u) {
        p0 = read_f32_point(c, off);
        p1 = read_f32_point(c, off + 2u);
        if (seg_type >= 2u) {
            p2 = read_f32_point(c, off + 4u);
            if (seg_type == 3u) p3 = read_f32_point(c, off + 6u);
        }
    } else {
        p0 = read_i16_point(c, off);
        p1 = read_i16_point(c, off + 1u);
        if (seg_type >= 2u) {
            p2 = read_i16_point(c, off + 2u);
            if (seg_type == 3u) p3 = read_i16_point(c, off + 3u);
        }
    }
    if (is_stroke_cap_marker && is_open) {
        p0 = p1;
        p1 = p2;
        seg_type = 1u;
    }
    const float third = 1.0f / 3.0f;
    if (seg_type == 1u) {
        p3 = p1;
        p2 = v2add(p3, v2scale(v2sub(p0, p3), third));
        p1 = v2add(p0, v2scale(v2sub(p3, p0), third));
    } else if (seg_type == 2u) {
        p3 = p2;
        p2 = v2add(p1, v2scale(v2sub(p2, p1), third));
        p1 = v2add(p1, v2scale(v2sub(p0, p1), third));
    }
    CubicPoints r = {p0, p1, p2, p3};
    return r;
}

/* flatten.wgsl:831-923 / cpu/flatten.rs:673-840 */
static void stage_flatten(vbo_ctx *c) {
    const vbo_layout *L = &c->cfg.layout;
    uint32_t n_paths = L->n_paths;
    PathBbox *pb = vec_resize(&c->path_bboxes, n_paths);
    for (uint32_t i = 0; i < n_paths; i++) { /* cpu/bbox_clear.rs */
        pb[i].x0 = 0x7fffffff; pb[i].y0 = 0x7fffffff;
        pb[i].x1 = (int32_t)0x80000000; pb[i].y1 = (int32_t)0x80000000;
        pb[i].draw_flags = 0; pb[i].trans_ix = 0;
    }
    c->lines.n = 0;
    uint32_t n_tags = (L->path_data_base - L->path_tag_base) * 4u;
    FlatCtx f;
    f.c = c;
    for (uint32_t ix = 0; ix < n_tags; ix++) {
        f.bbox[0] = 1e31f; f.bbox[1] = 1e31f; f.bbox[2] = -1e31f; f.bbox[3] = -1e31f;
        PathTagData tag = compute_tag_monoid(c, ix);
        uint32_t path_ix = tag.monoid.path_ix;
        uint32_t style_ix = tag.monoid.style_ix;
        uint32_t trans_ix = tag.monoid.trans_ix;
        uint32_t style_flags = scene_rd(c, L->style_base + style_ix);
        uint32_t draw_flags = (style_flags & STYLE_FLAGS_FILL) == 0u ? 0u : 1u;
        if ((tag.tag_byte & 0x10u) != 0u && path_ix < n_paths) {
            pb[path_ix].draw_flags = draw_flags;
            pb[path_ix].trans_ix = trans_ix;
        }
        uint32_t seg_type = tag.tag_byte & 3u;
        if (seg_type != 0u) {
            int is_stroke = (style_flags & STYLE_FLAGS_STYLE) != 0u;
            Xform transform = xf_read(c, L->transform_base, trans_ix);
            CubicPoints pts = read_path_segment(c, &tag, is_stroke);
            if (is_stroke) {
                float linewidth = u2f_bits(scene_rd(c, L->style_base + style_ix + 1u));
                float offset = 0.5f * linewidth;
                int is_open = seg_type != 1u;
                int is_stroke_cap_marker = (tag.tag_byte & 4u) != 0u;
                if (is_stroke_cap_marker) {
                    if (is_open) {
                        v2 tangent = v2sub(pts.p3, pts.p0);
                        v2 offset_tangent = v2scale(v2normalize(tangent), offset);
                        v2 n = V2(-offset_tangent.y, offset_tangent.x);
                        draw_cap(&f, path_ix, (style_flags & STYLE_FLAGS_START_CAP_MASK) >> 2, pts.p0, v2sub(pts.p0, n),
                                 v2add(pts.p0, n), V2(-offset_tangent.x, -offset_tangent.y), &transform);
                    }
                } else {
                    PathTagData ntag = compute_tag_monoid(c, ix + 1u);
                    CubicPoints npts = read_path_segment(c, &ntag, 1);
                    int n_is_closed = (ntag.tag_byte & 3u) == 1u;
                    int n_is_marker = (ntag.tag_byte & 4u) != 0u;
                    int do_join = !n_is_marker || n_is_closed;
                    v2 n_tangent = v2sub(npts.p3, npts.p0);
                    if (!n_is_marker) n_tangent = cubic_start_tangent(npts.p0, npts.p1, npts.p2, npts.p3);

                    v2 tan_start = cubic_start_tangent(pts.p0, pts.p1, pts.p2, pts.p3);
                    if (v2dot(tan_start, tan_start) < TANGENT_THRESH * TANGENT_THRESH) tan_start = V2(TANGENT_THRESH, 0.f);
                    v2 tan_prev = cubic_end_tangent(pts.p0, pts.p1, pts.p2, pts.p3);
                    if (v2dot(tan_prev, tan_prev) < TANGENT_THRESH * TANGENT_THRESH) tan_prev = V2(TANGENT_THRESH, 0.f);
                    v2 tan_next = n_tangent;
                    if (v2dot(tan_next, tan_next) < TANGENT_THRESH * TANGENT_THRESH) tan_next = V2(TANGENT_THRESH, 0.f);
                    v2 n_start = v2scale(v2normalize(V2(-tan_start.y, tan_start.x)), offset);
                    v2 offset_tangent = v2scale(v2normalize(tan_prev), offset);
                    v2 n_prev = V2(-offset_tangent.y, offset_tangent.x);
                    v2 tnn = v2scale(v2normalize(tan_next), offset);
                    v2 n_next = V2(-tnn.y, tnn.x);
                    flatten_euler(&f, &pts, path_ix, &transform, offset, v2add(pts.p0, n_start), v2add(pts.p3, n_prev));
                    flatten_euler(&f, &pts, path_ix, &transform, -offset, v2sub(pts.p0, n_start), v2sub(pts.p3, n_prev));
                    if (do_join) {
                        draw_join(&f, path_ix, style_flags, pts.p3, tan_prev, tan_next, n_prev, n_next, &transform);
                    } else {
                        draw_cap(&f, path_ix, style_flags & STYLE_FLAGS_END_CAP_MASK, pts.p3, v2add(pts.p3, n_prev),
                                 v2sub(pts.p3, n_prev), offset_tangent, &transform);
                    }
                }
            } else {
                flatten_euler(&f, &pts, path_ix, &transform, 0.f, pts.p0, pts.p3);
            }
            if ((f.bbox[2] > f.bbox[0] || f.bbox[3] > f.bbox[1]) && path_ix < n_paths) {
                PathBbox *o = &pb[path_ix];
                int32_t x0 = f2i_sat(floorf(f.bbox[0])), y0 = f2i_sat(floorf(f.bbox[1]));
                int32_t x1 = f2i_sat(ceilf(f.bbox[2])), y1 = f2i_sat(ceilf(f.bbox[3]));
                if (x0 < o->x0) o->x0 = x0;
                if (y0 < o->y0) o->y0 = y0;
                if (x1 > o->x1) o->x1 = x1;
                if (y1 > o->y1) o->y1 = y1;
            }
        }
    }
    c->bump.lines = (uint32_t)c->lines.n;
}

/* ------------------------------------------------------------------------------------------
 * 3. draw_reduce + draw_leaf: cpu/draw_reduce.rs, cpu/draw_leaf.rs, shader/draw_leaf.wgsl
 * ---------------------------------------------------------------------------------------- */
#define DRAWTAG_NOP 0u
#define DRAWTAG_FILL_COLOR 0x44u
#define DRAWTAG_FILL_LIN_GRADIENT 0x114u
#define DRAWTAG_FILL_RAD_GRADIENT 0x29cu
#define DRAWTAG_FILL_SWEEP_GRADIENT 0x254u
#define DRAWTAG_FILL_IMAGE 0x28Cu
#define DRAWTAG_BLURRED_ROUNDED_RECT 0x2d4u
#define DRAWTAG_BEGIN_CLIP 0x49u
#define DRAWTAG_END_CLIP 0x21u

static uint32_t read_draw_tag(const vbo_ctx *c, uint32_t ix) {
    return ix < c->cfg.layout.n_draw_objects ? scene_rd(c, c->cfg.layout.draw_tag_base + ix) : DRAWTAG_NOP;
}
/* shared/transform.wgsl */
static v2 xf_apply(const Xform *t, v2 p) {
    return V2(t->m[0] * p.x + t->m[2] * p.y + t->t[0], t->m[1] * p.x + t->m[3] * p.y + t->t[1]);
}
static Xform xf_inverse(const Xform *t) {
    float inv_det = 1.0f / (t->m[0] * t->m[3] - t->m[1] * t->m[2]);
    Xform r;
    r.m[0] = inv_det * t->m[3];
    r.m[1] = inv_det * -t->m[1];
    r.m[2] = inv_det * -t->m[2];
    r.m[3] = inv_det * t->m[0];
    r.t[0] = r.m[0] * -t->t[0] + r.m[2] * -t->t[1];
    r.t[1] = r.m[1] * -t->t[0] + r.m[3] * -t->t[1];
    return r;
}
static Xform xf_mul(const Xform *a, const Xform *b) {
    Xform r;
    r.m[0] = a->m[0] * b->m[0] + a->m[2] * b->m[1];
    r.m[1] = a->m[1] * b->m[0] + a->m[3] * b->m[1];
    r.m[2] = a->m[0] * b->m[2] + a->m[2] * b->m[3];
    r.m[3] = a->m[1] * b->m[2] + a->m[3] * b->m[3];
    r.t[0] = a->m[0] * b->t[0] + a->m[2] * b->t[1] + a->t[0];
    r.t[1] = a->m[1] * b->t[0] + a->m[3] * b->t[1] + a->t[1];
    return r;
}
static Xform from_poly2(v2 p0, v2 p1) { /* draw_leaf.wgsl:298-303 */
    Xform r = {{p1.y - p0.y, p0.x - p1.x, p1.x - p0.x, p1.y - p0.y}, {p0.x, p0.y}};
    return r;
}
static Xform two_point_to_unit_line(v2 p0, v2 p1) {
    Xform tmp1 = from_poly2(p0, p1);
    Xform inv = xf_inverse(&tmp1);
    Xform tmp2 = from_poly2(V2(0.f, 0.f), V2(1.f, 0.f));
    return xf_mul(&tmp2, &inv);
}
static void put_xform(uint32_t *info, const Xform *x) {
    for (int i = 0; i < 4; i++) info[i] = f2u_bits(x->m[i]);
    info[4] = f2u_bits(x->t[0]);
    info[5] = f2u_bits(x->t[1]);
}

static void stage_draw(vbo_ctx *c) {
    const vbo_layout *L = &c->cfg.layout;
    uint32_t n = L->n_draw_objects;
    DrawMonoid *dm = vec_resize(&c->draw_monoids, n);
    uint32_t *info = vec_resize(&c->info_bin_data, L->bin_data_start);
    ClipInp *clip_inp = vec_resize(&c->clip_inp, L->n_clips);
    const PathBbox *pbs = c->path_bboxes.p;
    DrawMonoid m = {0, 0, 0, 0};
    for (uint32_t ix = 0; ix < n; ix++) {
        uint32_t tag_word = read_draw_tag(c, ix);
        dm[ix] = m;
        uint32_t dd = L->draw_data_base + m.scene_offset;
        uint32_t di = m.info_offset;
        if (tag_word == DRAWTAG_FILL_COLOR || tag_word == DRAWTAG_FILL_LIN_GRADIENT || tag_word == DRAWTAG_FILL_RAD_GRADIENT ||
            tag_word == DRAWTAG_FILL_SWEEP_GRADIENT || tag_word == DRAWTAG_FILL_IMAGE || tag_word == DRAWTAG_BEGIN_CLIP ||
            tag_word == DRAWTAG_BLURRED_ROUNDED_RECT) {
            PathBbox bbox = pbs[m.path_ix];
            Xform transform = xf_read(c, L->transform_base, bbox.trans_ix);
            uint32_t draw_flags = bbox.draw_flags;
            switch (tag_word) {
            case DRAWTAG_FILL_COLOR:
            case DRAWTAG_BEGIN_CLIP:
                info[di] = draw_flags;
                break;
            case DRAWTAG_FILL_LIN_GRADIENT: {
                info[di] = draw_flags;
                v2 p0 = V2(u2f_bits(scene_rd(c, dd + 1)), u2f_bits(scene_rd(c, dd + 2)));
                v2 p1 = V2(u2f_bits(scene_rd(c, dd + 3)), u2f_bits(scene_rd(c, dd + 4)));
                p0 = xf_apply(&transform, p0);
                p1 = xf_apply(&transform, p1);
                v2 dxy = v2sub(p1, p0);
                float scale = 1.0f / v2dot(dxy, dxy);
                v2 line_xy = v2scale(dxy, scale);
                float line_c = -v2dot(p0, line_xy);
                info[di + 1] = f2u_bits(line_xy.x);
                info[di + 2] = f2u_bits(line_xy.y);
                info[di + 3] = f2u_bits(line_c);
                break;
            }
            case DRAWTAG_FILL_RAD_GRADIENT: {
                const float GRADIENT_EPSILON = 1.0f / (float)(1u << 12);
                info[di] = draw_flags;
                v2 p0 = V2(u2f_bits(scene_rd(c, dd + 1)), u2f_bits(scene_rd(c, dd + 2)));
                v2 p1 = V2(u2f_bits(scene_rd(c, dd + 3)), u2f_bits(scene_rd(c, dd + 4)));
                float r0 = u2f_bits(scene_rd(c, dd + 5));
                float r1 = u2f_bits(scene_rd(c, dd + 6));
                Xform user_to_gradient = xf_inverse(&transform);
                Xform xform = {{0, 0, 0, 0}, {0, 0}};
                float focal_x = 0.0f, radius = 0.0f;
                uint32_t kind = 0u, flags = 0u;
                if (fabsf(r0 - r1) <= GRADIENT_EPSILON) {
                    kind = 2u; /* STRIP */
                    float scaled = r0 / v2len(v2sub(p0, p1));
                    Xform tl = two_point_to_unit_line(p0, p1);
                    xform = xf_mul(&tl, &user_to_gradient);
                    radius = scaled * scaled;
                } else {
                    kind = 4u; /* CONE */
                    if (v2eq(p0, p1)) {
                        kind = 1u; /* CIRCULAR */
                        p0.x += GRADIENT_EPSILON;
                        p0.y += GRADIENT_EPSILON;
                    }
                    if (r1 == 0.0f) {
                        flags |= 1u; /* SWAPPED */
                        v2 tp = p0; p0 = p1; p1 = tp;
                        float tr = r0; r0 = r1; r1 = tr;
                    }
                    focal_x = r0 / (r0 - r1);
                    v2 cf = V2((1.0f - focal_x) * p0.x + focal_x * p1.x, (1.0f - focal_x) * p0.y + focal_x * p1.y);
                    radius = r1 / v2len(v2sub(cf, p1));
                    Xform tl = two_point_to_unit_line(cf, p1);
                    Xform user_to_unit_line = xf_mul(&tl, &user_to_gradient);
                    Xform user_to_scaled;
                    if (fabsf(radius - 1.0f) <= GRADIENT_EPSILON) {
                        kind = 3u; /* FOCAL_ON_CIRCLE */
                        float scale = 0.5f * fabsf(1.0f - focal_x);
                        Xform s = {{scale, 0.f, 0.f, scale}, {0.f, 0.f}};
                        user_to_scaled = xf_mul(&s, &user_to_unit_line);
                    } else {
                        float a = radius * radius - 1.0f;
                        float scale_ratio = fabsf(1.0f - focal_x) / a;
                        float scale_x = radius * scale_ratio;
                        float scale_y = sqrtf(fabsf(a)) * scale_ratio;
                        Xform s = {{scale_x, 0.f, 0.f, scale_y}, {0.f, 0.f}};
                        user_to_scaled = xf_mul(&s, &user_to_unit_line);
                    }
                    xform = user_to_scaled;
                }
                put_xform(info + di + 1, &xform);
                info[di + 7] = f2u_bits(focal_x);
                info[di + 8] = f2u_bits(radius);
                info[di + 9] = (flags << 3) | kind;
                break;
            }
            case DRAWTAG_FILL_SWEEP_GRADIENT: {
                info[di] = draw_flags;
                v2 p0 = V2(u2f_bits(scene_rd(c, dd + 1)), u2f_bits(scene_rd(c, dd + 2)));
                Xform tr = {{1.f, 0.f, 0.f, 1.f}, {p0.x, p0.y}};
                Xform xf = xf_mul(&transform, &tr);
                Xform inv = xf_inverse(&xf);
                put_xform(info + di + 1, &inv);
                info[di + 7] = scene_rd(c, dd + 3);
                info[di + 8] = scene_rd(c, dd + 4);
                break;
            }
            case DRAWTAG_FILL_IMAGE: {
                info[di] = draw_flags;
                Xform inv = xf_inverse(&transform);
                put_xform(info + di + 1, &inv);
                info[di + 7] = scene_rd(c, dd);
                info[di + 8] = scene_rd(c, dd + 1);
                info[di + 9] = scene_rd(c, dd + 2);
                break;
            }
            case DRAWTAG_BLURRED_ROUNDED_RECT: {
                info[di] = draw_flags;
                Xform inv = xf_inverse(&transform);
                put_xform(info + di + 1, &inv);
                info[di + 7] = scene_rd(c, dd + 1);
                info[di + 8] = scene_rd(c, dd + 2);
                info[di + 9] = scene_rd(c, dd + 3);
                info[di + 10] = scene_rd(c, dd + 4);
                break;
            }
            default: break;
            }
        }
        if (tag_word == DRAWTAG_BEGIN_CLIP || tag_word == DRAWTAG_END_CLIP) {
            uint32_t path_ix = ~ix;
            if (tag_word == DRAWTAG_BEGIN_CLIP) path_ix = m.path_ix;
            if (m.clip_ix < L->n_clips) {
                clip_inp[m.clip_ix].ix = ix;
                clip_inp[m.clip_ix].path_ix = (int32_t)path_ix;
            }
        }
        /* draw.rs:252-272 / drawtag.wgsl:47-54 */
        m.path_ix += (tag_word != DRAWTAG_NOP);
        m.clip_ix += tag_word & 1u;
        m.scene_offset += (tag_word >> 2) & 0x07u;
        m.info_offset += (tag_word >> 6) & 0x0fu;
    }
}

/* ------------------------------------------------------------------------------------------
 * 4. clip_leaf: cpu/clip_leaf.rs (sequential stack; no depth limit). clip_reduce's outputs
 *    (clip_bic / clip_els) are only consumed by the WGSL clip_leaf and are not materialised.
 * ---------------------------------------------------------------------------------------- */
typedef struct { uint32_t parent_ix, path_ix; float bbox[4]; } ClipStackEl;

static void stage_clip(vbo_ctx *c) {
    uint32_t n_clips = c->cfg.layout.n_clips;
    Bbox4 *cb = vec_resize(&c->clip_bboxes, n_clips);
    const ClipInp *inp = c->clip_inp.p;
    const PathBbox *pbs = c->path_bboxes.p;
    DrawMonoid *dm = c->draw_monoids.p;
    ClipStackEl *stack = malloc(sizeof(ClipStackEl) * (n_clips + 1));
    uint32_t sp = 0;
    for (uint32_t g = 0; g < n_clips; g++) {
        ClipInp el = inp[g];
        if (el.path_ix >= 0) {
            PathBbox pb = pbs[el.path_ix];
            float b[4] = {(float)pb.x0, (float)pb.y0, (float)pb.x1, (float)pb.y1};
            if (sp > 0) {
                const float *l = stack[sp - 1].bbox;
                b[0] = fmaxf(b[0], l[0]); b[1] = fmaxf(b[1], l[1]);
                b[2] = fminf(b[2], l[2]); b[3] = fminf(b[3], l[3]);
            }
            memcpy(cb[g].b, b, sizeof b);
            stack[sp].parent_ix = el.ix;
            stack[sp].path_ix = (uint32_t)el.path_ix;
            memcpy(stack[sp].bbox, b, sizeof b);
            sp++;
        } else {
            if (sp == 0) continue; /* unbalanced: the encoder never produces this */
            ClipStackEl tos = stack[--sp];
            float big[4] = {-1e9f, -1e9f, 1e9f, 1e9f};
            memcpy(cb[g].b, sp > 0 ? stack[sp - 1].bbox : big, sizeof big);
            dm[el.ix].path_ix = tos.path_ix;
            dm[el.ix].scene_offset = dm[tos.parent_ix].scene_offset;
            dm[el.ix].info_offset = dm[tos.parent_ix].info_offset;
        }
    }
    free(stack);
}

/* ------------------------------------------------------------------------------------------
 * 5. binning: cpu/binning.rs, shader/binning.wgsl
 * ---------------------------------------------------------------------------------------- */
static void stage_binning(vbo_ctx *c) {
    const Config *cfg = &c->cfg;
    const vbo_layout *L = &cfg->layout;
    const float SX = 1.0f / 256.0f, SY = 1.0f / 256.0f;
    int32_t width_in_bins = (int32_t)((cfg->width_in_tiles + 15u) / 16u);
    int32_t height_in_bins = (int32_t)((cfg->height_in_tiles + 15u) / 16u);
    uint32_t n_bins = (uint32_t)(width_in_bins * height_in_bins);
    uint32_t aligned_n_bins = (n_bins + 255u) & ~255u;
    uint32_t n_draw = L->n_draw_objects;
    uint32_t n_wg = (n_draw + 255u) / 256u;
    Bbox4 *ib = vec_resize(&c->draw_bboxes, n_draw);
    BinHeader *hdr = vec_resize(&c->bin_headers, (size_t)n_wg * aligned_n_bins);
    memset(hdr, 0, sizeof(BinHeader) * (size_t)n_wg * aligned_n_bins);
    const DrawMonoid *dm = c->draw_monoids.p;
    const PathBbox *pbs = c->path_bboxes.p;
    const Bbox4 *cbs = c->clip_bboxes.p;
    uint32_t *counts = malloc(sizeof(uint32_t) * (n_bins + 1));
    uint32_t *chunk = malloc(sizeof(uint32_t) * (n_bins + 1));
    c->bump.binning = 0;
    c->info_bin_data.n = L->bin_data_start;
    for (uint32_t wg = 0; wg < n_wg; wg++) {
        int32_t bb[256][4];
        memset(counts, 0, sizeof(uint32_t) * n_bins);
        for (uint32_t li = 0; li < 256; li++) {
            uint32_t el = wg * 256u + li;
            int32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
            if (el < n_draw) {
                DrawMonoid m = dm[el];
                float cbx[4] = {-1e9f, -1e9f, 1e9f, 1e9f};
                if (m.clip_ix > 0u) {
                    uint32_t ci = m.clip_ix - 1u;
                    if (ci > L->n_clips - 1u) ci = L->n_clips - 1u;
                    memcpy(cbx, cbs[ci].b, sizeof cbx);
                }
                PathBbox pb = pbs[m.path_ix];
                float b[4] = {fmaxf(cbx[0], (float)pb.x0), fmaxf(cbx[1], (float)pb.y0), fminf(cbx[2], (float)pb.x1),
                              fminf(cbx[3], (float)pb.y1)};
                memcpy(ib[el].b, b, sizeof b);
                if (b[0] < b[2] && b[1] < b[3]) {
                    x0 = f2i_sat(floorf(b[0] * SX));
                    y0 = f2i_sat(floorf(b[1] * SY));
                    x1 = f2i_sat(ceilf(b[2] * SX));
                    y1 = f2i_sat(ceilf(b[3] * SY));
                }
            }
            x0 = clampi(x0, 0, width_in_bins);
            x1 = clampi(x1, 0, width_in_bins);
            y0 = clampi(y0, (int32_t)c->win_by0, (int32_t)c->win_by1);
            y1 = clampi(y1, (int32_t)c->win_by0, (int32_t)c->win_by1);
            if (x0 == x1) y1 = y0;
            for (int32_t y = y0; y < y1; y++)
                for (int32_t x = x0; x < x1; x++) counts[y * width_in_bins + x]++;
            bb[li][0] = x0; bb[li][1] = y0; bb[li][2] = x1; bb[li][3] = y1;
        }
        for (uint32_t b = 0; b < n_bins; b++) {
            chunk[b] = c->bump.binning;
            c->bump.binning += counts[b];
            hdr[(size_t)wg * aligned_n_bins + b].element_count = counts[b];
            hdr[(size_t)wg * aligned_n_bins + b].chunk_offset = chunk[b];
        }
        uint32_t *ibd = vec_resize(&c->info_bin_data, (size_t)L->bin_data_start + c->bump.binning);
        for (uint32_t li = 0; li < 256; li++) {
            uint32_t el = wg * 256u + li;
            for (int32_t y = bb[li][1]; y < bb[li][3]; y++)
                for (int32_t x = bb[li][0]; x < bb[li][2]; x++) {
                    uint32_t b = (uint32_t)(y * width_in_bins + x);
                    ibd[L->bin_data_start + chunk[b]] = el;
                    chunk[b]++;
                }
        }
    }
    free(counts);
    free(chunk);
}

/* ------------------------------------------------------------------------------------------
 * 6. tile_alloc: cpu/tile_alloc.rs
 * ---------------------------------------------------------------------------------------- */
static void stage_tile_alloc(vbo_ctx *c) {
    const Config *cfg = &c->cfg;
    const vbo_layout *L = &cfg->layout;
    const float SX = 1.0f / 16.0f, SY = 1.0f / 16.0f;
    uint32_t n = L->n_draw_objects;
    PathRec *paths = vec_resize(&c->paths, (n + 255u) & ~255u);
    const Bbox4 *dbs = c->draw_bboxes.p;
    c->bump.tile = 0;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t drawtag = scene_rd(c, L->draw_tag_base + i);
        int32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
        if (drawtag != DRAWTAG_NOP && drawtag != DRAWTAG_END_CLIP) {
            const float *b = dbs[i].b;
            if (b[0] < b[2] && b[1] < b[3]) {
                x0 = f2i_sat(floorf(b[0] * SX));
                y0 = f2i_sat(floorf(b[1] * SY));
                x1 = f2i_sat(ceilf(b[2] * SX));
                y1 = f2i_sat(ceilf(b[3] * SY));
            }
        }
        uint32_t ux0 = (uint32_t)clampi(x0, 0, (int32_t)cfg->width_in_tiles);
        uint32_t ux1 = (uint32_t)clampi(x1, 0, (int32_t)cfg->width_in_tiles);
        uint32_t uy0 = (uint32_t)clampi(y0, (int32_t)c->win_ty0, (int32_t)c->win_ty1);
        uint32_t uy1 = (uint32_t)clampi(y1, (int32_t)c->win_ty0, (int32_t)c->win_ty1);
        uint32_t tile_count = (ux1 - ux0) * (uy1 - uy0);
        memset(&paths[i], 0, sizeof(PathRec));
        paths[i].bbox[0] = ux0; paths[i].bbox[1] = uy0; paths[i].bbox[2] = ux1; paths[i].bbox[3] = uy1;
        paths[i].tiles = c->bump.tile;
        c->bump.tile += tile_count;
    }
    Tile *tiles = vec_resize(&c->tiles, c->bump.tile);
    memset(tiles, 0, sizeof(Tile) * c->bump.tile);
}

/* ------------------------------------------------------------------------------------------
 * 7. path_count: shader/path_count.wgsl:51-202 (cull comparisons follow the WGSL: <=)
 * ---------------------------------------------------------------------------------------- */
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define TILE_SCALE 0.0625f

static void stage_path_count(vbo_ctx *c) {
    const LineSoup *lines = c->lines.p;
    const PathRec *paths = c->paths.p;
    Tile *tile = c->tiles.p;
    uint32_t n_lines = c->bump.lines;
    c->bump.seg_counts = 0;
    c->seg_counts.n = 0;
    for (uint32_t line_ix = 0; line_ix < n_lines; line_ix++) {
        LineSoup line = lines[line_ix];
        v2 lp0 = V2(line.p0[0], line.p0[1]), lp1 = V2(line.p1[0], line.p1[1]);
        int is_down = lp1.y >= lp0.y;
        v2 xy0 = is_down ? lp0 : lp1;
        v2 xy1 = is_down ? lp1 : lp0;
        v2 s0 = v2scale(xy0, TILE_SCALE);
        v2 s1 = v2scale(xy1, TILE_SCALE);
        uint32_t count_x = span_u(s0.x, s1.x) - 1u;
        uint32_t count = count_x + span_u(s0.y, s1.y);
        float dx = fabsf(s1.x - s0.x);
        float dy = s1.y - s0.y;
        if (dx + dy == 0.0f) continue;
        if (dy == 0.0f && floorf(s0.y) == s0.y) continue;
        float idxdy = 1.0f / (dx + dy);
        float a = dx * idxdy;
        int is_positive_slope = s1.x >= s0.x;
        float x_sign = is_positive_slope ? 1.0f : -1.0f;
        float xt0 = floorf(s0.x * x_sign);
        float cc = s0.x * x_sign - xt0;
        float y0 = floorf(s0.y);
        float ytop = (s0.y == s1.y) ? ceilf(s0.y) : y0 + 1.0f;
        float b = fminf((dy * cc + dx * (ytop - s0.y)) * idxdy, ONE_MINUS_ULP);
        float robust_err = floorf(a * ((float)count - 1.0f) + b) - (float)count_x;
        if (robust_err != 0.0f) a -= ROBUST_EPSILON * signf(robust_err);
        float x0 = xt0 * x_sign + (is_positive_slope ? 0.0f : -1.0f);

        if (line.path_ix >= c->cfg.layout.n_draw_objects) continue;
        PathRec path = paths[line.path_ix];
        int32_t bbox[4] = {(int32_t)path.bbox[0], (int32_t)path.bbox[1], (int32_t)path.bbox[2], (int32_t)path.bbox[3]};
        float xmin = fminf(s0.x, s1.x);
        int32_t stride = bbox[2] - bbox[0];
        if (s0.y >= (float)bbox[3] || s1.y <= (float)bbox[1] || xmin >= (float)bbox[2] || stride == 0) continue;
        uint32_t imin = 0u;
        if (s0.y < (float)bbox[1]) {
            float iminf = rintf(((float)bbox[1] - y0 + b - a) / (1.0f - a)) - 1.0f;
            if (y0 + iminf - floorf(a * iminf + b) < (float)bbox[1]) iminf += 1.0f;
            imin = f2u_sat(iminf);
        }
        uint32_t imax = count;
        if (s1.y > (float)bbox[3]) {
            float imaxf = rintf(((float)bbox[3] - y0 + b - a) / (1.0f - a)) - 1.0f;
            if (y0 + imaxf - floorf(a * imaxf + b) < (float)bbox[3]) imaxf += 1.0f;
            imax = f2u_sat(imaxf);
        }
        int32_t delta = is_down ? -1 : 1;
        int32_t ymin = 0, ymax = 0;
        if (fmaxf(s0.x, s1.x) <= (float)bbox[0]) {
            ymin = f2i_sat(ceilf(s0.y));
            ymax = f2i_sat(ceilf(s1.y));
            imax = imin;
        } else {
            float fudge = is_positive_slope ? 0.0f : 1.0f;
            if (xmin < (float)bbox[0]) {
                float f = rintf((x_sign * ((float)bbox[0] - x0) - b + fudge) / a);
                if ((x0 + x_sign * floorf(a * f + b) < (float)bbox[0]) == is_positive_slope) f += 1.0f;
                int32_t ynext = f2i_sat(y0 + f - floorf(a * f + b) + 1.0f);
                if (is_positive_slope) {
                    if (f2u_sat(f) > imin) {
                        ymin = f2i_sat(y0 + ((y0 == s0.y) ? 0.0f : 1.0f));
                        ymax = ynext;
                        imin = f2u_sat(f);
                    }
                } else {
                    if (f2u_sat(f) < imax) {
                        ymin = ynext;
                        ymax = f2i_sat(ceilf(s1.y));
                        imax = f2u_sat(f);
                    }
                }
            }
            if (fmaxf(s0.x, s1.x) > (float)bbox[2]) {
                float f = rintf((x_sign * ((float)bbox[2] - x0) - b + fudge) / a);
                if ((x0 + x_sign * floorf(a * f + b) < (float)bbox[2]) == is_positive_slope) f += 1.0f;
                if (is_positive_slope) {
                    uint32_t fu = f2u_sat(f);
                    if (fu < imax) imax = fu;
                } else {
                    uint32_t fu = f2u_sat(f);
                    if (fu > imin) imin = fu;
                }
            }
        }
        if (imax < imin) imax = imin;
        if (ymin < bbox[1]) ymin = bbox[1];
        if (ymax > bbox[3]) ymax = bbox[3];
        for (int32_t y = ymin; y < ymax; y++) {
            int32_t base = (int32_t)path.tiles + (y - bbox[1]) * stride;
            tile[base].backdrop += delta;
        }
        float last_z = floorf(a * ((float)imin - 1.0f) + b);
        uint32_t seg_base = c->bump.seg_counts;
        c->bump.seg_counts += imax - imin;
        SegmentCount *sc = vec_resize(&c->seg_counts, c->bump.seg_counts);
        for (uint32_t i = imin; i < imax; i++) {
            float zf = a * (float)i + b;
            float z = floorf(zf);
            int32_t y = f2i_sat(y0 + (float)i - z);
            int32_t x = f2i_sat(x0 + x_sign * z);
            int32_t base = (int32_t)path.tiles + (y - bbox[1]) * stride - bbox[0];
            int top_edge = (i == 0u) ? (y0 == s0.y) : (last_z == z);
            if (top_edge && x + 1 < bbox[2]) {
                int32_t x_bump = (x + 1 > bbox[0]) ? x + 1 : bbox[0];
                tile[base + x_bump].backdrop += delta;
            }
            uint32_t seg_within_slice = tile[base + x].segment_count_or_ix;
            tile[base + x].segment_count_or_ix += 1u;
            sc[seg_base + i - imin].line_ix = line_ix;
            sc[seg_base + i - imin].counts = (seg_within_slice << 16) | i;
            last_z = z;
        }
    }
    /* a copy of the counts for the tests: the CUDA backdrop turns them into slice starts, which coarse here overwrites */
    uint32_t *counts = vec_resize(&c->tile_counts, c->bump.tile);
    for (uint32_t t = 0; t < c->bump.tile; t++) counts[t] = tile[t].segment_count_or_ix;
}

/* ------------------------------------------------------------------------------------------
 * 8. backdrop: cpu/backdrop.rs
 * ---------------------------------------------------------------------------------------- */
static void stage_backdrop(vbo_ctx *c) {
    const PathRec *paths = c->paths.p;
    Tile *tiles = c->tiles.p;
    for (uint32_t i = 0; i < c->cfg.layout.n_draw_objects; i++) {
        PathRec p = paths[i];
        uint32_t width = p.bbox[2] - p.bbox[0];
        uint32_t height = p.bbox[3] - p.bbox[1];
        for (uint32_t y = 0; y < height; y++) {
            int32_t sum = 0;
            for (uint32_t x = 0; x < width; x++) {
                Tile *t = &tiles[p.tiles + y * width + x];
                sum += t->backdrop;
                t->backdrop = sum;
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * 9. coarse: cpu/coarse.rs with the WGSL's fixed 256-word chunks (coarse.wgsl:68-86)
 * ---------------------------------------------------------------------------------------- */
#define PTCL_INITIAL_ALLOC 64u
#define PTCL_INCREMENT 256u
#define PTCL_HEADROOM 2u
enum { CMD_END = 0, CMD_FILL = 1, CMD_SOLID = 3, CMD_COLOR = 5, CMD_LIN_GRAD = 6, CMD_RAD_GRAD = 7, CMD_SWEEP_GRAD = 8,
       CMD_IMAGE = 9, CMD_BEGIN_CLIP = 10, CMD_END_CLIP = 11, CMD_JUMP = 12, CMD_BLUR_RECT = 13 };
#define BLEND_STACK_SPLIT 4u

typedef struct { vbo_ctx *c; uint32_t cmd_offset, cmd_limit; } TileState;

static uint32_t *ptcl_at(vbo_ctx *c, uint32_t ix) {
    if (ix >= c->ptcl.n) vec_resize(&c->ptcl, (size_t)ix + 1);
    return (uint32_t *)c->ptcl.p + ix;
}
static void alloc_cmd(TileState *s, uint32_t size) {
    if (s->cmd_offset + size >= s->cmd_limit) {
        vbo_ctx *c = s->c;
        uint32_t dyn_start = c->cfg.width_in_tiles * c->cfg.height_in_tiles * PTCL_INITIAL_ALLOC;
        uint32_t new_cmd = dyn_start + c->bump.ptcl;
        c->bump.ptcl += PTCL_INCREMENT;
        vec_resize(&c->ptcl, (size_t)new_cmd + PTCL_INCREMENT);
        *ptcl_at(c, s->cmd_offset) = CMD_JUMP;
        *ptcl_at(c, s->cmd_offset + 1) = new_cmd;
        s->cmd_offset = new_cmd;
        s->cmd_limit = new_cmd + (PTCL_INCREMENT - PTCL_HEADROOM);
    }
}
static void wr(TileState *s, uint32_t off, uint32_t v) { *ptcl_at(s->c, s->cmd_offset + off) = v; }
static void write_path(TileState *s, Tile *tile, uint32_t draw_flags) {
    uint32_t n_segs = tile->segment_count_or_ix;
    if (n_segs != 0u) {
        uint32_t seg_ix = s->c->bump.segments;
        tile->segment_count_or_ix = ~seg_ix;
        s->c->bump.segments += n_segs;
        alloc_cmd(s, 4);
        wr(s, 0, CMD_FILL);
        wr(s, 1, (n_segs << 1) | (draw_flags & 1u));
        wr(s, 2, seg_ix);
        wr(s, 3, (uint32_t)tile->backdrop);
        s->cmd_offset += 4;
    } else {
        alloc_cmd(s, 1);
        wr(s, 0, CMD_SOLID);
        s->cmd_offset += 1;
    }
}

static void stage_coarse(vbo_ctx *c) {
    const Config *cfg = &c->cfg;
    const vbo_layout *L = &cfg->layout;
    uint32_t width_in_tiles = cfg->width_in_tiles, height_in_tiles = cfg->height_in_tiles;
    uint32_t width_in_bins = (width_in_tiles + 15u) / 16u, height_in_bins = (height_in_tiles + 15u) / 16u;
    uint32_t n_bins = width_in_bins * height_in_bins;
    uint32_t aligned_n_bins = (n_bins + 255u) & ~255u;
    uint32_t n_partitions = (L->n_draw_objects + 255u) / 256u;
    const BinHeader *hdr = c->bin_headers.p;
    const DrawMonoid *dms = c->draw_monoids.p;
    const PathRec *paths = c->paths.p;
    Tile *tiles = c->tiles.p;
    c->bump.ptcl = 0; c->bump.segments = 0; c->bump.blend = 0;
    vec_resize(&c->ptcl, (size_t)width_in_tiles * height_in_tiles * PTCL_INITIAL_ALLOC);
    memset(c->ptcl.p, 0, c->ptcl.n * 4);
    Vec compacted[256];
    for (int i = 0; i < 256; i++) vec_init(&compacted[i], 4);
    for (uint32_t bin = 0; bin < n_bins; bin++) {
        uint32_t bin_x = bin % width_in_bins, bin_y = bin / width_in_bins;
        if (bin_y < c->win_by0 || bin_y >= c->win_by1) continue;
        for (int i = 0; i < 256; i++) compacted[i].n = 0;
        uint32_t bin_tile_x = 16u * bin_x, bin_tile_y = 16u * bin_y;
        for (uint32_t part = 0; part < n_partitions; part++) {
            BinHeader h = hdr[(size_t)part * aligned_n_bins + bin];
            const uint32_t *ibd = c->info_bin_data.p;
            uint32_t start = L->bin_data_start + h.chunk_offset;
            for (uint32_t i = 0; i < h.element_count; i++) {
                uint32_t drawobj_ix = ibd[start + i];
                uint32_t tag = scene_rd(c, L->draw_tag_base + drawobj_ix);
                if (tag == DRAWTAG_NOP) continue;
                PathRec path = paths[dms[drawobj_ix].path_ix];
                int32_t dx = (int32_t)path.bbox[0] - (int32_t)bin_tile_x;
                int32_t dy = (int32_t)path.bbox[1] - (int32_t)bin_tile_y;
                int32_t x0 = clampi(dx, 0, 16), y0 = clampi(dy, 0, 16);
                int32_t x1 = clampi((int32_t)path.bbox[2] - (int32_t)bin_tile_x, 0, 16);
                int32_t y1 = clampi((int32_t)path.bbox[3] - (int32_t)bin_tile_y, 0, 16);
                for (int32_t y = y0; y < y1; y++)
                    for (int32_t x = x0; x < x1; x++) {
                        Vec *v = &compacted[y * 16 + x];
                        uint32_t *p = vec_reserve(v, v->n + 1);
                        p[v->n++] = drawobj_ix;
                    }
            }
        }
        for (uint32_t tile_ix = 0; tile_ix < 256; tile_ix++) {
            uint32_t tile_x = tile_ix % 16u, tile_y = tile_ix / 16u;
            uint32_t this_tile_ix = (bin_tile_y + tile_y) * width_in_tiles + bin_tile_x + tile_x;
            TileState st = {c, this_tile_ix * PTCL_INITIAL_ALLOC, this_tile_ix * PTCL_INITIAL_ALLOC + (PTCL_INITIAL_ALLOC - PTCL_HEADROOM)};
            uint32_t blend_offset = st.cmd_offset;
            st.cmd_offset += 1;
            uint32_t clip_depth = 0, render_blend_depth = 0, max_blend_depth = 0, clip_zero_depth = 0;
            const uint32_t *objs = compacted[tile_ix].p;
            for (size_t k = 0; k < compacted[tile_ix].n; k++) {
                uint32_t drawobj_ix = objs[k];
                uint32_t drawtag = scene_rd(c, L->draw_tag_base + drawobj_ix);
                DrawMonoid dm = dms[drawobj_ix];
                PathRec path = paths[dm.path_ix];
                uint32_t stride = path.bbox[2] - path.bbox[0];
                uint32_t x = bin_tile_x + tile_x - path.bbox[0];
                uint32_t y = bin_tile_y + tile_y - path.bbox[1];
                Tile *tile = &tiles[path.tiles + y * stride + x];
                int is_clip = (drawtag & 1u) != 0u;
                int is_blend = 0;
                uint32_t dd = L->draw_data_base + dm.scene_offset;
                uint32_t di = dm.info_offset;
                if (is_clip) is_blend = scene_rd(c, dd) != ((128u << 8) | 3u);
                uint32_t draw_flags = ((const uint32_t *)c->info_bin_data.p)[di];
                int even_odd = (draw_flags & 1u) != 0u;
                uint32_t n_segs = tile->segment_count_or_ix;
                int32_t bd = tile->backdrop;
                int backdrop_clear = (even_odd ? ((bd < 0 ? -bd : bd) & 1) : bd) == 0;
                int include_tile = n_segs != 0u || (backdrop_clear == is_clip) || is_blend;
                if (!include_tile) continue;
                if (clip_zero_depth == 0u) {
                    switch (drawtag) {
                    case DRAWTAG_FILL_COLOR:
                        write_path(&st, tile, draw_flags);
                        alloc_cmd(&st, 2); wr(&st, 0, CMD_COLOR); wr(&st, 1, scene_rd(c, dd)); st.cmd_offset += 2;
                        break;
                    case DRAWTAG_BLURRED_ROUNDED_RECT:
                        write_path(&st, tile, draw_flags);
                        alloc_cmd(&st, 3); wr(&st, 0, CMD_BLUR_RECT); wr(&st, 1, di + 1u); wr(&st, 2, scene_rd(c, dd)); st.cmd_offset += 3;
                        break;
                    case DRAWTAG_FILL_LIN_GRADIENT:
                    case DRAWTAG_FILL_RAD_GRADIENT:
                    case DRAWTAG_FILL_SWEEP_GRADIENT: {
                        uint32_t ty = drawtag == DRAWTAG_FILL_LIN_GRADIENT ? CMD_LIN_GRAD
                                      : drawtag == DRAWTAG_FILL_RAD_GRADIENT ? CMD_RAD_GRAD : CMD_SWEEP_GRAD;
                        write_path(&st, tile, draw_flags);
                        alloc_cmd(&st, 3); wr(&st, 0, ty); wr(&st, 1, scene_rd(c, dd)); wr(&st, 2, di + 1u); st.cmd_offset += 3;
                        break;
                    }
                    case DRAWTAG_FILL_IMAGE:
                        write_path(&st, tile, draw_flags);
                        alloc_cmd(&st, 2); wr(&st, 0, CMD_IMAGE); wr(&st, 1, di + 1u); st.cmd_offset += 2;
                        break;
                    case DRAWTAG_BEGIN_CLIP:
                        if (tile->segment_count_or_ix == 0u && backdrop_clear) {
                            clip_zero_depth = clip_depth + 1u;
                        } else {
                            alloc_cmd(&st, 1); wr(&st, 0, CMD_BEGIN_CLIP); st.cmd_offset += 1;
                            render_blend_depth += 1u;
                            if (render_blend_depth > max_blend_depth) max_blend_depth = render_blend_depth;
                        }
                        clip_depth += 1u;
                        break;
                    case DRAWTAG_END_CLIP:
                        clip_depth -= 1u;
                        write_path(&st, tile, draw_flags);
                        alloc_cmd(&st, 3); wr(&st, 0, CMD_END_CLIP); wr(&st, 1, scene_rd(c, dd)); wr(&st, 2, scene_rd(c, dd + 1u)); st.cmd_offset += 3;
                        render_blend_depth -= 1u;
                        break;
                    default: break;
                    }
                } else {
                    if (drawtag == DRAWTAG_BEGIN_CLIP) clip_depth += 1u;
                    else if (drawtag == DRAWTAG_END_CLIP) {
                        if (clip_depth == clip_zero_depth) clip_zero_depth = 0u;
                        clip_depth -= 1u;
                    }
                }
            }
            if (bin_tile_x + tile_x < width_in_tiles && bin_tile_y + tile_y < height_in_tiles) {
                *ptcl_at(c, st.cmd_offset) = CMD_END;
                uint32_t blend_ix = 0;
                if (max_blend_depth > BLEND_STACK_SPLIT) {
                    uint32_t scratch = (max_blend_depth - BLEND_STACK_SPLIT) * 256u;
                    blend_ix = c->bump.blend;
                    c->bump.blend += scratch;
                }
                *ptcl_at(c, blend_offset) = blend_ix;
            }
        }
    }
    for (int i = 0; i < 256; i++) vec_free(&compacted[i]);
}

/* ------------------------------------------------------------------------------------------
 * 10. path_tiling: shader/path_tiling.wgsl:40-172, cpu/path_tiling.rs
 * ---------------------------------------------------------------------------------------- */
static void stage_path_tiling(vbo_ctx *c) {
    const SegmentCount *scs = c->seg_counts.p;
    const LineSoup *lines = c->lines.p;
    const PathRec *paths = c->paths.p;
    const Tile *tiles = c->tiles.p;
    Segment *segments = vec_resize(&c->segments, c->bump.segments);
    memset(segments, 0, sizeof(Segment) * c->bump.segments);
    for (uint32_t g = 0; g < c->bump.seg_counts; g++) {
        SegmentCount sc = scs[g];
        LineSoup line = lines[sc.line_ix];
        uint32_t seg_within_slice = sc.counts >> 16;
        uint32_t seg_within_line = sc.counts & 0xffffu;
        v2 lp0 = V2(line.p0[0], line.p0[1]), lp1 = V2(line.p1[0], line.p1[1]);
        int is_down = lp1.y >= lp0.y;
        v2 xy0 = is_down ? lp0 : lp1;
        v2 xy1 = is_down ? lp1 : lp0;
        v2 s0 = v2scale(xy0, TILE_SCALE);
        v2 s1 = v2scale(xy1, TILE_SCALE);
        uint32_t count_x = span_u(s0.x, s1.x) - 1u;
        uint32_t count = count_x + span_u(s0.y, s1.y);
        float dx = fabsf(s1.x - s0.x);
        float dy = s1.y - s0.y;
        float idxdy = 1.0f / (dx + dy);
        float a = dx * idxdy;
        int is_positive_slope = s1.x >= s0.x;
        float x_sign = is_positive_slope ? 1.0f : -1.0f;
        float xt0 = floorf(s0.x * x_sign);
        float cc = s0.x * x_sign - xt0;
        float y0i = floorf(s0.y);
        float ytop = (s0.y == s1.y) ? ceilf(s0.y) : y0i + 1.0f;
        float b = fminf((dy * cc + dx * (ytop - s0.y)) * idxdy, ONE_MINUS_ULP);
        float robust_err = floorf(a * ((float)count - 1.0f) + b) - (float)count_x;
        if (robust_err != 0.0f) a -= ROBUST_EPSILON * signf(robust_err);
        int32_t x0i = f2i_sat(xt0 * x_sign + 0.5f * (x_sign - 1.0f));
        float z = floorf(a * (float)seg_within_line + b);
        int32_t x = x0i + f2i_sat(x_sign * z);
        int32_t y = f2i_sat(y0i + (float)seg_within_line - z);
        PathRec path = paths[line.path_ix];
        int32_t bbox[4] = {(int32_t)path.bbox[0], (int32_t)path.bbox[1], (int32_t)path.bbox[2], (int32_t)path.bbox[3]};
        int32_t stride = bbox[2] - bbox[0];
        int32_t tile_ix = (int32_t)path.tiles + (y - bbox[1]) * stride + x - bbox[0];
        Tile tile = tiles[tile_ix];
        uint32_t seg_start = ~tile.segment_count_or_ix;
        if ((int32_t)seg_start < 0) continue;
        v2 tile_xy = V2((float)x * 16.0f, (float)y * 16.0f);
        v2 tile_xy1 = V2(tile_xy.x + 16.0f, tile_xy.y + 16.0f);
        if (seg_within_line > 0u) {
            float z_prev = floorf(a * ((float)seg_within_line - 1.0f) + b);
            if (z == z_prev) {
                float xt = xy0.x + (xy1.x - xy0.x) * (tile_xy.y - xy0.y) / (xy1.y - xy0.y);
                xt = clampf(xt, tile_xy.x + 1e-3f, tile_xy1.x);
                xy0 = V2(xt, tile_xy.y);
            } else {
                float x_clip = is_positive_slope ? tile_xy.x : tile_xy1.x;
                float yt = xy0.y + (xy1.y - xy0.y) * (x_clip - xy0.x) / (xy1.x - xy0.x);
                yt = clampf(yt, tile_xy.y + 1e-3f, tile_xy1.y);
                xy0 = V2(x_clip, yt);
            }
        }
        if (seg_within_line < count - 1u) {
            float z_next = floorf(a * ((float)seg_within_line + 1.0f) + b);
            if (z == z_next) {
                float xt = xy0.x + (xy1.x - xy0.x) * (tile_xy1.y - xy0.y) / (xy1.y - xy0.y);
                xt = clampf(xt, tile_xy.x + 1e-3f, tile_xy1.x);
                xy1 = V2(xt, tile_xy1.y);
            } else {
                float x_clip = is_positive_slope ? tile_xy1.x : tile_xy.x;
                float yt = xy0.y + (xy1.y - xy0.y) * (x_clip - xy0.x) / (xy1.x - xy0.x);
                yt = clampf(yt, tile_xy.y + 1e-3f, tile_xy1.y);
                xy1 = V2(x_clip, yt);
            }
        }
        float y_edge = 1e9f;
        v2 p0 = v2sub(xy0, tile_xy);
        v2 p1 = v2sub(xy1, tile_xy);
        const float EPSILON = 1e-6f;
        if (p0.x == 0.0f) {
            if (p1.x == 0.0f) {
                p0.x = EPSILON;
                if (p0.y == 0.0f) {
                    p1.x = EPSILON;
                    p1.y = 16.0f;
                } else {
                    p1.x = 2.0f * EPSILON;
                    p1.y = p0.y;
                }
            } else if (p0.y == 0.0f) {
                p0.x = EPSILON;
            } else {
                y_edge = p0.y;
            }
        } else if (p1.x == 0.0f) {
            if (p1.y == 0.0f) {
                p1.x = EPSILON;
            } else {
                y_edge = p1.y;
            }
        }
        if (p0.x == floorf(p0.x) && p0.x != 0.0f) p0.x -= EPSILON;
        if (p1.x == floorf(p1.x) && p1.x != 0.0f) p1.x -= EPSILON;
        if (!is_down) { v2 t = p0; p0 = p1; p1 = t; }
        Segment *s = &segments[seg_start + seg_within_slice];
        s->p0[0] = p0.x; s->p0[1] = p0.y; s->p1[0] = p1.x; s->p1[1] = p1.y; s->y_edge = y_edge; s->_pad = 0;
    }
}

/* ------------------------------------------------------------------------------------------
 * context / driver
 * ---------------------------------------------------------------------------------------- */
vbo_ctx *vbo_create(void) {
    vbo_ctx *c = calloc(1, sizeof(vbo_ctx));
    vec_init(&c->tag_monoids, sizeof(TagMonoid));
    vec_init(&c->path_bboxes, sizeof(PathBbox));
    vec_init(&c->lines, sizeof(LineSoup));
    vec_init(&c->draw_monoids, sizeof(DrawMonoid));
    vec_init(&c->info_bin_data, 4);
    vec_init(&c->clip_inp, sizeof(ClipInp));
    vec_init(&c->clip_bboxes, sizeof(Bbox4));
    vec_init(&c->draw_bboxes, sizeof(Bbox4));
    vec_init(&c->bin_headers, sizeof(BinHeader));
    vec_init(&c->paths, sizeof(PathRec));
    vec_init(&c->tiles, sizeof(Tile));
    vec_init(&c->seg_counts, sizeof(SegmentCount));
    vec_init(&c->segments, sizeof(Segment));
    vec_init(&c->ptcl, 4);
    vec_init(&c->blend_spill, 4);
    vec_init(&c->tile_counts, 4);
    c->threads = 1;
    return c;
}
void vbo_destroy(vbo_ctx *c) {
    if (!c) return;
    Vec *vs[] = {&c->tag_monoids, &c->path_bboxes, &c->lines, &c->draw_monoids, &c->info_bin_data, &c->clip_inp,
                 &c->clip_bboxes, &c->draw_bboxes, &c->bin_headers, &c->paths, &c->tiles, &c->seg_counts, &c->segments,
                 &c->ptcl, &c->blend_spill, &c->tile_counts};
    for (size_t i = 0; i < sizeof vs / sizeof vs[0]; i++) vec_free(vs[i]);
    free(c);
}
void vbo_set_threads(vbo_ctx *c, int n) { c->threads = n < 1 ? 1 : n; }

int vbo_bind(vbo_ctx *c, const uint32_t *scene, size_t scene_words, const vbo_layout *layout, const uint32_t *ramps,
             uint32_t n_ramps, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, const vbo_params *params) {
    c->scene = scene; c->scene_words = scene_words;
    c->ramps = ramps; c->n_ramps = n_ramps;
    c->atlas = atlas; c->atlas_w = atlas_w; c->atlas_h = atlas_h;
    c->params = *params;
    memset(&c->cfg, 0, sizeof c->cfg);
    c->cfg.width_in_tiles = (params->width + 15u) / 16u;
    c->cfg.height_in_tiles = (params->height + 15u) / 16u;
    c->cfg.target_width = params->width;
    c->cfg.target_height = params->height;
    c->cfg.base_color = params->base_color;
    c->cfg.layout = *layout;
    uint32_t hb = (c->cfg.height_in_tiles + 15u) / 16u;
    c->win_by0 = 0; c->win_by1 = hb;
    if (params->bin_row1 > params->bin_row0) {
        c->win_by0 = params->bin_row0 < hb ? params->bin_row0 : hb;
        c->win_by1 = params->bin_row1 < hb ? params->bin_row1 : hb;
    }
    c->win_ty0 = c->win_by0 * 16u;
    c->win_ty1 = c->win_by1 * 16u < c->cfg.height_in_tiles ? c->win_by1 * 16u : c->cfg.height_in_tiles;
    memset(&c->bump, 0, sizeof c->bump);
    c->tile_counts.n = 0; /* no counts of this scene until its path_count runs */
    c->lines_overridden = 0;
    return 0;
}

int vbo_run(vbo_ctx *c, int first, int last, uint8_t *out) {
    for (int s = first; s <= last; s++) {
        switch (s) {
        case VBO_STAGE_PATHTAG: stage_pathtag(c); break;
        case VBO_STAGE_FLATTEN: if (!c->lines_overridden) stage_flatten(c); break;
        case VBO_STAGE_DRAW: stage_draw(c); break;
        case VBO_STAGE_CLIP: stage_clip(c); break;
        case VBO_STAGE_BINNING: stage_binning(c); break;
        case VBO_STAGE_TILE_ALLOC: stage_tile_alloc(c); break;
        case VBO_STAGE_PATH_COUNT: stage_path_count(c); break;
        case VBO_STAGE_BACKDROP: stage_backdrop(c); break;
        case VBO_STAGE_COARSE: stage_coarse(c); break;
        case VBO_STAGE_PATH_TILING: stage_path_tiling(c); break;
        case VBO_STAGE_FINE:
            if (!out) return -1;
            if (vbo_fine(c, out) != 0) return -3;
            break;
        default: return -2;
        }
    }
    /* mirror the capacities actually used into the uniform, as the CUDA renderer does */
    c->cfg.lines_size = c->bump.lines;
    c->cfg.binning_size = c->bump.binning;
    c->cfg.tiles_size = c->bump.tile;
    c->cfg.seg_counts_size = c->bump.seg_counts;
    c->cfg.segments_size = c->bump.segments;
    c->cfg.blend_size = c->bump.blend;
    c->cfg.ptcl_size = (uint32_t)c->ptcl.n;
    return 0;
}

const void *vbo_buffer(vbo_ctx *c, const char *name, size_t *bytes) {
    struct { const char *n; Vec *v; } tab[] = {
        {"tag_monoids", &c->tag_monoids}, {"path_bboxes", &c->path_bboxes}, {"lines", &c->lines},
        {"draw_monoids", &c->draw_monoids}, {"info_bin_data", &c->info_bin_data}, {"clip_inp", &c->clip_inp},
        {"clip_bboxes", &c->clip_bboxes}, {"draw_bboxes", &c->draw_bboxes}, {"bin_headers", &c->bin_headers},
        {"paths", &c->paths}, {"tiles", &c->tiles}, {"seg_counts", &c->seg_counts}, {"segments", &c->segments},
        {"ptcl", &c->ptcl}, {"blend_spill", &c->blend_spill}, {"tile_counts", &c->tile_counts}};
    for (size_t i = 0; i < sizeof tab / sizeof tab[0]; i++)
        if (!strcmp(name, tab[i].n)) {
            *bytes = tab[i].v->n * tab[i].v->elem;
            return tab[i].v->p;
        }
    if (!strcmp(name, "bump")) { *bytes = sizeof c->bump; return &c->bump; }
    if (!strcmp(name, "config")) { *bytes = sizeof c->cfg; return &c->cfg; }
    *bytes = 0;
    return NULL;
}

int vbo_set_buffer(vbo_ctx *c, const char *name, const void *data, size_t bytes) {
    if (!strcmp(name, "lines")) {
        size_t n = bytes / sizeof(LineSoup);
        void *p = vec_resize(&c->lines, n);
        memcpy(p, data, n * sizeof(LineSoup));
        c->bump.lines = (uint32_t)n;
        c->lines_overridden = 1;
        return 0;
    }
    if (!strcmp(name, "path_bboxes")) {
        size_t n = bytes / sizeof(PathBbox);
        void *p = vec_resize(&c->path_bboxes, n);
        memcpy(p, data, n * sizeof(PathBbox));
        return 0;
    }
    /* fine's inputs, so that `fine` alone interprets exactly the buffers another implementation's fine read */
    if (!strcmp(name, "ptcl")) {
        size_t n = bytes / 4;
        memcpy(vec_resize(&c->ptcl, n), data, n * 4);
        c->cfg.ptcl_size = (uint32_t)n;
        return 0;
    }
    if (!strcmp(name, "segments")) {
        size_t n = bytes / sizeof(Segment);
        memcpy(vec_resize(&c->segments, n), data, n * sizeof(Segment));
        c->bump.segments = (uint32_t)n;
        c->cfg.segments_size = (uint32_t)n;
        return 0;
    }
    if (!strcmp(name, "info_bin_data")) {
        size_t n = bytes / 4;
        memcpy(vec_resize(&c->info_bin_data, n), data, n * 4);
        c->bump.binning = n > c->cfg.layout.bin_data_start ? (uint32_t)(n - c->cfg.layout.bin_data_start) : 0u;
        c->cfg.binning_size = c->bump.binning;
        return 0;
    }
    /* sizes the spill area from the caller's count (the blend offsets in a replayed ptcl were allocated against it): fine
     * writes its spilled blend-stack levels there, at each tile's blend offset */
    if (!strcmp(name, "blend_spill")) {
        size_t n = bytes / 4;
        memcpy(vec_resize(&c->blend_spill, n), data, n * 4);
        c->bump.blend = (uint32_t)n;
        c->cfg.blend_size = (uint32_t)n;
        return 0;
    }
    return -1;
}

int vbo_uses_libm(void) {
#ifdef VBO_LIBM
    return 1;
#else
    return 0;
#endif
}

float vbo_math(int fn, float a, float b) {
    switch (fn) {
    case 0: return M_SINF(a);
    case 1: return M_COSF(a);
    case 2: return M_ATAN2F(a, b);
    case 3: return M_ASINF(a);
    case 4: return M_ACOSF(a);
    case 5: return M_POW23(a);
    case 6: return M_EXPF(a);
    case 7: return M_POWF(a, b);
#ifndef VBO_LIBM
    case 8: return vb_cbrtf(a);
    case 9: return vb_logf(a);
#else
    case 8: return cbrtf(a);
    case 9: return logf(a);
#endif
    default: return 0.0f;
    }
}
