// k_flatten.cu -- curve flattening + stroke expansion to LineSoup, per-path bounding boxes.
//
// Reference: vello_shaders/shader/flatten.wgsl (Euler-spiral flatten :326-481, arcs :494-519,
// caps :521-545, joins :547-631, segment decode :683-766, main :831-923) and its CPU twin
// vello_shaders/src/cpu/{flatten,euler}.rs. Also folds in bbox_clear.wgsl.
//
// Design (differs from the WGSL on purpose; the pieces are described where they are defined below):
//  * The WGSL bump-allocates every line with a global atomicAdd, so the line order is a race. Here line order is
//    deterministic -- tag order, then emission order, i.e. the serial CPU shader's -- and independent of any atomic:
//    the tag pass (thread per TAG: k_flatten_lean, then k_flatten for the partitions that need the general path) emits
//    literal-line and job records plus per-warp counts, k_flatten_scan turns the counts into offsets, k_flatten_place
//    (thread per LINE) writes every line at its final position.
//  * Fast paths for line-tos (filled: one line; stroked: one line per side) behind guards that are derived in place,
//    property-tested on the CPU against the oracle and compared bit for bit on the GPU.
//  * With a stripe window set (multi-GPU), tags that cannot reach the window's rows are skipped.
//  * Transcendentals come from vb_detmath.h (IEEE-only) and the TU is compiled with -fmad=false,
//    so `lines` is bit-identical to the oracle's, and so is everything downstream.
// Algorithmic bytes: 1 B tag + 20/4 B monoid + <= 32 B coords per segment, 24 B per line out.
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include "vb_detmath.h"
#include "vb_device.cuh"
#include "vb_stages.h"

#ifndef FL_THREADS
#define FL_THREADS 256
#endif
#ifndef FL_MINB
#define FL_MINB 2
#endif

namespace cg = cooperative_groups;

struct fv2 { float x, y; };
__device__ __forceinline__ fv2 F2(float x, float y) { fv2 r; r.x = x; r.y = y; return r; }
__device__ __forceinline__ fv2 operator+(fv2 a, fv2 b) { return F2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ fv2 operator-(fv2 a, fv2 b) { return F2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ fv2 operator*(fv2 a, float s) { return F2(a.x * s, a.y * s); }
__device__ __forceinline__ float fdot(fv2 a, fv2 b) { return a.x * b.x + a.y * b.y; }
__device__ __forceinline__ float flen(fv2 a) { return sqrtf(a.x * a.x + a.y * a.y); }
__device__ __forceinline__ fv2 fnorm(fv2 a) { float l = flen(a); return F2(a.x / l, a.y / l); }
__device__ __forceinline__ bool feq(fv2 a, fv2 b) { return a.x == b.x && a.y == b.y; }

struct FXform { float m0, m1, m2, m3, tx, ty; };
__device__ __forceinline__ fv2 fx_apply(const FXform &t, fv2 p) { // flatten.wgsl:668-672 (explicit fma)
    return F2(fmaf(t.m0, p.x, fmaf(t.m2, p.y, t.tx)), fmaf(t.m1, p.x, fmaf(t.m3, p.y, t.ty)));
}

// One pass over the tags, then one pass over the LINES.
//  * k_flatten (thread per tag) runs the control flow of the reference -- subdivision into Euler segments, caps,
//    joins -- but does not evaluate long runs of lines itself: an Euler segment or arc of >= FL_DEFER_MIN lines
//    becomes a 96 B FlJob record ("these n lines, at tag-relative offset rel"). Short output (the one line of a
//    line-to, cap / join lines) is kept in a small shared-memory cache and leaves as 32 B FlLit records.
//  * k_flatten_scan turns per-warp line counts into final offsets (tag order == the serial CPU shader's order).
//  * k_flatten_place (thread per LINE) scatters the literals and expands the jobs, 32 jobs per warp with a
//    load-balanced lane <-> line mapping, so the cost of a frame no longer hangs on its slowest tag.
// Every point is a pure function of (job, i); whoever evaluates it gets the same bits.
#define FL_CACHE 6     // literal lines a thread keeps in shared memory
#define FL_DEFER_MIN 3 // runs of at least this many lines are deferred to k_flatten_place
#define FL_ARC_MAX 64  // arcs longer than this are emitted in place (line i costs i rotations when deferred)

struct FlLit { uint32_t tag_ix, rel, path_ix, pad; float x0, y0, x1, y1; }; // 32 B
struct FlJob {                                                             // 96 B = 6 x 16 B
    float p0x, p0y, p1x, p1y;      // Euler: chord end points (local space) | arc: begin, end (local space)
    float th0, k0, k1, ch;         // Euler: EulerParams                    | arc: centre.x, centre.y, cos, sin
    float noff, n, integral, int0; // Euler: normalized offset, float(n), integral, int0
    float a, b, lp0x, lp0y;        // Euler: a, b | both: start point of line 0, DEVICE space
    float tex, tey;                // Euler: t_end (local space)
    uint32_t tag_ix, rel;          // destination = offset of the tag + rel
    uint32_t path_ix, trans_ix, meta, pad;
};
static_assert(sizeof(FlLit) == 32 && sizeof(FlJob) == 96, "record layout");
#define FJ_N(m) ((m) & 0xffu)
#define FJ_ROBUST(m) (((m) >> 8) & 3u)
#define FJ_TEND 0x400u  // the last line ends at t_end exactly
#define FJ_NEG 0x800u   // negative offset: swap the end points of every line
#define FJ_IDENT 0x1000u // points are already in device space
#define FJ_ARC 0x2000u

struct FlCtx {
    FlLit *lits;
    FlJob *jobs;
    uint32_t lits_cap, jobs_cap;
    uint32_t *ctrs; // [0] literal records, [1] jobs
};

__device__ __forceinline__ uint32_t fl_alloc(uint32_t *ctr) { // one atomic per converged group of lanes
    cg::coalesced_group g = cg::coalesced_threads();
    uint32_t base = 0u;
    if (g.thread_rank() == 0u) base = atomicAdd(ctr, g.size());
    return g.shfl(base, 0) + g.thread_rank();
}

__device__ __noinline__ void fl_spill_line(const FlCtx c, uint32_t tag_ix, uint32_t rel, uint32_t path_ix, fv2 p0, fv2 p1) {
    const uint32_t slot = fl_alloc(c.ctrs); // literal beyond the shared-memory cache: rare
    if (slot < c.lits_cap) {
        uint4 *dst = reinterpret_cast<uint4 *>(c.lits + slot);
        dst[0] = make_uint4(tag_ix, rel, path_ix, 0u);
        dst[1] = make_uint4(__float_as_uint(p0.x), __float_as_uint(p0.y), __float_as_uint(p1.x), __float_as_uint(p1.y));
    }
}

// SPILL = false (k_flatten_lean): a tag never has more than FL_CACHE literal lines, so there is no overflow path.
template <bool SPILL>
struct FlatT {
    FlCtx c;
    uint32_t tag_ix, path_ix, trans_ix;
    uint32_t ix;   // lines of this tag so far
    uint32_t nlit; // of which literal (cached or spilled)
    float bx0, by0, bx1, by1; // bbox of the literal lines
    bool force;    // a job was deferred: the tag's bbox is known to be non-degenerate
    float4 *cache; // &cache[0][threadIdx.x], stride FL_THREADS
    uint32_t *cache_rel;
    __device__ __forceinline__ void write_line(fv2 p0, fv2 p1) { // device-space end points
        bx0 = fminf(bx0, fminf(p0.x, p1.x));
        by0 = fminf(by0, fminf(p0.y, p1.y));
        bx1 = fmaxf(bx1, fmaxf(p0.x, p1.x));
        by1 = fmaxf(by1, fmaxf(p0.y, p1.y));
        if (!SPILL || nlit < FL_CACHE) {
            cache[nlit * FL_THREADS] = make_float4(p0.x, p0.y, p1.x, p1.y);
            cache_rel[nlit * FL_THREADS] = ix;
        } else {
            fl_spill_line(c, tag_ix, ix, path_ix, p0, p1);
        }
        nlit++;
        ix++;
    }
    __device__ __forceinline__ void line_xf(fv2 p0, fv2 p1, const FXform &t) { write_line(fx_apply(t, p0), fx_apply(t, p1)); }
    __device__ __forceinline__ void push_job(FlJob &j, uint32_t n_lines) {
        j.tag_ix = tag_ix; j.rel = ix; j.path_ix = path_ix; j.trans_ix = trans_ix; j.pad = 0u;
        const uint32_t slot = fl_alloc(c.ctrs + 1);
        if (slot < c.jobs_cap) {
            float4 *dst = reinterpret_cast<float4 *>(c.jobs + slot);
            dst[0] = make_float4(j.p0x, j.p0y, j.p1x, j.p1y);
            dst[1] = make_float4(j.th0, j.k0, j.k1, j.ch);
            dst[2] = make_float4(j.noff, j.n, j.integral, j.int0);
            dst[3] = make_float4(j.a, j.b, j.lp0x, j.lp0y);
            dst[4] = make_float4(j.tex, j.tey, __uint_as_float(j.tag_ix), __uint_as_float(j.rel));
            dst[5] = make_float4(__uint_as_float(j.path_ix), __uint_as_float(j.trans_ix), __uint_as_float(j.meta), 0.f);
        }
        ix += n_lines;
        force = true;
    }
};
using Flat = FlatT<true>;

#define DERIV_THRESH 1e-6f
#define DERIV_THRESH_SQUARED (DERIV_THRESH * DERIV_THRESH)
#define DERIV_EPS 1e-6f
#define SUBDIV_LIMIT (1.0f / 65536.0f)
#define K1_THRESH 1e-3f
#define DIST_THRESH 1e-3f
#define TANGENT_THRESH 1e-6f

struct CubicParams { float th0, th1, chord_len, err; };
struct EulerParams { float th0, k0, k1, ch; };

__device__ CubicParams cubic_from_points_derivs(fv2 p0, fv2 p1, fv2 q0, fv2 q1, float dt) { // flatten.wgsl:94-133
    CubicParams r;
    fv2 chord = p1 - p0;
    float chord_squared = fdot(chord, chord);
    float chord_len = sqrtf(chord_squared);
    if (chord_squared < DERIV_THRESH_SQUARED) {
        float chord_err = sqrtf((9.f / 32.0f) * (fdot(q0, q0) + fdot(q1, q1))) * dt;
        r.th0 = 0.f; r.th1 = 0.f; r.chord_len = DERIV_THRESH; r.err = chord_err;
        return r;
    }
    float scale = dt / chord_squared;
    fv2 h0 = F2(q0.x * chord.x + q0.y * chord.y, q0.y * chord.x - q0.x * chord.y);
    float th0 = vb_atan2f(h0.y, h0.x);
    float d0 = flen(h0) * scale;
    fv2 h1 = F2(q1.x * chord.x + q1.y * chord.y, q1.x * chord.y - q1.y * chord.x);
    float th1 = vb_atan2f(h1.y, h1.x);
    float d1 = flen(h1) * scale;
    float s0, cth0, s1, cth1;
    vb_sincosf(th0, &s0, &cth0);
    vb_sincosf(th1, &s1, &cth1);
    float err = 2.0f;
    if (cth0 * cth1 >= 0.0f) {
        float e0 = (2.f / 3.f) / fmaxf(1.0f + cth0, 1e-9f);
        float e1 = (2.f / 3.f) / fmaxf(1.0f + cth1, 1e-9f);
        float s01 = cth0 * s1 + cth1 * s0;
        float amin = 0.15f * (2.f * e0 * s0 + 2.f * e1 * s1 - e0 * e1 * s01);
        float a = 0.15f * (2.f * d0 * s0 + 2.f * d1 * s1 - d0 * d1 * s01);
        float aerr = fabsf(a - amin);
        float symm = fabsf(th0 + th1);
        float asymm = fabsf(th0 - th1);
        float dist = flen(F2(d0 - e0, d1 - e1));
        float symm2 = symm * symm;
        float ctr = (4.625e-6f * symm * symm2 + 7.5e-3f * asymm) * symm2;
        float halo = (5e-3f * symm + 7e-2f * asymm) * dist;
        err = ctr + 1.55f * aerr + halo;
    }
    err *= chord_len;
    r.th0 = th0; r.th1 = th1; r.chord_len = chord_len; r.err = err;
    return r;
}

__device__ EulerParams es_params_from_angles(float th0, float th1) { // flatten.wgsl:135-161
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
__device__ __forceinline__ float es_eval_th(const EulerParams &p, float t) { return (p.k0 + 0.5f * p.k1 * (t - 1.0f)) * t - p.th0; }

__device__ fv2 integ_euler_10(float k0, float k1) { // flatten.wgsl:168-202
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
    return F2(u, v);
}
__device__ fv2 es_seg_eval_with_offset(fv2 p0, fv2 p1, const EulerParams &p, float t, float normalized_offset) {
    // es_params_eval_with_offset + es_params_eval (flatten.wgsl:204-231)
    float th = es_eval_th(p, t);
    float sth, cth;
    vb_sincosf(th, &sth, &cth);
    fv2 v = F2(normalized_offset * sth, normalized_offset * cth);
    float thm = es_eval_th(p, t * 0.5f);
    fv2 uv = integ_euler_10((p.k0 + p.k1 * (0.5f * t - 0.5f)) * t, p.k1 * t * t);
    float scale = t / p.ch;
    float sm, cm;
    vb_sincosf(thm, &sm, &cm);
    float s = scale * sm;
    float c = scale * cm;
    fv2 e = F2(uv.x * c - uv.y * s, -uv.y * c - uv.x * s);
    fv2 xy = e + v;
    fv2 chord = p1 - p0;
    return F2(p0.x + (chord.x * xy.x - chord.y * xy.y), p0.y + (chord.x * xy.y + chord.y * xy.x));
}
__device__ __forceinline__ float pow_1_5_signed(float x) { return x * sqrtf(fabsf(x)); }

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

__device__ float espc_int_approx(float x) { // flatten.wgsl:246-259
    float y = fabsf(x);
    float a;
    if (y < BREAK1) {
        a = vb_sinf(SIN_SCALE * y) * (1.0f / SIN_SCALE);
    } else if (y < BREAK2) {
        a = (sqrtf(8.0f) / 3.0f) * pow_1_5_signed(y - 1.0f) + FRAC_PI_4;
    } else {
        float qa = y < BREAK3 ? QUAD_A1 : QUAD_A2;
        float qb = y < BREAK3 ? QUAD_B1 : QUAD_B2;
        float qc = y < BREAK3 ? QUAD_C1 : QUAD_C2;
        a = (qa * y + qb) * y + qc;
    }
    return a * vb_signf(x);
}
__device__ float espc_int_inv_approx(float x) { // flatten.wgsl:261-275
    float y = fabsf(x);
    float a;
    if (y < 0.7010707591262915f) {
        a = vb_asinf(y * SIN_SCALE) * (1.0f / SIN_SCALE);
    } else if (y < 0.903249293595206f) {
        float b = y - FRAC_PI_4;
        float u = vb_pow_2_3(fabsf(b)) * vb_signf(b);
        a = u * CBRT_9_8 + 1.0f;
    } else {
        const float W1 = 0.5f * QUAD_B1 / QUAD_A1, V1 = 1.0f / QUAD_A1, U1 = W1 * W1 - QUAD_C1 / QUAD_A1;
        const float W2 = 0.5f * QUAD_B2 / QUAD_A2, V2_ = 1.0f / QUAD_A2, U2 = W2 * W2 - QUAD_C2 / QUAD_A2;
        bool first = y < 2.038857793595206f;
        float u = first ? U1 : U2, v = first ? V1 : V2_, w = first ? W1 : W2;
        a = sqrtf(u + v * y) - w;
    }
    return a * vb_signf(x);
}

struct PointDeriv { fv2 p, q; };
__device__ PointDeriv eval_cubic_and_deriv(fv2 p0, fv2 p1, fv2 p2, fv2 p3, float t) { // flatten.wgsl:282-290
    float m = 1.0f - t;
    float mm = m * m;
    float mt = m * t;
    float tt = t * t;
    PointDeriv r;
    float a = mm * m, b = 3.0f * mm, c = 3.0f * mt;
    r.p.x = p0.x * a + ((p1.x * b + p2.x * c) + p3.x * tt) * t;
    r.p.y = p0.y * a + ((p1.y * b + p2.y * c) + p3.y * tt) * t;
    float d = 2.0f * mt;
    r.q.x = ((p1.x - p0.x) * mm + (p2.x - p1.x) * d) + (p3.x - p2.x) * tt;
    r.q.y = ((p1.y - p0.y) * mm + (p2.y - p1.y) * d) + (p3.y - p2.y) * tt;
    return r;
}
__device__ fv2 cubic_start_tangent(fv2 p0, fv2 p1, fv2 p2, fv2 p3) {
    const float EPS = 1e-12f;
    fv2 d01 = p1 - p0, d02 = p2 - p0, d03 = p3 - p0;
    if (fdot(d01, d01) > EPS) return d01;
    if (fdot(d02, d02) > EPS) return d02;
    return d03;
}
__device__ fv2 cubic_end_tangent(fv2 p0, fv2 p1, fv2 p2, fv2 p3) {
    const float EPS = 1e-12f;
    fv2 d23 = p3 - p2, d13 = p3 - p1, d03 = p3 - p0;
    if (fdot(d23, d23) > EPS) return d23;
    if (fdot(d13, d13) > EPS) return d13;
    return d03;
}

struct CubicPoints { fv2 p0, p1, p2, p3; };

// End point (local space) of line i of an Euler-segment job: the body of the inner loop of flatten.wgsl:441-466.
__device__ fv2 fl_euler_point(const FlJob &j, uint32_t i) {
    if (i + 1u == FJ_N(j.meta) && (j.meta & FJ_TEND) != 0u) return F2(j.tex, j.tey);
    float t = (float)(i + 1u) / j.n;
    float s = t;
    const uint32_t robust = FJ_ROBUST(j.meta);
    if (robust != 1u) {
        float u = j.integral * t + j.int0;
        float inv;
        if (robust == 2u) inv = vb_pow_2_3(fabsf(u)) * vb_signf(u);
        else inv = espc_int_inv_approx(u);
        s = (inv - j.b) / j.a;
    }
    EulerParams ep = {j.th0, j.k0, j.k1, j.ch};
    return es_seg_eval_with_offset(F2(j.p0x, j.p0y), F2(j.p1x, j.p1y), ep, s, j.noff);
}

__device__ void flatten_euler(Flat &f, const CubicPoints &cubic, const FXform &local_to_device, float offset, fv2 start_p,
                              fv2 end_p) { // flatten.wgsl:326-481
    fv2 p0, p1, p2, p3;
    float scale;
    FXform transform;
    fv2 t_start = start_p, t_end = end_p;
    if (offset == 0.f) {
        p0 = fx_apply(local_to_device, cubic.p0);
        p1 = fx_apply(local_to_device, cubic.p1);
        p2 = fx_apply(local_to_device, cubic.p2);
        p3 = fx_apply(local_to_device, cubic.p3);
        scale = 1.f;
        transform.m0 = 1.f; transform.m1 = 0.f; transform.m2 = 0.f; transform.m3 = 1.f; transform.tx = 0.f; transform.ty = 0.f;
        t_start = p0;
        t_end = p3;
    } else {
        p0 = cubic.p0; p1 = cubic.p1; p2 = cubic.p2; p3 = cubic.p3;
        transform = local_to_device;
        scale = 0.5f * (flen(F2(transform.m0 + transform.m3, transform.m1 - transform.m2)) +
                        flen(F2(transform.m0 - transform.m3, transform.m1 + transform.m2)));
    }
    if (feq(p0, p1) && feq(p0, p2) && feq(p0, p3)) return;
    const float tol = 0.25f;
    uint32_t t0_u = 0u;
    float dt = 1.0f;
    fv2 last_p = p0;
    fv2 last_q = p1 - p0;
    if (fdot(last_q, last_q) < DERIV_THRESH_SQUARED) last_q = eval_cubic_and_deriv(p0, p1, p2, p3, DERIV_EPS).q;
    float last_t = 0.0f;
    fv2 lp0 = t_start;
    for (;;) {
        float t0 = (float)t0_u * dt;
        if (t0 == 1.0f) break;
        float t1 = t0 + dt;
        fv2 this_p0 = last_p;
        fv2 this_q0 = last_q;
        PointDeriv this_pq1 = eval_cubic_and_deriv(p0, p1, p2, p3, t1);
        if (fdot(this_pq1.q, this_pq1.q) < DERIV_THRESH_SQUARED) {
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
            float k0 = ep.k0 - 0.5f * ep.k1;
            float k1 = ep.k1;
            float normalized_offset = offset / cp.chord_len;
            float dist_scaled = normalized_offset * ep.ch;
            float scale_multiplier = sqrtf(0.125f * scale * cp.chord_len / (ep.ch * tol));
            float a = 0.0f, b = 0.0f, integral = 0.0f, int0 = 0.0f, n_frac;
            uint32_t robust = 0u;
            if (fabsf(k1) < K1_THRESH) {
                float k = ep.k0;
                n_frac = sqrtf(fabsf(k * (k * dist_scaled + 1.0f)));
                robust = 1u;
            } else if (fabsf(dist_scaled) < DIST_THRESH) {
                a = k1;
                b = k0;
                int0 = pow_1_5_signed(b);
                float int1 = pow_1_5_signed(a + b);
                integral = int1 - int0;
                n_frac = (2.f / 3.f) * integral / a;
                robust = 2u;
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
            float n = vb_clampf(ceilf(n_frac * scale_multiplier), 1.0f, 100.0f);
            uint32_t n_u = vb_f2u_sat(n);
            FlJob j;
            j.p0x = this_p0.x; j.p0y = this_p0.y; j.p1x = this_pq1.p.x; j.p1y = this_pq1.p.y;
            j.th0 = ep.th0; j.k0 = ep.k0; j.k1 = ep.k1; j.ch = ep.ch;
            j.noff = normalized_offset; j.n = n; j.integral = integral; j.int0 = int0;
            j.a = a; j.b = b;
            j.tex = t_end.x; j.tey = t_end.y;
            j.meta = n_u | (robust << 8) | (t1 == 1.0f ? FJ_TEND : 0u) | (offset >= 0.f ? 0u : FJ_NEG) | (offset == 0.f ? FJ_IDENT : 0u);
            bool deferred = false;
            if (n_u >= FL_DEFER_MIN) {
                // The tag's bbox is only published when it is non-degenerate (flatten.wgsl:916); deferring is safe
                // when the run itself already spans two distinct device-space points.
                const fv2 last = fl_euler_point(j, n_u - 1u);
                const fv2 d0 = fx_apply(transform, lp0), d1 = fx_apply(transform, last);
                if (!feq(d0, d1)) {
                    j.lp0x = d0.x; j.lp0y = d0.y;
                    f.push_job(j, n_u);
                    lp0 = last;
                    deferred = true;
                }
            }
            if (!deferred) {
                for (uint32_t i = 0u; i < n_u; i++) {
                    const fv2 lp1 = fl_euler_point(j, i);
                    fv2 l0 = offset >= 0.f ? lp0 : lp1;
                    fv2 l1 = offset >= 0.f ? lp1 : lp0;
                    f.line_xf(l0, l1, transform);
                    lp0 = lp1;
                }
            }
            last_p = this_pq1.p;
            last_q = this_pq1.q;
            last_t = t1;
            t0_u += 1u;
            uint32_t shift = (uint32_t)(__ffs((int)t0_u) - 1);
            t0_u >>= shift;
            dt *= (float)(1u << shift);
        } else {
            t0_u = t0_u * 2u;
            dt *= 0.5f;
        }
    }
}

// Device-space end point of line i of an arc job (flatten.wgsl:494-519): i + 1 rotations of the start radius.
__device__ fv2 fl_arc_point(const FlJob &j, uint32_t i, const FXform &t) {
    if (i + 1u == FJ_N(j.meta)) return fx_apply(t, F2(j.p1x, j.p1y));
    const fv2 center = F2(j.th0, j.k0);
    const float c = j.k1, s = j.ch;
    fv2 r = F2(j.p0x, j.p0y) - center;
    for (uint32_t k = 0u; k <= i; k++) r = F2(c * r.x + s * r.y, -s * r.x + c * r.y);
    return fx_apply(t, center + r);
}

// How an arc is flattened: its first point (device space), the rotation step, its line count and whether it is deferred.
struct ArcSteps {
    fv2 p0;
    float s, c;
    uint32_t n_lines;
    bool job;
};
__device__ __forceinline__ ArcSteps arc_steps(fv2 begin, fv2 end, fv2 center, float angle, const FXform &t) {
    ArcSteps a;
    a.p0 = fx_apply(t, begin);
    const float MIN_THETA = 0.0001f;
    const float tol = 0.25f;
    float radius = fmaxf(tol, flen(a.p0 - fx_apply(t, center)));
    float theta = fmaxf(MIN_THETA, 2.f * vb_acosf(1.f - tol / radius));
    a.n_lines = max(1u, vb_f2u_sat(ceilf(angle / theta)));
    vb_sincosf(theta, &a.s, &a.c);
    a.job = a.n_lines >= FL_DEFER_MIN && a.n_lines <= FL_ARC_MAX && !feq(a.p0, fx_apply(t, end));
    return a;
}

template <class F>
__device__ void flatten_arc(F &f, fv2 begin, fv2 end, fv2 center, float angle, const FXform &t) {
    const ArcSteps a = arc_steps(begin, end, center, angle, t);
    fv2 p0 = a.p0;
    fv2 r = begin - center;
    const uint32_t n_lines = a.n_lines;
    const float s = a.s, c = a.c;
    if (a.job) {
        FlJob j;
        j.p0x = begin.x; j.p0y = begin.y; j.p1x = end.x; j.p1y = end.y;
        j.th0 = center.x; j.k0 = center.y; j.k1 = c; j.ch = s;
        j.noff = 0.f; j.n = 0.f; j.integral = 0.f; j.int0 = 0.f; j.a = 0.f; j.b = 0.f;
        j.lp0x = p0.x; j.lp0y = p0.y; j.tex = 0.f; j.tey = 0.f;
        j.meta = n_lines | FJ_ARC;
        f.push_job(j, n_lines);
        return;
    }
    for (uint32_t i = 0u; i + 1u < n_lines; i++) {
        r = F2(c * r.x + s * r.y, -s * r.x + c * r.y);
        fv2 p1 = fx_apply(t, center + r);
        f.write_line(p0, p1);
        p0 = p1;
    }
    fv2 p1 = fx_apply(t, end);
    f.write_line(p0, p1);
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

// What a cap or join adds after the offset curves: at most one arc, then at most three straight lines (the slot
// order of the WGSL). Caps and joins only DESCRIBE their output here; flatten_tag emits it at a single site, so the
// instruction stream holds one copy of the arc / line writers (the fully inlined kernel was 133 KB of code and
// stalled on instruction fetch).
struct TailOps {
    bool have_arc;
    fv2 arc_begin, arc_end, arc_center;
    float arc_angle;
    uint32_t n_lines;
    fv2 a0, b0, a1, b1, a2, b2;
    __device__ __forceinline__ void line(fv2 a, fv2 b) {
        if (n_lines == 0u) { a0 = a; b0 = b; }
        else if (n_lines == 1u) { a1 = a; b1 = b; }
        else { a2 = a; b2 = b; }
        n_lines++;
    }
    __device__ __forceinline__ void arc(fv2 begin, fv2 end, fv2 center, float angle) {
        have_arc = true; arc_begin = begin; arc_end = end; arc_center = center; arc_angle = angle;
    }
};

__device__ __forceinline__ void draw_cap(TailOps &o, uint32_t cap_style, fv2 point, fv2 cap0, fv2 cap1, fv2 offset_tangent) {
    // flatten.wgsl:521-545
    if (cap_style == STYLE_FLAGS_CAP_ROUND) {
        o.arc(cap0, cap1, point, 3.1415927f);
        return;
    }
    fv2 start = cap0, end = cap1;
    if (cap_style == STYLE_FLAGS_CAP_SQUARE) {
        fv2 v = offset_tangent;
        fv2 p0 = start + v;
        fv2 p1 = end + v;
        o.line(p0, p1);
        o.line(start, p0);
        o.line(p1, end);
        return;
    }
    o.line(start, end);
}

__device__ __forceinline__ float f16_bits_to_f32(uint32_t h) { return __half2float(__ushort_as_half((unsigned short)(h & 0xffffu))); }

__device__ __forceinline__ void draw_join(TailOps &o, uint32_t style_flags, fv2 p0, fv2 tan_prev, fv2 tan_next, fv2 n_prev, fv2 n_next) {
    // flatten.wgsl:547-631
    fv2 front0 = p0 + n_prev;
    fv2 front1 = p0 + n_next;
    fv2 back0 = p0 - n_next;
    fv2 back1 = p0 - n_prev;
    float cr = tan_prev.x * tan_next.y - tan_prev.y * tan_next.x;
    float d = fdot(tan_prev, tan_next);
    switch (style_flags & STYLE_FLAGS_JOIN_MASK) {
    case STYLE_FLAGS_JOIN_BEVEL:
        o.line(front0, front1);
        o.line(back0, back1);
        break;
    case STYLE_FLAGS_JOIN_MITER: {
        float hyp = flen(F2(cr, d));
        float miter_limit = f16_bits_to_f32(style_flags & STYLE_MITER_LIMIT_MASK);
        if (2.f * hyp < (hyp + d) * miter_limit * miter_limit && fabsf(cr) > TANGENT_THRESH * TANGENT_THRESH) {
            bool is_backside = cr > 0.f;
            fv2 fp_last = is_backside ? back1 : front0;
            fv2 fp_this = is_backside ? back0 : front1;
            fv2 p = is_backside ? back0 : front0;
            fv2 v = fp_this - fp_last;
            float h = (tan_prev.x * v.y - tan_prev.y * v.x) / cr;
            fv2 miter_pt = fp_this - tan_next * h;
            o.line(p, miter_pt);
            if (is_backside) back0 = miter_pt; else front0 = miter_pt;
        }
        o.line(front0, front1);
        o.line(back0, back1);
        break;
    }
    case STYLE_FLAGS_JOIN_ROUND: {
        fv2 arc0, arc1, other0, other1;
        if (cr > 0.f) { arc0 = back0; arc1 = back1; other0 = front0; other1 = front1; }
        else { arc0 = front0; arc1 = front1; other0 = back0; other1 = back1; }
        o.arc(arc0, arc1, p0, fabsf(vb_atan2f(cr, d)));
        o.line(other0, other1);
        break;
    }
    default: break;
    }
}

struct PathTagData { uint32_t tag_byte; uint32_t trans_ix, pathseg_offset, style_ix, path_ix; };

__device__ __forceinline__ void fl_reduce_prefix(uint32_t w, uint32_t &trans, uint32_t &off, uint32_t &style, uint32_t &path) {
    // reduce_tag (shared/pathtag.wgsl:58-71) of the bytes below this thread's byte
    uint32_t point_count = w & 0x3030303u;
    trans = __popc(w & (0x20u * 0x1010101u));
    uint32_t n_points = point_count + ((w >> 2) & 0x1010101u);
    uint32_t a = n_points + (n_points & (((w >> 3) & 0x1010101u) * 15u));
    a += a >> 8;
    a += a >> 16;
    off = a & 0xffu;
    path = __popc(w & (0x10u * 0x1010101u));
    style = __popc(w & (0x40u * 0x1010101u)) * 2u;
}

__device__ PathTagData compute_tag_monoid(const VbConfig &cfg, const uint32_t *__restrict__ scene,
                                          const VbTagMonoid *__restrict__ tag_monoids, uint32_t ix) { // flatten.wgsl:683-699
    PathTagData r;
    uint32_t wi = ix >> 2;
    if (wi >= cfg.n_tag_words) { // one past the padded stream: an all-zero tag
        r.tag_byte = 0; r.trans_ix = 0; r.pathseg_offset = 0; r.style_ix = 0; r.path_ix = 0;
        return r;
    }
    uint32_t tag_word = __ldg(scene + cfg.layout.path_tag_base + wi);
    uint32_t shift = (ix & 3u) * 8u;
    uint32_t tr, of, st, pa;
    fl_reduce_prefix(tag_word & ((1u << shift) - 1u), tr, of, st, pa);
    VbTagMonoid base = tag_monoids[wi];
    r.tag_byte = (tag_word >> shift) & 0xffu;
    r.trans_ix = base.trans_ix + tr - 1u;
    r.pathseg_offset = base.pathseg_offset + of;
    r.style_ix = base.style_ix + st - 2u;
    r.path_ix = base.path_ix + pa;
    return r;
}

__device__ __forceinline__ fv2 read_f32_point(const VbConfig &cfg, const uint32_t *__restrict__ scene, uint32_t ix) {
    uint32_t b = cfg.layout.path_data_base + ix;
    return F2(__uint_as_float(vb_scene(scene, cfg, b)), __uint_as_float(vb_scene(scene, cfg, b + 1)));
}
__device__ __forceinline__ fv2 read_i16_point(const VbConfig &cfg, const uint32_t *__restrict__ scene, uint32_t ix) {
    uint32_t raw = vb_scene(scene, cfg, cfg.layout.path_data_base + ix);
    return F2((float)(((int32_t)(raw << 16)) >> 16), (float)(((int32_t)raw) >> 16));
}

__device__ CubicPoints read_path_segment(const VbConfig &cfg, const uint32_t *__restrict__ scene, const PathTagData &tag,
                                         bool is_stroke) { // flatten.wgsl:708-766
    fv2 p0, p1, p2 = F2(0, 0), p3 = F2(0, 0);
    uint32_t seg_type = tag.tag_byte & 3u;
    uint32_t off = tag.pathseg_offset;
    bool is_stroke_cap_marker = is_stroke && (tag.tag_byte & 4u) != 0u;
    bool is_open = seg_type == 2u;
    if (tag.tag_byte & 8u) {
        p0 = read_f32_point(cfg, scene, off);
        p1 = read_f32_point(cfg, scene, off + 2u);
        if (seg_type >= 2u) {
            p2 = read_f32_point(cfg, scene, off + 4u);
            if (seg_type == 3u) p3 = read_f32_point(cfg, scene, off + 6u);
        }
    } else {
        p0 = read_i16_point(cfg, scene, off);
        p1 = read_i16_point(cfg, scene, off + 1u);
        if (seg_type >= 2u) {
            p2 = read_i16_point(cfg, scene, off + 2u);
            if (seg_type == 3u) p3 = read_i16_point(cfg, scene, off + 3u);
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
        p2 = p3 + (p0 - p3) * third;
        p1 = p0 + (p3 - p0) * third;
    } else if (seg_type == 2u) {
        p3 = p2;
        p2 = p1 + (p2 - p1) * third;
        p1 = p1 + (p0 - p1) * third;
    }
    CubicPoints r = {p0, p1, p2, p3};
    return r;
}

// What one tag byte produces, decided before anything is emitted: 0, 1 or 2 offset curves for the Euler machinery (none
// when a line-to fast path applies), then the tail of a cap or join. Both tag kernels plan with this one function.
struct TagPlan {
    FXform transform;
    CubicPoints pts;
    bool is_stroke, fast_stroke; // fast_stroke: one line per side, (p0 + n_start, p3 + n_prev) and (p3 - n_prev, p0 - n_start)
    int n_sides;
    float offset;
    fv2 n_start, n_prev;
    TailOps tail;
};

// false: the tag emits nothing.
__device__ __forceinline__ bool plan_tag(TagPlan &plan, const VbConfig &cfg, const uint32_t *__restrict__ scene,
                                         const VbTagMonoid *__restrict__ tag_monoids, const PathTagData &tag, uint32_t ix,
                                         uint32_t style_flags) {
    uint32_t seg_type = tag.tag_byte & 3u;
    if (seg_type == 0u) return false;
    bool is_stroke = (style_flags & STYLE_FLAGS_STYLE) != 0u;
    FXform &transform = plan.transform;
    {
        uint32_t b = cfg.layout.transform_base + tag.trans_ix * 6u;
        transform.m0 = __uint_as_float(vb_scene(scene, cfg, b));
        transform.m1 = __uint_as_float(vb_scene(scene, cfg, b + 1));
        transform.m2 = __uint_as_float(vb_scene(scene, cfg, b + 2));
        transform.m3 = __uint_as_float(vb_scene(scene, cfg, b + 3));
        transform.tx = __uint_as_float(vb_scene(scene, cfg, b + 4));
        transform.ty = __uint_as_float(vb_scene(scene, cfg, b + 5));
    }
    CubicPoints &pts = plan.pts;
    pts = read_path_segment(cfg, scene, tag, is_stroke);
    if (cfg.win_cull != 0u) {
        // Stripe rendering (one bin-row window per GPU): everything this tag emits lies within R of the convex hull of
        // its control points (R = half width x max(miter limit, sqrt 2) for strokes), so a tag whose hull, grown by R
        // and one pixel, misses the window's rows cannot contribute a line, a backdrop or a bbox extent to them.
        // Rows are independent in this algorithm (backdrop runs left to right inside a tile row), so the rows of the
        // window still see every line that touches them: pixels are unchanged (test_stripes_equal_full_frame).
        const float y_0 = fmaf(transform.m1, pts.p0.x, fmaf(transform.m3, pts.p0.y, transform.ty));
        const float y_1 = fmaf(transform.m1, pts.p1.x, fmaf(transform.m3, pts.p1.y, transform.ty));
        const float y_2 = fmaf(transform.m1, pts.p2.x, fmaf(transform.m3, pts.p2.y, transform.ty));
        const float y_3 = fmaf(transform.m1, pts.p3.x, fmaf(transform.m3, pts.p3.y, transform.ty));
        float grow = 1.0f;
        if (is_stroke) {
            const float lw = __uint_as_float(vb_scene(scene, cfg, cfg.layout.style_base + tag.style_ix + 1u));
            const float lim = fmaxf(f16_bits_to_f32(style_flags & STYLE_MITER_LIMIT_MASK), 1.5f);
            grow += 0.5f * fabsf(lw) * lim * (fabsf(transform.m0) + fabsf(transform.m1) + fabsf(transform.m2) + fabsf(transform.m3));
        }
        const float lo = fminf(fminf(y_0, y_1), fminf(y_2, y_3)) - grow, hi = fmaxf(fmaxf(y_0, y_1), fmaxf(y_2, y_3)) + grow;
        if (hi < (float)(cfg.win_ty0 * VB_TILE_HEIGHT) || lo > (float)(cfg.win_ty1 * VB_TILE_HEIGHT)) return false; // NaN: kept
    }
    // the offset curves to flatten (0, 1 or 2 of them) and what follows them
    plan.is_stroke = is_stroke;
    int &n_sides = plan.n_sides;
    bool &fast_stroke = plan.fast_stroke;
    float &offset = plan.offset;
    fv2 &n_start = plan.n_start, &n_prev = plan.n_prev;
    TailOps &tail = plan.tail;
    n_sides = 0;
    fast_stroke = false;
    offset = 0.f;
    n_start = n_prev = F2(0.f, 0.f);
    tail.have_arc = false; tail.n_lines = 0u; tail.arc_angle = 0.f;
    tail.arc_begin = tail.arc_end = tail.arc_center = F2(0.f, 0.f);
    tail.a0 = tail.b0 = tail.a1 = tail.b1 = tail.a2 = tail.b2 = F2(0.f, 0.f);
    if (is_stroke) {
        float linewidth = __uint_as_float(vb_scene(scene, cfg, cfg.layout.style_base + tag.style_ix + 1u));
        offset = 0.5f * linewidth;
        bool is_open = seg_type != 1u;
        bool is_stroke_cap_marker = (tag.tag_byte & 4u) != 0u;
        if (is_stroke_cap_marker) {
            if (is_open) {
                fv2 tangent = pts.p3 - pts.p0;
                fv2 offset_tangent = fnorm(tangent) * offset;
                fv2 n = F2(-offset_tangent.y, offset_tangent.x);
                draw_cap(tail, (style_flags & STYLE_FLAGS_START_CAP_MASK) >> 2, pts.p0, pts.p0 - n, pts.p0 + n,
                         F2(-offset_tangent.x, -offset_tangent.y));
            }
        } else {
            PathTagData ntag = compute_tag_monoid(cfg, scene, tag_monoids, ix + 1u);
            CubicPoints npts = read_path_segment(cfg, scene, ntag, true);
            bool n_is_closed = (ntag.tag_byte & 3u) == 1u;
            bool n_is_marker = (ntag.tag_byte & 4u) != 0u;
            bool do_join = !n_is_marker || n_is_closed;
            fv2 n_tangent = npts.p3 - npts.p0;
            if (!n_is_marker) n_tangent = cubic_start_tangent(npts.p0, npts.p1, npts.p2, npts.p3);
            fv2 tan_start = cubic_start_tangent(pts.p0, pts.p1, pts.p2, pts.p3);
            if (fdot(tan_start, tan_start) < TANGENT_THRESH * TANGENT_THRESH) tan_start = F2(TANGENT_THRESH, 0.f);
            fv2 tan_prev = cubic_end_tangent(pts.p0, pts.p1, pts.p2, pts.p3);
            if (fdot(tan_prev, tan_prev) < TANGENT_THRESH * TANGENT_THRESH) tan_prev = F2(TANGENT_THRESH, 0.f);
            fv2 tan_next = n_tangent;
            if (fdot(tan_next, tan_next) < TANGENT_THRESH * TANGENT_THRESH) tan_next = F2(TANGENT_THRESH, 0.f);
            n_start = fnorm(F2(-tan_start.y, tan_start.x)) * offset;
            fv2 offset_tangent = fnorm(tan_prev) * offset;
            n_prev = F2(-offset_tangent.y, offset_tangent.x);
            fv2 tnn = fnorm(tan_next) * offset;
            fv2 n_next = F2(-tnn.y, tnn.x);
            n_sides = 2;
            // Fast path for a stroked line-to. The offset curves of a (degree-raised) line are the two parallel lines;
            // the general algorithm accepts the whole range at its first step and emits exactly one line per side,
            // (p0 + n_start, p3 + n_prev) and, end points swapped for the negative offset, (p3 - n_prev, p0 - n_start),
            // provided the rounding noise in the raised control points stays small against the chord:
            //   with u = ulp of the local coordinates, c = chord, s = scale: tangent-angle noise is ~3u/c, the error
            //   estimate O((3u/c)^2) c s and the line count ceil(sqrt(|k (k d + 1)| c s / 2)), |k| <~ 6u/c,
            //   d = offset / c; both stay below their thresholds when  u s <= 2^-8,  c >= 16 u  and  c^2 >= u * offset.
            // (u is taken as 2^-22 max|coord|, s as |m0|+|m1|+|m2|+|m3| -- both over-estimates.) Anything else, and any
            // NaN, takes the general path. tests/test_gpu_parity.py compares `lines` bit-for-bit with the oracle, which has
            // no such shortcut, on adversarial strokes (tiny segments, huge widths, large coordinates, odd transforms).
            if (seg_type == 1u && offset > 0.f) {
                const fv2 chord = pts.p3 - pts.p0;
                const float c2 = fdot(chord, chord);
                const float mag = fmaxf(fmaxf(fabsf(pts.p0.x), fabsf(pts.p0.y)), fmaxf(fabsf(pts.p3.x), fabsf(pts.p3.y)));
                const float s1 = fabsf(transform.m0) + fabsf(transform.m1) + fabsf(transform.m2) + fabsf(transform.m3);
                const float u = mag * 2.3841858e-07f; // 2^-22
                if (mag * s1 < 16384.0f && c2 >= 256.0f * u * u && c2 >= u * offset && c2 >= 1e-10f && c2 < 1e30f) fast_stroke = true;
            }
            if (do_join) draw_join(tail, style_flags, pts.p3, tan_prev, tan_next, n_prev, n_next);
            else draw_cap(tail, style_flags & STYLE_FLAGS_END_CAP_MASK, pts.p3, pts.p3 + n_prev, pts.p3 - n_prev, offset_tangent);
        }
    } else {
        // Fast path for a line-to in a fill (the bulk of map-like scenes). For a degree-raised line the general
        // algorithm provably accepts the whole range at the first step and emits exactly ONE line (p0', p3'):
        //  * err = O(angle^2) * chord, and the tangent angles of a degree-raised line are pure rounding noise
        //    (~3 ulp(coord)/chord); for chords shorter than that noise err <= 2 * chord <= 0.024 px  -> accepted;
        //  * n = ceil(n_frac * sqrt(chord/2)) with n_frac <= sqrt(|k0|) ~ sqrt(3 ulp/chord) -> n_frac*mult <= sqrt(1.5 ulp) < 1;
        //  * the single line runs from t_start = p0' to t_end = p3' (t1 == 1 exactly).
        // The bounds need ulp(coord) <= 2^-8, hence the |coord| < 65536 guard; anything else takes the general path.
        // tests/test_gpu_parity.py compares `lines` bit-for-bit with the oracle, which has no such shortcut.
        n_sides = 1;
        if (seg_type == 1u) {
            const fv2 q0 = fx_apply(transform, pts.p0), q1 = fx_apply(transform, pts.p1);
            const fv2 q2 = fx_apply(transform, pts.p2), q3 = fx_apply(transform, pts.p3);
            const float lim = 65536.0f;
            if (fabsf(q0.x) < lim && fabsf(q0.y) < lim && fabsf(q3.x) < lim && fabsf(q3.y) < lim && fabsf(q1.x) < lim && fabsf(q1.y) < lim &&
                fabsf(q2.x) < lim && fabsf(q2.y) < lim) {
                n_sides = 0;
                if (!(feq(q0, q1) && feq(q0, q2) && feq(q0, q3))) tail.line(q0, q3); // device space
            }
        }
    }
    if (fast_stroke) n_sides = 0;
    return true;
}

// A tag's output in order: the lines of the stroke fast path, the offset curves (flatten_tag only), the tail.
template <class F>
__device__ __forceinline__ void emit_fast_stroke(F &f, const TagPlan &p) {
    if (!p.fast_stroke) return;
    f.line_xf(p.pts.p0 + p.n_start, p.pts.p3 + p.n_prev, p.transform);
    f.line_xf(p.pts.p3 - p.n_prev, p.pts.p0 - p.n_start, p.transform);
}
template <class F>
__device__ __forceinline__ void emit_tail(F &f, const TagPlan &p) {
    const TailOps &tail = p.tail;
    if (tail.have_arc) flatten_arc(f, tail.arc_begin, tail.arc_end, tail.arc_center, tail.arc_angle, p.transform);
    // the fast-path line of a fill is in device space already; cap / join lines are in local space
    if (tail.n_lines > 0u)
        f.write_line(p.is_stroke ? fx_apply(p.transform, tail.a0) : tail.a0, p.is_stroke ? fx_apply(p.transform, tail.b0) : tail.b0);
    if (tail.n_lines > 1u) f.line_xf(tail.a1, tail.b1, p.transform);
    if (tail.n_lines > 2u) f.line_xf(tail.a2, tail.b2, p.transform);
}

// Everything one tag byte produces.
__device__ void flatten_tag(Flat &f, const VbConfig &cfg, const uint32_t *__restrict__ scene,
                            const VbTagMonoid *__restrict__ tag_monoids, const PathTagData &tag, uint32_t ix, uint32_t style_flags) {
    TagPlan p;
    if (!plan_tag(p, cfg, scene, tag_monoids, tag, ix, style_flags)) return;
    emit_fast_stroke(f, p);
#pragma unroll 1
    for (int side = 0; side < p.n_sides; side++) { // one copy of the Euler machinery in the instruction stream
        const bool fwd = side == 0;
        flatten_euler(f, p.pts, p.transform, fwd ? p.offset : -p.offset, fwd ? p.pts.p0 + p.n_start : p.pts.p0 - p.n_start,
                      fwd ? p.pts.p3 + p.n_prev : p.pts.p3 - p.n_prev);
    }
    emit_tail(f, p);
}

// bbox_clear.wgsl: path bboxes start at (+INT_MAX, -INT_MAX)
__global__ void k_bbox_clear(uint32_t n_paths, VbPathBbox *path_bboxes) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_paths) {
        VbPathBbox b;
        b.x0 = 0x7fffffff; b.y0 = 0x7fffffff; b.x1 = (int32_t)0x80000000; b.y1 = (int32_t)0x80000000;
        b.draw_flags = 0; b.trans_ix = 0;
        path_bboxes[i] = b;
    }
}

__device__ __forceinline__ int fl_floor_i(float v) { return v != v ? 0x7fffffff : vb_f2i_sat(floorf(v)); }
__device__ __forceinline__ int fl_ceil_i(float v) { return v != v ? (int)0x80000000 : vb_f2i_sat(ceilf(v)); }

// Per-partition prologue of both tag kernels: this lane's tag and style word, the draw flags / transform of the path it
// opens; then an empty Flat over the block's shared-memory line cache.
__device__ __forceinline__ void fl_load_tag(PathTagData &tag, uint32_t &style_flags, const VbConfig &cfg, const uint32_t *__restrict__ scene,
                                            const VbTagMonoid *__restrict__ tag_monoids, VbPathBbox *path_bboxes, uint32_t ix) {
    const uint32_t n_tags = cfg.n_tag_words * 4u;
    const uint32_t n_paths = cfg.layout.n_paths;
    tag.tag_byte = 0; tag.trans_ix = 0; tag.pathseg_offset = 0; tag.style_ix = 0; tag.path_ix = 0;
    style_flags = 0;
    if (ix < n_tags) {
        tag = compute_tag_monoid(cfg, scene, tag_monoids, ix);
        style_flags = vb_scene(scene, cfg, cfg.layout.style_base + tag.style_ix);
        if ((tag.tag_byte & 0x10u) != 0u && tag.path_ix < n_paths) {
            path_bboxes[tag.path_ix].draw_flags = (style_flags & STYLE_FLAGS_FILL) == 0u ? 0u : 1u;
            path_bboxes[tag.path_ix].trans_ix = tag.trans_ix;
        }
    }
}
template <class F>
__device__ __forceinline__ void fl_flat_init(F &f, const FlCtx &ctx, const PathTagData &tag, uint32_t ix, float4 *cache, uint32_t *cache_rel) {
    f.c = ctx;
    f.tag_ix = ix; f.path_ix = tag.path_ix; f.trans_ix = tag.trans_ix;
    f.ix = 0u; f.nlit = 0u; f.force = false;
    f.bx0 = 1e31f; f.by0 = 1e31f; f.bx1 = -1e31f; f.by1 = -1e31f;
    f.cache = cache;
    f.cache_rel = cache_rel;
}

// Per-partition epilogue of both tag kernels: per-warp line count, per-tag offset inside its warp's block, the cached
// literal records, and the bbox contribution of the literal lines.
template <class F>
__device__ __forceinline__ void fl_tag_end(F &f, const VbConfig &cfg, VbPathBbox *path_bboxes, const FlCtx &ctx, uint32_t *part_count,
                                           uint32_t *tag_off) {
    const uint32_t ix = f.tag_ix, path_ix = f.path_ix, part = ix >> 5, lane = ix & 31u;
    const uint32_t n_paths = cfg.layout.n_paths;
    __syncwarp();
    const uint32_t incl = vb_warp_incl_scan(f.ix);
    if (lane == 31u) part_count[part] = incl;
    tag_off[ix] = incl - f.ix;
    const uint32_t ncache = min(f.nlit, (uint32_t)FL_CACHE);
    const uint32_t lincl = vb_warp_incl_scan(ncache);
    const uint32_t ltotal = __shfl_sync(VB_FULL, lincl, 31);
    uint32_t lbase = 0u;
    if (lane == 31u && ltotal != 0u) lbase = atomicAdd(ctx.ctrs, ltotal);
    lbase = __shfl_sync(VB_FULL, lbase, 31);
    // The warp's literal records are one range [lbase, lbase + ltotal), lane i's ncache records after lane i-1's. They are
    // written lane-strided, record j of the range by lane j % 32 from its owner's cache, so that a warp's stores cover
    // consecutive 32 B records (each lane writing its own records made every store a scatter of partial sectors).
    const uint32_t lexcl = lincl - ncache;
    const float4 *wcache = f.cache - lane;
    const uint32_t *wrel = f.cache_rel - lane;
    for (uint32_t b = 0u; b < ltotal; b += 32u) {
        const uint32_t j = b + lane;
        uint32_t o = 0u; // owner: the number of lanes whose records all lie before j
#pragma unroll
        for (uint32_t step = 16u; step > 0u; step >>= 1)
            if (__shfl_sync(VB_FULL, lincl, o + step - 1u) <= j) o += step;
        const uint32_t k = j - __shfl_sync(VB_FULL, lexcl, o);
        const uint32_t o_path = __shfl_sync(VB_FULL, path_ix, o);
        const uint32_t slot = lbase + j;
        if (j < ltotal && slot < ctx.lits_cap) {
            const float4 l = wcache[k * FL_THREADS + o];
            uint4 *dst = reinterpret_cast<uint4 *>(ctx.lits + slot);
            dst[0] = make_uint4(ix - lane + o, wrel[k * FL_THREADS + o], o_path, 0u);
            dst[1] = make_uint4(__float_as_uint(l.x), __float_as_uint(l.y), __float_as_uint(l.z), __float_as_uint(l.w));
        }
    }
    // bbox: consecutive tags mostly belong to the same path, so reduce across the lanes of a path first (floor / ceil
    // commute with min / max) and issue one set of atomics per (warp, path) instead of one per tag
    const bool pub = f.nlit != 0u && (f.force || f.bx1 > f.bx0 || f.by1 > f.by0) && path_ix < n_paths;
    const uint32_t pubmask = __ballot_sync(VB_FULL, pub);
    if (pub) {
        int x0 = fl_floor_i(f.bx0), y0 = fl_floor_i(f.by0), x1 = fl_ceil_i(f.bx1), y1 = fl_ceil_i(f.by1);
        const uint32_t peers = __match_any_sync(pubmask, path_ix);
        x0 = __reduce_min_sync(peers, x0);
        y0 = __reduce_min_sync(peers, y0);
        x1 = __reduce_max_sync(peers, x1);
        y1 = __reduce_max_sync(peers, y1);
        if (lane == (uint32_t)(__ffs((int)peers) - 1)) {
            VbPathBbox *o = path_bboxes + path_ix;
            atomicMin(&o->x0, x0);
            atomicMin(&o->y0, y0);
            atomicMax(&o->x1, x1);
            atomicMax(&o->y1, y1);
        }
    }
}

// A: the tag pass, thread per tag, warp per partition of 32 tags. It is split by what the tags need, because the general
// path (Euler subdivision) needs 128 registers and most partitions of a map-like scene need none of it:
//  * k_flatten_lean runs every partition [part_base, part_end) -- all of them, or this GPU's share of a frame whose
//    flatten is sharded by tag range (k_exchange.cu); every array is indexed by the GLOBAL partition / tag. A partition
//    whose tags all take a line-to fast path or need no lines, and whose caps and joins are straight or round arcs that
//    are deferred or have at most 2 lines, is finished here (at most 5 literal lines per tag -- 2 + 3 straight, or
//    2 + 2 + 1 with an arc -- so all of them stay in the shared-memory cache).
//    Any other partition (a curve, a failed fast-path guard, an arc emitted in place) is left untouched and appended to
//    a work list.
//  * k_flatten runs the partitions of the work list with the general code.
// Both plan a tag with plan_tag and emit its lines through the same functions, so a partition's outputs are the same
// bits whichever kernel ran it.
#ifndef FL_LEAN_MINB
#define FL_LEAN_MINB 4
#endif

__global__ void __launch_bounds__(FL_THREADS, FL_LEAN_MINB)
k_flatten_lean(VbConfig cfg, const uint32_t *__restrict__ scene, const VbTagMonoid *__restrict__ tag_monoids, VbPathBbox *path_bboxes,
               FlCtx ctx, uint32_t *part_count, uint32_t *tag_off, uint32_t *work, uint32_t part_base, uint32_t part_end) {
    const uint32_t lane = vb_lane();
    const uint32_t part = part_base + blockIdx.x * (FL_THREADS / 32) + (threadIdx.x >> 5);
    if (part >= part_end) return;
    const uint32_t ix = part * 32u + lane;
    __shared__ float4 sh_cache[FL_CACHE][FL_THREADS];
    __shared__ uint32_t sh_rel[FL_CACHE][FL_THREADS];
    PathTagData tag;
    uint32_t style_flags;
    fl_load_tag(tag, style_flags, cfg, scene, tag_monoids, path_bboxes, ix);
    TagPlan p;
    const bool emits = plan_tag(p, cfg, scene, tag_monoids, tag, ix, style_flags);
    bool general = emits && p.n_sides != 0;
    if (emits && !general && p.tail.have_arc) {
        const ArcSteps a = arc_steps(p.tail.arc_begin, p.tail.arc_end, p.tail.arc_center, p.tail.arc_angle, p.transform);
        general = !a.job && a.n_lines > 2u;
    }
    if (__any_sync(VB_FULL, general)) {
        if (lane == 0u) work[atomicAdd(ctx.ctrs + 2, 1u)] = part;
        return;
    }
    FlatT<false> f;
    fl_flat_init(f, ctx, tag, ix, &sh_cache[0][threadIdx.x], &sh_rel[0][threadIdx.x]);
    if (emits) {
        emit_fast_stroke(f, p);
        emit_tail(f, p);
    }
    fl_tag_end(f, cfg, path_bboxes, ctx, part_count, tag_off);
}

// Outputs as k_flatten_lean's, plus the job records. The grid covers every partition the lean kernel could have left;
// the number it did leave is read on the device (frames are replayed as CUDA graphs). (History: a single-pass look-back
// kernel was gated by the slowest tag in flight; a count+emit kernel computed long tags twice and its 200 KB of code
// thrashed the instruction cache.)
__global__ void __launch_bounds__(FL_THREADS, FL_MINB)
k_flatten(VbConfig cfg, const uint32_t *__restrict__ scene, const VbTagMonoid *__restrict__ tag_monoids,
          VbPathBbox *path_bboxes, FlCtx ctx, uint32_t *part_count, uint32_t *tag_off, const uint32_t *__restrict__ work) {
    const uint32_t lane = vb_lane();
    const uint32_t slot = blockIdx.x * (FL_THREADS / 32) + (threadIdx.x >> 5);
    if (slot >= ctx.ctrs[2]) return;
    const uint32_t part = work[slot];
    const uint32_t ix = part * 32u + lane;
    __shared__ float4 sh_cache[FL_CACHE][FL_THREADS];
    __shared__ uint32_t sh_rel[FL_CACHE][FL_THREADS];
    PathTagData tag;
    uint32_t style_flags;
    fl_load_tag(tag, style_flags, cfg, scene, tag_monoids, path_bboxes, ix);
    Flat f;
    fl_flat_init(f, ctx, tag, ix, &sh_cache[0][threadIdx.x], &sh_rel[0][threadIdx.x]);
    flatten_tag(f, cfg, scene, tag_monoids, tag, ix, style_flags);
    fl_tag_end(f, cfg, path_bboxes, ctx, part_count, tag_off);
}

// B: exclusive scan of part_count -> destination offsets; publishes bump.lines. One CTA per 8192 partitions (8 values per
// thread, 128-bit accesses); the carry between CTAs is the single-pass look-back of vb_device.cuh (round 1 walked the whole
// array with ONE CTA, on the critical path of every frame and of every rank of a multi-GPU frame).
#define FS_THREADS 1024
#define FS_PER_THREAD 8
static_assert(FS_PER_THREAD == 8, "k_flatten_scan is written for 8 values per thread");
__global__ void __launch_bounds__(FS_THREADS)
k_flatten_scan(VbConfig cfg, uint32_t n_parts, const uint32_t *__restrict__ part_count, uint32_t *part_dst, VbBump *bump, uint32_t *lb_mem,
               uint32_t n_blocks) {
    __shared__ uint32_t sh_scan[FS_THREADS / 32 + 2];
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_carry;
    const VbLookback lb = vb_lookback_view(lb_mem, n_blocks, 1);
    const uint32_t blk = vb_take_ticket(lb, &sh_ticket);
    if (blk >= n_blocks) return;
    const uint32_t i0 = blk * (FS_THREADS * FS_PER_THREAD) + threadIdx.x * FS_PER_THREAD;
    uint32_t v[FS_PER_THREAD], sum = 0u;
    if (i0 + FS_PER_THREAD <= n_parts) { // two 128-bit loads (the arrays are 16-byte aligned, i0 is a multiple of 8)
        const uint4 a = *reinterpret_cast<const uint4 *>(part_count + i0);
        const uint4 b = *reinterpret_cast<const uint4 *>(part_count + i0 + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int k = 0; k < FS_PER_THREAD; k++) v[k] = i0 + k < n_parts ? part_count[i0 + k] : 0u;
    }
#pragma unroll
    for (int k = 0; k < FS_PER_THREAD; k++) sum += v[k];
    uint32_t total;
    const uint32_t ex = vb_block_excl_scan(sum, sh_scan, &total);
    if (threadIdx.x < 32u) {
        uint32_t agg[1] = {total}, excl[1];
        vb_lookback<1>(lb, blk, agg, excl);
        if (threadIdx.x == 0u) sh_carry = excl[0];
    }
    __syncthreads();
    const uint32_t carry = sh_carry;
    uint32_t run = carry + ex;
    if (i0 + FS_PER_THREAD <= n_parts) {
        uint4 a, b;
        a.x = run; a.y = a.x + v[0]; a.z = a.y + v[1]; a.w = a.z + v[2];
        b.x = a.w + v[3]; b.y = b.x + v[4]; b.z = b.y + v[5]; b.w = b.z + v[6];
        *reinterpret_cast<uint4 *>(part_dst + i0) = a;
        *reinterpret_cast<uint4 *>(part_dst + i0 + 4) = b;
    } else {
#pragma unroll
        for (int k = 0; k < FS_PER_THREAD; k++) {
            if (i0 + k < n_parts) part_dst[i0 + k] = run;
            run += v[k];
        }
    }
    if (blk == n_blocks - 1u && threadIdx.x == 0u) { // the block holding the end of the array knows the grand total
        const uint32_t lines = carry + total;
        bump->lines = lines;
        if (lines > cfg.lines_size) atomicOr(&bump->failed, VB_STAGE_FLATTEN);
    }
}

// C: thread per LINE. Phase 1 scatters the literal records; phase 2 expands the jobs, 32 per warp: the warp scans the
// jobs' line counts and walks the concatenated line range 32 lines at a time, so lanes stay busy whatever the mix of
// job sizes. A line's start point is its predecessor's end point: taken from the neighbouring lane when that lane
// holds the predecessor, recomputed otherwise (same function, same bits).
#define FP_THREADS 256
#define FP_WARPS (FP_THREADS / 32)

__global__ void __launch_bounds__(FP_THREADS)
k_flatten_place(VbConfig cfg, const uint32_t *__restrict__ scene, FlCtx ctx, const uint32_t *__restrict__ part_dst,
                const uint32_t *__restrict__ tag_off, VbPathBbox *path_bboxes, VbLineSoup *lines) {
    const uint32_t n_lit = min(ctx.ctrs[0], ctx.lits_cap);
    const uint32_t n_job = min(ctx.ctrs[1], ctx.jobs_cap);
    const uint32_t n_paths = cfg.layout.n_paths;
    for (uint32_t i = blockIdx.x * FP_THREADS + threadIdx.x; i < n_lit; i += gridDim.x * FP_THREADS) {
        const uint4 *src = reinterpret_cast<const uint4 *>(ctx.lits + i);
        const uint4 h = src[0], l = src[1];
        const uint32_t dst = part_dst[h.x >> 5] + tag_off[h.x] + h.y;
        if (dst < cfg.lines_size) {
            uint2 *d = reinterpret_cast<uint2 *>(lines + dst);
            d[0] = make_uint2(h.z, 0u);
            d[1] = make_uint2(l.x, l.y);
            d[2] = make_uint2(l.z, l.w);
        }
    }
    __shared__ float4 sh_job[FP_WARPS][6][32];
    __shared__ uint32_t sh_excl[FP_WARPS][32];
    __shared__ uint32_t sh_dst[FP_WARPS][32];
    const uint32_t lane = vb_lane(), w = threadIdx.x >> 5;
    const uint32_t n_batches = (n_job + 31u) / 32u;
    for (uint32_t batch = blockIdx.x * FP_WARPS + w; batch < n_batches; batch += gridDim.x * FP_WARPS) {
        const uint32_t jix = batch * 32u + lane;
        uint32_t n_l = 0u;
        if (jix < n_job) {
            const float4 *src = reinterpret_cast<const float4 *>(ctx.jobs + jix);
            float4 r4 = src[4], r5 = src[5];
#pragma unroll
            for (int k = 0; k < 4; k++) sh_job[w][k][lane] = src[k];
            sh_job[w][4][lane] = r4;
            sh_job[w][5][lane] = r5;
            n_l = FJ_N(__float_as_uint(r5.z));
            const uint32_t tix = __float_as_uint(r4.z);
            sh_dst[w][lane] = part_dst[tix >> 5] + tag_off[tix] + __float_as_uint(r4.w);
        }
        const uint32_t incl = vb_warp_incl_scan(n_l);
        const uint32_t total = __shfl_sync(VB_FULL, incl, 31);
        sh_excl[w][lane] = jix < n_job ? incl - n_l : 0xffffffffu;
        __syncwarp();
        for (uint32_t base = 0u; base < total; base += 32u) {
            const uint32_t l = base + lane;
            const bool act = l < total;
            const uint32_t actmask = __ballot_sync(VB_FULL, act);
            uint32_t k = 0u, i = 0u, meta = 0u, path_ix = 0u;
            fv2 q1 = F2(0.f, 0.f);
            FlJob j;
            FXform t;
            if (act) {
#pragma unroll
                for (uint32_t step = 16u; step > 0u; step >>= 1)
                    if (sh_excl[w][k + step] <= l) k += step;
                i = l - sh_excl[w][k];
                const float4 a0 = sh_job[w][0][k], a1 = sh_job[w][1][k], a2 = sh_job[w][2][k], a3 = sh_job[w][3][k], a4 = sh_job[w][4][k],
                             a5 = sh_job[w][5][k];
                j.p0x = a0.x; j.p0y = a0.y; j.p1x = a0.z; j.p1y = a0.w;
                j.th0 = a1.x; j.k0 = a1.y; j.k1 = a1.z; j.ch = a1.w;
                j.noff = a2.x; j.n = a2.y; j.integral = a2.z; j.int0 = a2.w;
                j.a = a3.x; j.b = a3.y; j.lp0x = a3.z; j.lp0y = a3.w;
                j.tex = a4.x; j.tey = a4.y;
                path_ix = __float_as_uint(a5.x);
                j.trans_ix = __float_as_uint(a5.y);
                meta = j.meta = __float_as_uint(a5.z);
                if (meta & FJ_IDENT) {
                    t.m0 = 1.f; t.m1 = 0.f; t.m2 = 0.f; t.m3 = 1.f; t.tx = 0.f; t.ty = 0.f;
                } else {
                    const uint32_t b = cfg.layout.transform_base + j.trans_ix * 6u;
                    t.m0 = __uint_as_float(vb_scene(scene, cfg, b));
                    t.m1 = __uint_as_float(vb_scene(scene, cfg, b + 1));
                    t.m2 = __uint_as_float(vb_scene(scene, cfg, b + 2));
                    t.m3 = __uint_as_float(vb_scene(scene, cfg, b + 3));
                    t.tx = __uint_as_float(vb_scene(scene, cfg, b + 4));
                    t.ty = __uint_as_float(vb_scene(scene, cfg, b + 5));
                }
                q1 = (meta & FJ_ARC) ? fl_arc_point(j, i, t) : fx_apply(t, fl_euler_point(j, i));
            }
            fv2 q0;
            q0.x = __shfl_up_sync(VB_FULL, q1.x, 1);
            q0.y = __shfl_up_sync(VB_FULL, q1.y, 1);
            if (act) {
                if (i == 0u) q0 = F2(j.lp0x, j.lp0y);
                else if (lane == 0u) q0 = (meta & FJ_ARC) ? fl_arc_point(j, i - 1u, t) : fx_apply(t, fl_euler_point(j, i - 1u));
                const fv2 l0 = (meta & FJ_NEG) ? q1 : q0, l1 = (meta & FJ_NEG) ? q0 : q1;
                const uint32_t dst = sh_dst[w][k] + i;
                if (dst < cfg.lines_size) {
                    uint2 *d = reinterpret_cast<uint2 *>(lines + dst);
                    d[0] = make_uint2(path_ix, 0u);
                    d[1] = make_uint2(__float_as_uint(l0.x), __float_as_uint(l0.y));
                    d[2] = make_uint2(__float_as_uint(l1.x), __float_as_uint(l1.y));
                }
                // bbox: floor / ceil commute with min / max, so reduce the integers across the lanes of a path
                int x0 = fl_floor_i(fminf(q0.x, q1.x)), y0 = fl_floor_i(fminf(q0.y, q1.y));
                int x1 = fl_ceil_i(fmaxf(q0.x, q1.x)), y1 = fl_ceil_i(fmaxf(q0.y, q1.y));
                const uint32_t peers = __match_any_sync(actmask, path_ix);
                x0 = __reduce_min_sync(peers, x0);
                y0 = __reduce_min_sync(peers, y0);
                x1 = __reduce_max_sync(peers, x1);
                y1 = __reduce_max_sync(peers, y1);
                if (lane == (uint32_t)(__ffs((int)peers) - 1) && path_ix < n_paths) {
                    VbPathBbox *o = path_bboxes + path_ix;
                    atomicMin(&o->x0, x0);
                    atomicMin(&o->y0, y0);
                    atomicMax(&o->x1, x1);
                    atomicMax(&o->y1, y1);
                }
            }
        }
        __syncwarp();
    }
}

extern "C" uint32_t vb_launch_flatten(const VbConfig &cfg, const VbFrameBufs &b, bool clear_bboxes, uint32_t part_base, uint32_t part_end,
                                      cudaStream_t st) {
    const uint32_t n_paths = cfg.layout.n_paths, n_parts = b.parts_flatten;
    uint32_t launches = 0;
    const uint32_t *scene = b.scene;
    const VbTagMonoid *tag_monoids = b.tag_monoids;
    VbPathBbox *path_bboxes = b.path_bboxes;
    // whole frames reset the boxes in k_frame_init (vb_api.cu); a stage range that starts later does it here
    if (n_paths && clear_bboxes) {
        k_bbox_clear<<<(n_paths + 255) / 256, 256, 0, st>>>(n_paths, path_bboxes);
        launches++;
    }
    if (n_parts) {
        const size_t np4 = ((size_t)n_parts + 3u) & ~(size_t)3u; // 16-byte aligned sub-arrays (k_flatten_scan uses 128-bit accesses)
        uint32_t *part_mem = b.flatten_parts; // vb_flatten_part_words
        uint32_t *part_count = part_mem, *part_dst = part_mem + np4, *tag_off = part_mem + 2 * np4, *work = part_mem + 34 * np4;
        FlCtx ctx;
        ctx.lits = b.line_scratch;
        ctx.jobs = b.flatten_jobs;
        ctx.lits_cap = cfg.lines_size;
        ctx.jobs_cap = cfg.lines_size / FL_DEFER_MIN + 1u;
        ctx.ctrs = b.lb_flatten;
        const uint32_t warps_per_cta = FL_THREADS / 32;
        if (part_end > n_parts) part_end = n_parts;
        if (part_base >= part_end) { // an empty share still has to publish bump.lines = 0
            part_base = part_end = 0u;
        }
        const uint32_t n_own = part_end - part_base; // part_base is a multiple of 8: the scan's 128-bit accesses stay aligned
        if (n_own) {
            const uint32_t grid = (n_own + warps_per_cta - 1) / warps_per_cta;
            k_flatten_lean<<<grid, FL_THREADS, 0, st>>>(cfg, scene, tag_monoids, path_bboxes, ctx, part_count, tag_off, work, part_base,
                                                        part_end);
            k_flatten<<<grid, FL_THREADS, 0, st>>>(cfg, scene, tag_monoids, path_bboxes, ctx, part_count, tag_off, work);
            launches += 2;
        }
        const uint32_t n_blocks = n_own ? (n_own + FS_THREADS * FS_PER_THREAD - 1u) / (FS_THREADS * FS_PER_THREAD) : 1u;
        k_flatten_scan<<<n_blocks, FS_THREADS, 0, st>>>(cfg, n_own, part_count + part_base, part_dst + part_base, b.bump(), ctx.ctrs + 4, n_blocks);
        k_flatten_place<<<(uint32_t)b.sm_count * 4u, FP_THREADS, 0, st>>>(cfg, scene, ctx, part_dst, tag_off, path_bboxes, b.lines);
        launches += 2;
    }
    return launches;
}
extern "C" uint32_t vb_flatten_parts(uint32_t n_tag_words) { return (n_tag_words * 4u + 31u) / 32u; }
// part_mem: part_count, part_dst (one word per partition each), tag_off (32), the work list of k_flatten (1); 16-byte aligned
extern "C" size_t vb_flatten_part_words(uint32_t n_parts) { return 35u * (((size_t)n_parts + 3u) & ~(size_t)3u); }
extern "C" void vb_flatten_arena_bytes(uint32_t cap_lines, size_t *lit_bytes, size_t *job_bytes) {
    *lit_bytes = (size_t)cap_lines * sizeof(FlLit);
    *job_bytes = ((size_t)cap_lines / FL_DEFER_MIN + 1u) * sizeof(FlJob);
}
