// k_device_dashes.cu -- dashed strokes from device arrays (vb_fragment_from_device_dashes): the host dasher (kurbo's
// DashIterator as vb_scene.cpp's dash_path and shapes.py's `dash` restate it) run on the device, one warp per ring, writing a
// ragged intermediate of sub-rings that k_device_paths.cu then encodes like any other device paths.
//
// Each ring of two or more points is dashed on its own (the phase resets at every M and Z and the held-back first dash is
// flushed at the ring's end, so a path's dashes are its rings' dashes joined); a ring of fewer points contributes nothing. A
// ring's walk is the host's state machine, step for step in f64 with every operation rounded on its own (__dadd_rn, ...), so
// each cut point is the host's bit for bit:
//  - W: what the walk writes once it has left the first dash, in order;
//  - S: the first dash (the stash), held back and written after W. When a closed ring's last dash is still active at the close,
//    S continues it without its M; when the ring never leaves its first dash and closes, S is `M p0, seg_0 .. seg_{n-2}, Z,
//    seg_{n-1}` (the last segment after the Z, as the host's walk pushes it).
// The output elements become sub-rings: M starts one; a piece of an L, Q or C appends its points (kinds 0 / 1 0 / 1 1 0); Z
// flags the sub-ring closed, and the one segment after it becomes a sub-ring of its own, the ring's first point then the
// segment's points, flagged conditional: the encoder, in its START state, draws it from the first point only when the path
// has already kept a segment (DpArgs::ring_flags).
//
// Launches, in stream order (vb_launch_device_dashes):
//  1. k_device_paths_points over the input arrays: the checks of vb_fragment_from_device_paths / _curves;
//  2. k_device_dashes_phase, one thread per path, with per-path offsets only: the offset's check and its pre-roll into the
//     pattern (the dash index, what remains of it and whether it is drawn), at most 2^24 steps as the native front end allows;
//  3. k_device_dashes_count, one warp per ring: a bound on the ring's dash breaks from its control polygon's length (a ring
//     past 2^31 is refused unwalked), then the walk, counting each ring's intermediate points and sub-rings and those of S;
//  4. k_device_dashes_scan, 256 rings per partition with the decoupled look-back: each ring's exclusive prefix, saturating at
//     2^31, and the totals, which the caller reads back to size the intermediate;
// and after that synchronisation (vb_launch_device_dashes_emit):
//  5. k_device_dashes_emit, one warp per ring: the walk again, writing W from the ring's first row and S from its last rows,
//     and one thread per path: the path offsets over the sub-rings.
// Every launch after the checks returns at once when a check failed. The lanes of a warp hold the walk's state alike; they
// share a Bézier arc length's 128 Gauss-Legendre terms, which lane 0's order sums as the host does, and lane 0 writes.
#include "vb_device.cuh"
#include "vb_stages.h"

#define DD_THREADS 256u
#define DD_WARPS (DD_THREADS / 32u)
#define DD_CAP 0x80000000u // the counts saturate here: past int32 offsets

__device__ __forceinline__ double dd_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dd_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd_mul(double a, double b) { return __dmul_rn(a, b); }

// a segment in absolute coordinates: degree k (1 line, 2 quad, 3 cubic), points 0..k
struct DdSeg {
    uint32_t k;
    double x[4], y[4];
};

__device__ __forceinline__ double2 dd_eval(const DdSeg &s, double t) {
    if (s.k == 1u) return make_double2(dd_add(s.x[0], dd_mul(t, dd_sub(s.x[1], s.x[0]))), dd_add(s.y[0], dd_mul(t, dd_sub(s.y[1], s.y[0]))));
    const double mt = dd_sub(1.0, t);
    if (s.k == 2u) {
        const double a = dd_mul(mt, mt), b = dd_mul(dd_mul(2.0, mt), t), c = dd_mul(t, t);
        return make_double2(dd_add(dd_add(dd_mul(a, s.x[0]), dd_mul(b, s.x[1])), dd_mul(c, s.x[2])),
                            dd_add(dd_add(dd_mul(a, s.y[0]), dd_mul(b, s.y[1])), dd_mul(c, s.y[2])));
    }
    const double a = dd_mul(dd_mul(mt, mt), mt), b = dd_mul(dd_mul(dd_mul(3.0, mt), mt), t), c = dd_mul(dd_mul(dd_mul(3.0, mt), t), t),
                 d = dd_mul(dd_mul(t, t), t);
    return make_double2(dd_add(dd_add(dd_add(dd_mul(a, s.x[0]), dd_mul(b, s.x[1])), dd_mul(c, s.x[2])), dd_mul(d, s.x[3])),
                        dd_add(dd_add(dd_add(dd_mul(a, s.y[0]), dd_mul(b, s.y[1])), dd_mul(c, s.y[2])), dd_mul(d, s.y[3])));
}
__device__ __forceinline__ double2 dd_deriv(const DdSeg &s, double t) {
    const double mt = dd_sub(1.0, t);
    if (s.k == 2u)
        return make_double2(dd_mul(2.0, dd_add(dd_mul(mt, dd_sub(s.x[1], s.x[0])), dd_mul(t, dd_sub(s.x[2], s.x[1])))),
                            dd_mul(2.0, dd_add(dd_mul(mt, dd_sub(s.y[1], s.y[0])), dd_mul(t, dd_sub(s.y[2], s.y[1])))));
    const double a = dd_mul(dd_mul(3.0, mt), mt), b = dd_mul(dd_mul(6.0, mt), t), c = dd_mul(dd_mul(3.0, t), t);
    return make_double2(dd_add(dd_add(dd_mul(a, dd_sub(s.x[1], s.x[0])), dd_mul(b, dd_sub(s.x[2], s.x[1]))), dd_mul(c, dd_sub(s.x[3], s.x[2]))),
                        dd_add(dd_add(dd_mul(a, dd_sub(s.y[1], s.y[0])), dd_mul(b, dd_sub(s.y[2], s.y[1]))), dd_mul(c, dd_sub(s.y[3], s.y[2]))));
}
__device__ __forceinline__ double dd_norm(double2 d) { return __dsqrt_rn(dd_add(dd_mul(d.x, d.x), dd_mul(d.y, d.y))); }
__device__ __forceinline__ double dd_shfl(double v, uint32_t lane) { return __shfl_sync(VB_FULL, v, lane); }

// The arc length of a quad or cubic over [t0, t1]: composite 8-point Gauss-Legendre on 16 pieces. Lane l takes piece l / 2
// and nodes 2 (l & 1), 2 (l & 1) + 1 (both signs); every lane returns the host's sum, `acc` over the nodes in order, then
// `total` over the pieces in order.
__device__ __forceinline__ double dd_curve_arclen(const DdSeg &s, double t0, double t1) {
    const uint32_t lane = vb_lane();
    const bool odd = lane & 1u;
    const double h = __ddiv_rn(dd_sub(t1, t0), 16.0);
    const double a = dd_add(t0, dd_mul(h, (double)(lane >> 1)));
    const double mid = dd_add(a, dd_mul(0.5, h)), half = dd_mul(0.5, h);
    const double xa = odd ? 0.7966664774136267 : 0.1834346424956498, wa = odd ? 0.2223810344533745 : 0.3626837833783620;
    const double xb = odd ? 0.9602898564975363 : 0.5255324099163290, wb = odd ? 0.1012285362903763 : 0.3137066458778873;
    const double ta = dd_mul(wa, dd_add(dd_norm(dd_deriv(s, dd_sub(mid, dd_mul(half, xa)))), dd_norm(dd_deriv(s, dd_add(mid, dd_mul(half, xa))))));
    const double tb = dd_mul(wb, dd_add(dd_norm(dd_deriv(s, dd_sub(mid, dd_mul(half, xb)))), dd_norm(dd_deriv(s, dd_add(mid, dd_mul(half, xb))))));
    const double t2 = __shfl_down_sync(VB_FULL, ta, 1), t3 = __shfl_down_sync(VB_FULL, tb, 1);
    const double piece = dd_mul(dd_add(dd_add(dd_add(dd_add(0.0, ta), tb), t2), t3), half); // meaningful in the even lanes
    double total = 0.0;
#pragma unroll
    for (uint32_t i = 0; i < 16u; i++) total = dd_add(total, dd_shfl(piece, 2u * i));
    return total;
}
__device__ __forceinline__ double dd_arclen(const DdSeg &s) {
    if (s.k == 1u) return dd_norm(make_double2(dd_sub(s.x[1], s.x[0]), dd_sub(s.y[1], s.y[0])));
    return dd_curve_arclen(s, 0.0, 1.0);
}
__device__ __forceinline__ double dd_inv_arclen(const DdSeg &s, double len) {
    if (s.k == 1u) return __ddiv_rn(len, dd_arclen(s));
    double lo = 0.0, hi = 1.0;
    for (int it = 0; it < 48; it++) {
        const double mid = dd_mul(0.5, dd_add(lo, hi));
        if (dd_curve_arclen(s, 0.0, mid) < len) lo = mid;
        else hi = mid;
    }
    return dd_mul(0.5, dd_add(lo, hi));
}
__device__ __forceinline__ DdSeg dd_sub_seg(const DdSeg &s, double t0, double t1) {
    DdSeg r;
    r.k = s.k;
    const double2 p0 = dd_eval(s, t0), pe = dd_eval(s, t1);
    r.x[0] = p0.x, r.y[0] = p0.y;
    r.x[1] = r.y[1] = r.x[2] = r.y[2] = r.x[3] = r.y[3] = 0.0;
    if (s.k == 1u) {
        r.x[1] = pe.x, r.y[1] = pe.y;
    } else if (s.k == 2u) {
        const double ax = dd_sub(s.x[1], s.x[0]), ay = dd_sub(s.y[1], s.y[0]), bx = dd_sub(s.x[2], s.x[1]), by = dd_sub(s.y[2], s.y[1]);
        const double dx = dd_add(ax, dd_mul(t0, dd_sub(bx, ax))), dy = dd_add(ay, dd_mul(t0, dd_sub(by, ay))), dt = dd_sub(t1, t0);
        r.x[1] = dd_add(p0.x, dd_mul(dx, dt)), r.y[1] = dd_add(p0.y, dd_mul(dy, dt));
        r.x[2] = pe.x, r.y[2] = pe.y;
    } else {
        const double scale = dd_mul(dd_sub(t1, t0), 1.0 / 3.0);
        const double2 d0 = dd_deriv(s, t0), d1 = dd_deriv(s, t1);
        r.x[1] = dd_add(p0.x, dd_mul(scale, d0.x)), r.y[1] = dd_add(p0.y, dd_mul(scale, d0.y));
        r.x[2] = dd_sub(pe.x, dd_mul(scale, d1.x)), r.y[2] = dd_sub(pe.y, dd_mul(scale, d1.y));
        r.x[3] = pe.x, r.y[3] = pe.y;
    }
    return r;
}

__device__ __forceinline__ double2 dd_point(const DdArgs &a, uint32_t j) {
    const float *p = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(a.points) + (size_t)j * a.point_pitch);
    return make_double2((double)__ldg(p), (double)__ldg(p + 1));
}
__device__ __forceinline__ uint32_t dd_kind(const DdArgs &a, uint32_t j) { return a.kinds ? (uint32_t)__ldg(a.kinds + j) : 0u; }
__device__ __forceinline__ uint32_t dd_path_of(const DdArgs &a, uint32_t r) {
    return a.path_offsets ? cp_find(reinterpret_cast<const uint32_t *>(a.path_offsets), 0u, a.n_paths - 1u, r) : r;
}
__device__ __forceinline__ bool dd_failed(const DdArgs &a) { return *(volatile unsigned long long *)a.err != ~0ull; }

// A place the walk writes elements to: the next point row and sub-ring; `tail` is set after a Z, when the next segment starts
// a conditional sub-ring at the ring's first point. Counting, only p and r move.
struct DdCursor {
    uint32_t p, r, tail;
};
template <bool EMIT> struct DdOut {
    const DdArgs &a;
    float2 first; // the ring's first point, where a conditional sub-ring starts
    __device__ __forceinline__ void point(DdCursor &c, double x, double y, uint32_t kind) {
        if (EMIT && vb_lane() == 0u) {
            reinterpret_cast<float2 *>(a.out_points)[c.p] = make_float2(__double2float_rn(x), __double2float_rn(y));
            a.out_kinds[c.p] = (uint8_t)kind;
        }
        c.p++;
    }
    __device__ __forceinline__ void start(DdCursor &c, uint32_t flags) {
        if (EMIT && vb_lane() == 0u) {
            a.out_ring_offsets[c.r] = (int32_t)c.p;
            a.out_flags[c.r] = (uint8_t)flags;
        }
        c.r++;
    }
    __device__ __forceinline__ void move(DdCursor &c, double2 p) {
        start(c, 0u);
        point(c, p.x, p.y, 0u);
    }
    // the element of a piece: its points after the first
    __device__ __forceinline__ void seg(DdCursor &c, const DdSeg &s) {
        if (c.tail) {
            c.tail = 0u;
            start(c, VB_DP_RING_CONDITIONAL);
            if (EMIT && vb_lane() == 0u) {
                reinterpret_cast<float2 *>(a.out_points)[c.p] = first;
                a.out_kinds[c.p] = 0u;
            }
            c.p++;
        }
        if (s.k == 1u) {
            point(c, s.x[1], s.y[1], 0u);
        } else if (s.k == 2u) {
            point(c, s.x[1], s.y[1], 1u);
            point(c, s.x[2], s.y[2], 0u);
        } else {
            point(c, s.x[1], s.y[1], 1u);
            point(c, s.x[2], s.y[2], 1u);
            point(c, s.x[3], s.y[3], 0u);
        }
    }
    __device__ __forceinline__ void close(DdCursor &c) {
        if (EMIT && vb_lane() == 0u) a.out_flags[c.r - 1u] |= (uint8_t)VB_DP_RING_CLOSED;
        c.tail = 1u;
    }
};

// The walk of ring r (b1 - b0 >= 2 points), dash_path's state machine for one ring. Counting (EMIT false), returns {W's
// points, W's sub-rings, S's points, S's sub-rings}, S without its M when it continues the last dash; emitting, writes W from
// w and S from s (the rows the count pass made room for), skipping S's M when rec says it has no sub-ring of its own.
template <bool EMIT> __device__ __forceinline__ uint4 dd_walk(const DdArgs &a, uint32_t r, uint32_t b0, uint32_t b1, DdCursor w, DdCursor s,
                                                           uint4 rec) {
    enum { TO_STASH, WORKING };
    const uint32_t path = dd_path_of(a, r);
    uint32_t ix = a.phase_ix ? a.phase_ix[path] : a.scalar_ix;
    double rem = a.phase_ix ? a.phase_rem[path] : a.scalar_rem;
    bool active = !(ix >> 31);
    ix &= 0x7fffffffu;
    const double2 start = dd_point(a, b0);
    DdOut<EMIT> out{a, make_float2((float)start.x, (float)start.y)};
    const uint32_t s_p = s.p, s_r = s.r;
    uint32_t state = TO_STASH;
    bool stash_empty = true, skip = false;
    double2 last = start;
    uint32_t e = b0 + 1u;
    bool closing = false; // the closing line is the segment being walked
    for (;;) {
        // the next segment: the input's up to the last point, then (closed) the line back to the first point unless the last
        // point equals it in value
        DdSeg seg;
        seg.k = 1u;
        seg.x[0] = last.x, seg.y[0] = last.y;
        seg.x[2] = seg.y[2] = seg.x[3] = seg.y[3] = 0.0;
        if (e < b1) {
            // checked kinds: none, one or two off-curve points, then the on-curve end
            seg.k = 1u;
            if (dd_kind(a, e) == 1u) {
                const double2 c1 = dd_point(a, e++);
                seg.x[1] = c1.x, seg.y[1] = c1.y, seg.k = 2u;
                if (dd_kind(a, e) == 1u) {
                    const double2 c2 = dd_point(a, e++);
                    seg.x[2] = c2.x, seg.y[2] = c2.y, seg.k = 3u;
                }
            }
            last = dd_point(a, e++);
            if (seg.k == 1u) seg.x[1] = last.x, seg.y[1] = last.y;
            else if (seg.k == 2u) seg.x[2] = last.x, seg.y[2] = last.y;
            else seg.x[3] = last.x, seg.y[3] = last.y;
        } else {
            closing = true;
            seg.x[1] = start.x, seg.y[1] = start.y;
            last = start;
        }
        // the segment that ends the input: after it comes the Z (closed) or the ring's end
        const bool final_seg = closing || (e >= b1 && !(a.closed && (last.x != start.x || last.y != start.y)));
        double seg_rem = dd_arclen(seg), t = 0.0;
        for (;;) {
            if (!EMIT && w.p + s.p >= DD_CAP) return make_uint4(DD_CAP, 0u, 0u, 0u); // the count passes int32
            if (state == TO_STASH && stash_empty) {
                if (active) {
                    if (!EMIT || rec.w != 0u) out.move(s, make_double2(seg.x[0], seg.y[0]));
                    stash_empty = false;
                } else {
                    state = WORKING;
                }
                continue;
            }
            // where this step's element goes: S while the first dash is held back (both cursors stay in registers)
            const bool to_s = state == TO_STASH;
            if (rem < seg_rem) {
                const DdSeg rest = dd_sub_seg(seg, t, 1.0);
                const double t1 = dd_inv_arclen(rest, rem);
                if (active) {
                    const DdSeg piece = dd_sub_seg(rest, 0.0, t1);
                    if (to_s) out.seg(s, piece);
                    else out.seg(w, piece);
                    state = WORKING;
                } else {
                    const double2 p = dd_eval(rest, t1);
                    if (to_s) out.move(s, p);
                    else out.move(w, p);
                }
                active = !active;
                t = dd_add(t, dd_mul(t1, dd_sub(1.0, t)));
                seg_rem = dd_sub(seg_rem, rem);
                ix = ix + 1u == a.n_pattern ? 0u : ix + 1u;
                rem = __ldg(a.pattern + ix);
            } else {
                rem = dd_sub(rem, seg_rem);
                if (final_seg && a.closed) { // the close comes before the piece is pushed
                    if (state == TO_STASH) out.close(s);
                    else if (active) skip = true;
                }
                if (active) {
                    const DdSeg piece = dd_sub_seg(seg, t, 1.0);
                    if (to_s) out.seg(s, piece);
                    else out.seg(w, piece);
                }
                break;
            }
        }
        if (final_seg) break;
    }
    if (EMIT) return rec;
    uint32_t sp = s.p - s_p, sr = s.r - s_r;
    if (skip && sr) sp--, sr--; // S continues the last dash: its M is not written
    return make_uint4(w.p, w.r, sp, sr);
}

__global__ void __launch_bounds__(DD_THREADS) k_device_dashes_phase(DdArgs a) {
    const uint32_t g = blockIdx.x * DD_THREADS + threadIdx.x;
    if (g >= a.n_paths) return;
    const float off = __ldg(reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(a.offsets) + (size_t)g * a.offset_pitch));
    uint32_t ix = 0u, inactive = 0u;
    double rem = dd_sub(__ldg(a.pattern), (double)off);
    bool bad = !isfinite(off);
    for (uint32_t guard = 0u; !bad && rem < 0.0; guard++) {
        if (guard > (1u << 24)) bad = true;
        else ix = ix + 1u == a.n_pattern ? 0u : ix + 1u, rem = dd_add(rem, __ldg(a.pattern + ix)), inactive ^= 1u;
    }
    if (bad) {
        atomicMin(a.err, ((unsigned long long)VB_DP_ERR_DASH_OFFSETS << 32) | g);
        return;
    }
    a.phase_rem[g] = rem;
    a.phase_ix[g] = ix | (inactive << 31);
}

__global__ void __launch_bounds__(DD_THREADS) k_device_dashes_count(DdArgs a) {
    const uint32_t r = blockIdx.x * DD_WARPS + (threadIdx.x >> 5);
    if (r >= a.n_rings || dd_failed(a)) return;
    const uint32_t b0 = (uint32_t)__ldg(a.ring_offsets + r), b1 = (uint32_t)__ldg(a.ring_offsets + r + 1u);
    uint4 c = make_uint4(0u, 0u, 0u, 0u);
    if (b1 - b0 >= 2u) {
        // Before the walk, a bound on its dash breaks: a Bézier is no longer than its control polygon, and each pattern period
        // along the ring breaks at most n_pattern times, so breaks <= n_pattern (L / period + 2) (1% on L for the quadrature and
        // the f64 chain). Every break writes a point, so a ring whose bound passes DD_CAP is refused without walking: no warp
        // walks more breaks than the intermediate can hold, and a pattern too fine for the ring's coordinates (where
        // seg_rem - rem stops shrinking in f64) is refused at once.
        double len = 0.0;
        for (uint32_t j = b0 + 1u + vb_lane(); j <= b1; j += 32u) {
            if (j == b1 && !a.closed) break;
            const double2 p = dd_point(a, j - 1u), q = dd_point(a, j == b1 ? b0 : j);
            len = dd_add(len, dd_norm(make_double2(dd_sub(q.x, p.x), dd_sub(q.y, p.y))));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) len = dd_add(len, __shfl_xor_sync(VB_FULL, len, o));
        const double breaks = (double)a.n_pattern * (len * 1.01 / a.pattern_period + 2.0);
        if (!(breaks < (double)DD_CAP)) c = make_uint4(DD_CAP, 0u, 0u, 0u);
        else c = dd_walk<false>(a, r, b0, b1, DdCursor{0u, 0u, 0u}, DdCursor{0u, 0u, 0u}, c);
    }
    if (vb_lane() == 0u) a.rec[r] = make_uint4(min(c.x + c.z, DD_CAP), c.y + c.w, c.z, c.w);
}

// the counts' look-back monoid: the sum, saturating at DD_CAP
struct DdSatOp {
    static constexpr bool commutative = false; // vb_lookback's commutative path sums without saturating
    template <int K> __device__ __forceinline__ static void combine(const uint32_t (&x)[K], const uint32_t (&y)[K], uint32_t (&r)[K]) {
#pragma unroll
        for (int k = 0; k < K; k++) r[k] = (uint32_t)min((unsigned long long)x[k] + y[k], (unsigned long long)DD_CAP);
    }
};

__global__ void __launch_bounds__(DD_THREADS) k_device_dashes_scan(DdArgs a) {
    __shared__ unsigned long long sh[2][DD_WARPS];
    __shared__ uint32_t sh_ticket;
    if (dd_failed(a)) return;
    const VbLookback lb = vb_lookback_view(a.lookback, a.n_parts, 2);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t r = part * DD_THREADS + threadIdx.x, lane = vb_lane(), warp = threadIdx.x >> 5;
    const uint4 rec = r < a.n_rings ? a.rec[r] : make_uint4(0u, 0u, 0u, 0u);
    // a block scan in 64 bits: each count is at most 2^31
    unsigned long long v[2] = {rec.x, rec.y};
#pragma unroll
    for (int k = 0; k < 2; k++) {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long u = __shfl_up_sync(VB_FULL, v[k], o);
            if ((int)lane >= o) v[k] += u;
        }
        if (lane == 31u) sh[k][warp] = v[k];
    }
    __syncthreads();
    unsigned long long before[2] = {0ull, 0ull}, total[2] = {0ull, 0ull};
#pragma unroll
    for (int k = 0; k < 2; k++)
        for (uint32_t q = 0; q < DD_WARPS; q++) {
            if (q < warp) before[k] += sh[k][q];
            total[k] += sh[k][q];
        }
    uint32_t excl[2] = {0u, 0u};
    __shared__ uint32_t sh_excl[2];
    if (warp == 0u) {
        const uint32_t agg[2] = {(uint32_t)min(total[0], (unsigned long long)DD_CAP), (uint32_t)min(total[1], (unsigned long long)DD_CAP)};
        vb_lookback<2, DdSatOp>(lb, part, agg, excl);
        if (lane == 0u) {
            sh_excl[0] = excl[0], sh_excl[1] = excl[1];
            if (part == a.n_parts - 1u) {
                uint32_t incl[2];
                DdSatOp::combine<2>(excl, agg, incl);
                a.excl[a.n_rings] = make_uint2(incl[0], incl[1]);
            }
        }
    }
    __syncthreads();
    if (r < a.n_rings) {
        const unsigned long long p = sh_excl[0] + before[0] + v[0] - rec.x, q = sh_excl[1] + before[1] + v[1] - rec.y;
        a.excl[r] = make_uint2((uint32_t)min(p, (unsigned long long)DD_CAP), (uint32_t)min(q, (unsigned long long)DD_CAP));
    }
}

__global__ void __launch_bounds__(DD_THREADS) k_device_dashes_emit(DdArgs a) {
    if (dd_failed(a)) return;
    const uint32_t g = blockIdx.x * DD_THREADS + threadIdx.x;
    // the path offsets over the sub-rings, and the sub-rings' end
    if (g <= a.n_paths) {
        const uint32_t ring = g == a.n_paths ? a.n_rings : (a.path_offsets ? (uint32_t)__ldg(a.path_offsets + g) : g);
        a.out_path_offsets[g] = (int32_t)a.excl[ring].y;
        if (g == a.n_paths) a.out_ring_offsets[a.excl[a.n_rings].y] = (int32_t)a.excl[a.n_rings].x;
    }
    const uint32_t r = blockIdx.x * DD_WARPS + (threadIdx.x >> 5);
    if (r >= a.n_rings) return;
    const uint32_t b0 = (uint32_t)__ldg(a.ring_offsets + r), b1 = (uint32_t)__ldg(a.ring_offsets + r + 1u);
    if (b1 - b0 < 2u) return;
    const uint4 rec = a.rec[r];
    const uint2 at = a.excl[r];
    // rec.w: S's sub-rings; 0 with S's points means S continues the last dash (its M is skipped)
    dd_walk<true>(a, r, b0, b1, DdCursor{at.x, at.y, 0u}, DdCursor{at.x + rec.x - rec.z, at.y + rec.y - rec.w, 0u}, rec);
}

extern "C" uint32_t vb_launch_device_dashes(const DpArgs &checks, const DdArgs &a, cudaStream_t st) {
    uint32_t n = vb_launch_device_paths_checks(checks, st);
    if (a.offsets && a.n_paths) k_device_dashes_phase<<<(a.n_paths + DD_THREADS - 1u) / DD_THREADS, DD_THREADS, 0, st>>>(a), n++;
    if (a.n_rings) {
        k_device_dashes_count<<<(a.n_rings + DD_WARPS - 1u) / DD_WARPS, DD_THREADS, 0, st>>>(a);
        k_device_dashes_scan<<<a.n_parts, DD_THREADS, 0, st>>>(a);
        n += 2u;
    }
    return n;
}
extern "C" uint32_t vb_launch_device_dashes_emit(const DdArgs &a, cudaStream_t st) {
    const uint32_t ring_ctas = (a.n_rings + DD_WARPS - 1u) / DD_WARPS, path_ctas = (a.n_paths + 1u + DD_THREADS - 1u) / DD_THREADS;
    k_device_dashes_emit<<<ring_ctas > path_ctas ? ring_ctas : path_ctas, DD_THREADS, 0, st>>>(a);
    return 1u;
}
extern "C" uint32_t vb_device_dashes_parts(uint32_t n_rings) { return (n_rings + DD_THREADS - 1u) / DD_THREADS; }
