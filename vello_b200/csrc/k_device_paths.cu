// k_device_paths.cu -- fragments from device arrays (vb_fragment_from_device_paths, vb_fragment_from_device_curves): the
// encoding of ragged polygons, polylines or Bézier paths held in device memory (points, optional point kinds, ring offsets,
// optional path offsets, colours), built on the device, word for word what the host encoder writes for
//     for each path i: scene.fill(rule, IDENTITY, Color(colors[i]), None, shape_i)   (or scene.stroke(stroke, ...))
// where shape_i is, for each ring of path i, M p_first, then one segment per following on-curve point e (kind 0), chosen by
// the off-curve points (kind 1) in front of it: none L e, one Q c e, two C c1 c2 e; then Z (fills always, strokes when
// `closed`). Without kinds every point is on-curve: M p_first, L p... The PathEncoder's rules (encoding.py's PathEncoder,
// vb_scene.cpp's) decide what each segment writes:
//  - before a ring's first kept segment (MoveTo state) a segment is kept when one of its points is EPS-far (1e-12 on the f32
//    differences) from the ring's first point (the start-tangent tests); that segment gives the ring's start tangent end;
//  - after it, a segment is kept when the EPS span of the last kept end point and the segment's points exceeds EPS in x or y
//    (is_zero_length_segment);
//  - a ring that keeps no segment writes nothing at all (its move-to is replaced or dropped);
//  - a kept ring ends with the closing line when its last kept end point differs bit for bit from its first point (fills and
//    closed strokes), then for a stroke its cap marker (closed: a line to the start tangent's end; open: a quad through the
//    first point to it), which is itself dropped when EPS-close to where the ring stands; its last tag gets SUBPATH_END;
//  - a path that keeps a ring ends with a PATH tag and draws one FILL_COLOR draw object.
// A kept segment's points write their own two path-data words each, and its tag byte belongs to its end point.
//
// Four launches, in stream order, all sized from the caller's counts:
//  1. k_device_paths_points, one thread per point, per ring offset, per path offset and per colour row: the device-side
//     checks (one 64-bit atomicMin of (kind << 32 | row), so the first offending row of the first kind wins), and for each
//     point: the start-tangent test against the ring's first point, and for an on-curve point the span test of its segment
//     against the segment's own start (the previous on-curve point). Warp-aggregated atomics give each ring its first kept
//     segment (the lowest end point whose segment passes the tangent test: exact, with no sequential dependency), the last end
//     point that passes the span test, and the last end point whose segment fails it while ending unequal in value to its
//     start. The span rule "against the last kept end point" equals the test against the segment's own start unless such a
//     dropped segment lies after the first kept one (coordinates below about 1.7e-5): only those rings are walked. +0 beside
//     -0 is equal in value and its differences are the same, so it needs no walk; the closing line compares bits on either
//     route.
//  2. k_device_paths_rings, one thread per ring: a flagged ring is walked in order with the exact rule (its keep flags go to
//     a byte per end point); then the ring's record: kept or not, last kept end point, closing line, cap marker, start tangent
//     end. A kept ring marks its path kept.
//  3. k_device_paths_count, 256 points per partition in ticket order: each point's tag bytes, path-data words and draw objects
//     (the ring-end and path-end contributions belong to the ring's and the path's last point), summed with one packed block
//     scan and the decoupled look-back (K = 3). The last partition writes the totals.
//  4. k_device_paths_emit: the header and the six streams, straight into the fragment's allocation in vb_fragment_upload's
//     layout (the header's word offsets, then the streams back to back, tags padded to whole words with zero bytes), and
//     draw_index.
// Every launch after the first returns at once when a check failed: the offsets and kinds are then not trusted to index
// anything.
// With ring_flags (the sub-rings of vb_fragment_from_device_dashes, k_device_dashes.cu) a ring closes by its flag instead of
// `kind == 0 || closed`, and a conditional ring (the segment a dasher's walk pushes after Z) is kept only when a lower,
// unconditional ring of its path keeps a segment (path_min): the encoder draws it from the first point only after the path
// has encoded a segment.
#include "vb_device.cuh"
#include "vb_stages.h"

#define DP_THREADS 256u
#define DP_TAG_LINE 0x09u // + 1 per control point: QUAD 0x0a, CUBIC 0x0b
#define DP_TAG_QUAD 0x0au
#define DP_TAG_PATH 0x10u
#define DP_TAG_TRANSFORM 0x20u
#define DP_TAG_STYLE 0x40u
#define DP_SUBPATH_END 0x04u
#define DP_EPS 1e-12f // path.rs:841; f32(1e-12) < 1e-12, so `d > DP_EPS` is the encoders' test for every f32 d

// a ring record (DpArgs::rings) is {last kept end point, code, start tangent end x, y}; the code's bits:
#define DP_KEPT 1u
#define DP_CLOSE 2u   // the closing line to the first point
#define DP_CAP_LINE 4u
#define DP_CAP_QUAD 8u
#define DP_WALKED 16u // keep flags in keep_fix

__device__ __forceinline__ float2 dp_point(const DpArgs &a, uint32_t j) {
    const float *p = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(a.points) + (size_t)j * a.point_pitch);
    return make_float2(__ldg(p), __ldg(p + 1));
}
// a point's kind: 0 on-curve, 1 off-curve; without kinds every point is on-curve
__device__ __forceinline__ uint32_t dp_kind(const DpArgs &a, uint32_t j) { return a.kinds ? (uint32_t)__ldg(a.kinds + j) : 0u; }
// the encoders' EPS test of two points (PathEncoder._neq; _zero_len of a line)
__device__ __forceinline__ bool dp_neq(float2 p, float2 q) {
    return fabsf(__fsub_rn(p.x, q.x)) > DP_EPS || fabsf(__fsub_rn(p.y, q.y)) > DP_EPS;
}
__device__ __forceinline__ float dp_span3(float a, float b, float c) { return __fsub_rn(fmaxf(fmaxf(a, b), c), fminf(fminf(a, b), c)); }
__device__ __forceinline__ bool dp_same_bits(float2 p, float2 q) {
    return __float_as_uint(p.x) == __float_as_uint(q.x) && __float_as_uint(p.y) == __float_as_uint(q.y);
}
// the segment that point j (b0 < j < b1) belongs to ends at the first on-curve point at or after j; with checked kinds that is
// j, j + 1 or j + 2, and before the checks it stays inside the ring
__device__ __forceinline__ uint32_t dp_seg_end(const DpArgs &a, uint32_t j, uint32_t b1) {
    uint32_t e = j;
    if (a.kinds)
        while (e + 1u < b1 && e < j + 2u && dp_kind(a, e) == 1u) e++;
    return e;
}
// the degree of the segment ending at on-curve point e (b0 < e): 1 + the off-curve points in front of it, at most 3, never
// reaching the ring's first point. Its start is point e - degree.
__device__ __forceinline__ uint32_t dp_degree(const DpArgs &a, uint32_t b0, uint32_t e) {
    uint32_t d = 1u;
    if (a.kinds)
        while (d < 3u && e - d > b0 && dp_kind(a, e - d) == 1u) d++;
    return d;
}
// is_zero_length_segment, negated: the EPS span of `at` (where the ring stands) and points s + 1 .. e exceeds EPS in x or y;
// pe is point e (a line reads no other point)
__device__ __forceinline__ bool dp_span_keeps(const DpArgs &a, float2 at, uint32_t s, uint32_t e, float2 pe) {
    float x0 = fminf(at.x, pe.x), x1 = fmaxf(at.x, pe.x), y0 = fminf(at.y, pe.y), y1 = fmaxf(at.y, pe.y);
    for (uint32_t k = s + 1u; k < e; k++) {
        const float2 q = dp_point(a, k);
        x0 = fminf(x0, q.x), x1 = fmaxf(x1, q.x), y0 = fminf(y0, q.y), y1 = fmaxf(y1, q.y);
    }
    return __fsub_rn(x1, x0) > DP_EPS || __fsub_rn(y1, y0) > DP_EPS;
}
// the last k in [0, n) with off[k] <= x (offsets checked: non-decreasing from 0). n >= 1: the launches after the first run only
// when the checks passed, and then points imply a ring (ring_offsets[0] = 0 < n_points = ring_offsets[n_rings]) and rings a
// path (path_offsets[n_paths] = n_rings)
__device__ __forceinline__ uint32_t dp_find(const int32_t *__restrict__ off, uint32_t n, uint32_t x) {
    return cp_find(reinterpret_cast<const uint32_t *>(off), 0u, n - 1u, x);
}
__device__ __forceinline__ void dp_fail(const DpArgs &a, uint32_t kind, uint32_t row) {
    atomicMin(a.err, ((unsigned long long)kind << 32) | row);
}
__device__ __forceinline__ bool dp_failed(const DpArgs &a) { return *(volatile unsigned long long *)a.err != ~0ull; }

__global__ void __launch_bounds__(DP_THREADS) k_device_paths_points(DpArgs a) {
    const uint32_t g = blockIdx.x * DP_THREADS + threadIdx.x;
    // offsets: ring_offsets over points, path_offsets over rings
    if (a.ring_offsets && g <= a.n_rings) {
        const int32_t v = __ldg(a.ring_offsets + g);
        // the end test applies to entry 0 too: with no ring, ring_offsets[0] must be n_points (0)
        const bool bad = (g == 0u ? v != 0 : v < __ldg(a.ring_offsets + g - 1u)) || (g == a.n_rings && v != (int32_t)a.n_points);
        if (bad) dp_fail(a, VB_DP_ERR_RING_OFFSETS, g);
    }
    if (a.path_offsets && g <= a.n_paths) {
        const int32_t v = __ldg(a.path_offsets + g);
        const bool bad = (g == 0u ? v != 0 : v < __ldg(a.path_offsets + g - 1u)) || (g == a.n_paths && v != (int32_t)a.n_rings);
        if (bad) dp_fail(a, VB_DP_ERR_PATH_OFFSETS, g);
    }
    if (g < a.n_paths) {
        const float *c = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(a.colors) + (size_t)g * a.color_pitch);
        if (!(isfinite(__ldg(c)) && isfinite(__ldg(c + 1)) && isfinite(__ldg(c + 2)) && isfinite(__ldg(c + 3)))) dp_fail(a, VB_DP_ERR_COLOR, g);
    }
    // points: every lane of the warp takes part in the aggregation below. `tangent` is the end point of this point's segment
    // when the point is EPS-far from the ring's first one; `span` an end point whose segment passes the span test against its
    // own start; `odd` one whose segment fails it but ends unequal in value to its start.
    uint32_t ring = 0xffffffffu, tangent = 0xffffffffu, span = 0u, odd = 0u;
    if (g < a.n_points && a.n_rings) {
        const float2 p = dp_point(a, g);
        if (!(isfinite(p.x) && isfinite(p.y))) dp_fail(a, VB_DP_ERR_POINTS, g);
        ring = dp_find(a.ring_offsets, a.n_rings, g);
        const int32_t first = __ldg(a.ring_offsets + ring);
        const uint32_t b1 = a.kinds ? min((uint32_t)__ldg(a.ring_offsets + ring + 1u), a.n_points) : 0u; // unchecked yet
        if (a.kinds) {
            // a value other than 0 or 1; an off-curve point first or last in its ring, or third in a row (a run across rings
            // has an off-curve last point at a lower row, so the first offending row is the same)
            const uint32_t k = dp_kind(a, g);
            if (k > 1u || (k == 1u && ((int32_t)g == first || g + 1u == b1 || (g >= 2u && dp_kind(a, g - 1u) == 1u && dp_kind(a, g - 2u) == 1u))))
                dp_fail(a, VB_DP_ERR_KINDS, g);
        }
        if (first >= 0 && (uint32_t)first < g) {
            const uint32_t b0 = (uint32_t)first;
            if (dp_neq(p, dp_point(a, b0))) tangent = a.kinds ? dp_seg_end(a, g, b1) : g;
            if (dp_kind(a, g) == 0u) {
                const uint32_t s = g - dp_degree(a, b0, g);
                const float2 q = dp_point(a, s);
                if (dp_span_keeps(a, q, s, g, p)) span = g;
                else if (!(p.x == q.x && p.y == q.y)) odd = g;
            }
        }
    }
    const uint32_t group = __match_any_sync(VB_FULL, ring);
    const uint32_t lo = __reduce_min_sync(group, tangent), hi = __reduce_max_sync(group, span);
    const uint32_t last_odd = __reduce_max_sync(group, odd);
    if (ring != 0xffffffffu && vb_lane() == (uint32_t)__ffs(group) - 1u) {
        if (lo != 0xffffffffu) atomicMin(a.ring_first + ring, lo);
        if (hi) atomicMax(a.ring_last + ring, hi);
        if (last_odd) atomicMax(a.ring_odd + ring, last_odd);
    }
}

__global__ void __launch_bounds__(DP_THREADS) k_device_paths_rings(DpArgs a) {
    const uint32_t r = blockIdx.x * DP_THREADS + threadIdx.x;
    if (r >= a.n_rings || dp_failed(a)) return;
    const uint32_t b0 = (uint32_t)__ldg(a.ring_offsets + r), b1 = (uint32_t)__ldg(a.ring_offsets + r + 1u);
    const uint32_t first = a.ring_first[r];
    uint32_t last = a.ring_last[r], code = 0u;
    float2 ste = make_float2(0.0f, 0.0f);
    if (first != 0xffffffffu) {
        code |= DP_KEPT;
        if (a.ring_odd[r] > first) { // the encoders' walk after the first kept segment: the span against the last kept end
            code |= DP_WALKED;
            last = first;
            float2 at = dp_point(a, first);
            for (uint32_t e = first + 1u; e < b1; e++) {
                if (dp_kind(a, e) != 0u) continue;
                const float2 pe = dp_point(a, e);
                const bool k = dp_span_keeps(a, at, e - dp_degree(a, b0, e), e, pe);
                a.keep_fix[e] = k ? 1u : 0u;
                if (k) {
                    last = e;
                    at = pe;
                }
            }
        } else if (last < first) {
            last = first;
        }
        // the start tangent's end, from the first kept segment (start_tangent_for_line / _quad / _curve)
        const uint32_t d = dp_degree(a, b0, first);
        const float2 p0 = dp_point(a, b0), pe = dp_point(a, first), pl = dp_point(a, last);
        const float third = __fdiv_rn(1.0f, 3.0f);
        auto toward = [&](float2 from, float2 to) {
            return make_float2(__fadd_rn(from.x, __fmul_rn(third, __fsub_rn(to.x, from.x))), __fadd_rn(from.y, __fmul_rn(third, __fsub_rn(to.y, from.y))));
        };
        if (d == 1u) {
            ste = toward(p0, pe);
        } else if (d == 2u) {
            const float2 c = dp_point(a, first - 1u);
            ste = dp_neq(c, p0) ? toward(c, p0) : toward(c, pe);
        } else {
            const float2 c1 = dp_point(a, first - 2u), c2 = dp_point(a, first - 1u);
            ste = dp_neq(c1, p0) ? c1 : (dp_neq(c2, p0) ? c2 : pe);
        }
        const uint32_t flags = a.ring_flags ? (uint32_t)a.ring_flags[r] : 0u;
        const bool closes = a.ring_flags ? (flags & VB_DP_RING_CLOSED) != 0u : (a.kind == 0u || a.closed);
        if (closes && !dp_same_bits(pl, p0)) code |= DP_CLOSE;
        if (a.kind == 1u) {
            if (closes) {
                if (dp_neq(ste, p0)) code |= DP_CAP_LINE; // the ring stands at its first point (or its bit-equal last one)
            } else if (dp_span3(pl.x, p0.x, ste.x) > DP_EPS || dp_span3(pl.y, p0.y, ste.y) > DP_EPS) {
                code |= DP_CAP_QUAD;
            }
        }
        // a conditional ring is kept after a kept unconditional one of its path (dp_out), which has marked the path
        if (!(flags & VB_DP_RING_CONDITIONAL)) {
            const uint32_t i = a.path_offsets ? dp_find(a.path_offsets, a.n_paths, r) : r;
            a.path_kept[i] = 1u;
            if (a.ring_flags) atomicMin(a.path_min + i, r);
        }
    }
    a.rings[r] = make_uint4(last, code, __float_as_uint(ste.x), __float_as_uint(ste.y));
}

// What point j writes, in stream order: its tag bytes (`tags` of them, the first in the low byte); its path-data words, 2 per
// point: `p` when `main`, then p0 for the ring's closing line, ste for a closed stroke's cap line, p0 and ste for an open
// one's cap quad (`tail`); and draw object of path `path` when `draws`.
struct DpOut {
    uint32_t tag_bytes, tags, words, draws, main, tail, path;
    float2 p, p0, ste;
};
__device__ __forceinline__ DpOut dp_out(const DpArgs &a, uint32_t j) {
    DpOut o;
    o.tag_bytes = o.tags = o.words = o.draws = o.main = o.tail = o.path = 0u;
    if (j >= a.n_points) return o;
    const uint32_t r = dp_find(a.ring_offsets, a.n_rings, j);
    const uint4 rec = a.rings[r];
    const uint32_t b0 = (uint32_t)__ldg(a.ring_offsets + r), b1 = (uint32_t)__ldg(a.ring_offsets + r + 1u), code = rec.y;
    bool kept = code & DP_KEPT;
    if (kept && a.ring_flags && (a.ring_flags[r] & VB_DP_RING_CONDITIONAL))
        kept = a.path_min[dp_find(a.path_offsets, a.n_paths, r)] < r; // ring_flags come with path_offsets
    if (kept) {
        o.p = dp_point(a, j);
        const uint32_t tail = code & (DP_CLOSE | DP_CAP_LINE | DP_CAP_QUAD);
        if (j == b0) {
            o.main = 1u;
        } else {
            // the segment of point j: kept when it is the first kept one, or after it and kept by the span test
            const uint32_t e = dp_seg_end(a, j, b1), first = a.ring_first[r], d = dp_degree(a, b0, e);
            bool keep = e == first;
            if (e > first)
                keep = (code & DP_WALKED) ? a.keep_fix[e] != 0u : dp_span_keeps(a, dp_point(a, e - d), e - d, e, e == j ? o.p : dp_point(a, e));
            if (keep) {
                o.main = 1u;
                if (j == e) {
                    o.tag_bytes = (DP_TAG_LINE + d - 1u) | (j == rec.x && !tail ? DP_SUBPATH_END : 0u);
                    o.tags = 1u;
                }
            }
        }
        o.words = 2u * o.main;
        if (j == b1 - 1u && tail) {
            o.tail = tail;
            o.p0 = dp_point(a, b0);
            o.ste = make_float2(__uint_as_float(rec.z), __uint_as_float(rec.w));
            // the ring's tags end with the closing line, then the cap marker; the last of them gets SUBPATH_END
            uint32_t t = 0u, n = 0u;
            if (tail & DP_CLOSE) t |= DP_TAG_LINE << (8u * n++), o.words += 2u;
            if (tail & DP_CAP_LINE) t |= DP_TAG_LINE << (8u * n++), o.words += 2u;
            if (tail & DP_CAP_QUAD) t |= DP_TAG_QUAD << (8u * n++), o.words += 4u;
            t |= DP_SUBPATH_END << (8u * (n - 1u));
            o.tag_bytes |= t << (8u * o.tags);
            o.tags += n;
        }
    }
    const uint32_t i = a.path_offsets ? dp_find(a.path_offsets, a.n_paths, r) : r;
    const uint32_t path_end = a.path_offsets ? (uint32_t)__ldg(a.ring_offsets + __ldg(a.path_offsets + i + 1u)) : b1;
    if (j == path_end - 1u && a.path_kept[i]) {
        o.tag_bytes |= DP_TAG_PATH << (8u * o.tags++);
        o.draws = 1u;
        o.path = i;
    }
    return o;
}
// one point's counts packed for the block scan: tags (<= 4 a point: its segment's, the closing line, the cap marker, PATH) in
// bits 0..10, words (<= 6: its own, then a closing line and a cap line, or a cap quad) in 11..21, draws in 22..31
__device__ __forceinline__ uint32_t dp_pack(const DpOut &o) { return o.tags | (o.words << 11) | (o.draws << 22); }

__global__ void __launch_bounds__(DP_THREADS) k_device_paths_count(DpArgs a) {
    __shared__ uint32_t sh[DP_THREADS / 32u + 1u];
    __shared__ uint32_t sh_ticket;
    if (dp_failed(a)) return; // every CTA returns: no partition waits on another
    const VbLookback lb = vb_lookback_view(a.lookback, a.n_parts, 3);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const DpOut o = dp_out(a, part * DP_THREADS + threadIdx.x);
    uint32_t total;
    vb_block_excl_scan(dp_pack(o), sh, &total);
    if (threadIdx.x < 32u) {
        const uint32_t agg[3] = {total & 0x7ffu, (total >> 11) & 0x7ffu, total >> 22};
        uint32_t excl[3];
        vb_lookback<3>(lb, part, agg, excl);
        if (threadIdx.x == 0u) {
            for (int k = 0; k < 3; k++) a.part_excl[3u * part + k] = excl[k];
            if (part == a.n_parts - 1u)
                for (int k = 0; k < 3; k++) a.totals[k] = excl[k] + agg[k];
        }
    }
}

__global__ void __launch_bounds__(DP_THREADS) k_device_paths_emit(DpArgs a) {
    __shared__ uint32_t sh[DP_THREADS / 32u + 1u];
    if (dp_failed(a)) return;
    const uint32_t g = blockIdx.x * DP_THREADS + threadIdx.x;
    const uint32_t head = a.n_paths ? 2u : 0u; // the TRANSFORM and STYLE tags
    const uint32_t n_tags = head + a.totals[0], n_words = a.totals[1], n_draws = a.totals[2];
    uint32_t *frag = a.fragment;
    // the header: each stream's word offset (vb_fragment_upload's layout)
    const uint32_t o_tags = CMP_HEADER_WORDS, o_pd = o_tags + (n_tags + 3u) / 4u, o_dt = o_pd + n_words, o_dd = o_dt + n_draws,
                   o_tr = o_dd + n_draws, o_st = o_tr + (a.n_paths ? 6u : 0u);
    uint8_t *tags = reinterpret_cast<uint8_t *>(frag + o_tags);
    if (g == 0u) {
        const uint32_t h[CMP_HEADER_WORDS] = {o_tags, o_pd, o_dt, o_dd, o_tr, o_st, 0u, 0u};
        for (uint32_t k = 0; k < CMP_HEADER_WORDS; k++) frag[k] = h[k];
        if (a.n_paths) {
            tags[0] = DP_TAG_TRANSFORM;
            tags[1] = DP_TAG_STYLE;
            const float id[6] = {1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f};
            for (int k = 0; k < 6; k++) frag[o_tr + k] = __float_as_uint(id[k]);
            frag[o_st] = a.style_flags;
            frag[o_st + 1u] = a.style_width;
        }
        for (uint32_t t = n_tags; t & 3u; t++) tags[t] = 0u;
    }
    if (g < a.n_paths && !a.path_kept[g] && a.draw_index) a.draw_index[g] = -1;
    if (blockIdx.x >= a.n_parts) return; // the CTAs past the points' partitions only write draw_index
    const DpOut o = dp_out(a, g);
    uint32_t total;
    const uint32_t x = vb_block_excl_scan(dp_pack(o), sh, &total);
    const uint32_t t0 = head + a.part_excl[3u * blockIdx.x] + (x & 0x7ffu);
    const uint32_t w0 = o_pd + a.part_excl[3u * blockIdx.x + 1u] + ((x >> 11) & 0x7ffu);
    const uint32_t d = a.part_excl[3u * blockIdx.x + 2u] + (x >> 22);
    for (uint32_t k = 0; k < o.tags; k++) tags[t0 + k] = (uint8_t)(o.tag_bytes >> (8u * k));
    uint32_t w = w0;
    auto put = [&](float2 p) {
        frag[w++] = __float_as_uint(p.x);
        frag[w++] = __float_as_uint(p.y);
    };
    if (o.main) put(o.p);
    if (o.tail & (DP_CLOSE | DP_CAP_QUAD)) put(o.p0);
    if (o.tail & (DP_CAP_LINE | DP_CAP_QUAD)) put(o.ste);
    if (o.draws) {
        const float *c = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(a.colors) + (size_t)o.path * a.color_pitch);
        frag[o_dt + d] = VB_DRAWTAG_FILL_COLOR;
        frag[o_dd + d] = dc_premul_rgba8(__ldg(c), __ldg(c + 1), __ldg(c + 2), __ldg(c + 3));
        if (a.draw_index) a.draw_index[o.path] = (int32_t)d;
    }
}

extern "C" uint32_t vb_launch_device_paths(const DpArgs &a, cudaStream_t st) {
    uint32_t n = vb_launch_device_paths_checks(a, st);
    if (a.n_rings) k_device_paths_rings<<<(a.n_rings + DP_THREADS - 1u) / DP_THREADS, DP_THREADS, 0, st>>>(a), n++;
    if (a.n_parts) k_device_paths_count<<<a.n_parts, DP_THREADS, 0, st>>>(a), n++;
    const uint32_t path_ctas = (a.n_paths + DP_THREADS - 1u) / DP_THREADS;
    k_device_paths_emit<<<a.n_parts > path_ctas ? a.n_parts : (path_ctas ? path_ctas : 1u), DP_THREADS, 0, st>>>(a);
    return n + 1u;
}
extern "C" uint32_t vb_launch_device_paths_checks(const DpArgs &a, cudaStream_t st) {
    const uint32_t checks = a.n_points > a.n_rings + 1u ? a.n_points : a.n_rings + 1u;
    const uint32_t rows = checks > a.n_paths + 1u ? checks : a.n_paths + 1u;
    k_device_paths_points<<<(rows + DP_THREADS - 1u) / DP_THREADS, DP_THREADS, 0, st>>>(a);
    return 1u;
}
extern "C" uint32_t vb_device_paths_parts(uint32_t n_points) { return (n_points + DP_THREADS - 1u) / DP_THREADS; }
