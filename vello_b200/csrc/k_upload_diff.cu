// k_upload_diff.cu -- the damage of the first frame after a re-uploaded scene (vb_set_upload_diff): which draw objects of the
// scene the base frame rendered are still there, unchanged and in the same order, in the uploaded one.
//
// A draw object's inputs are its draw tag and draw data, the ramp row or atlas rectangle the draw data names, the path tag
// bytes from the byte after the previous path's end tag through its own TAG_PATH, the path data words those tags read, and
// the transforms and styles in effect at them (VbUdRec). eq(i, j) compares all of them word for word between old draw object i
// and new draw object j, each read through its own scene's layout and buffers: a gradient's ramp word by its extend bits and
// the bytes of its 512-texel row (a ramp that moved to another row is equal: k_make_ramps writes a row from its stops alone),
// an image by its draw data, atlas place included, and the texels of its rectangle (a moved slot is not equal: fine clamps
// its samples to the slot, so bilinear rounding may differ).
//
// Matching. With m = min(n_old, n_new), p the common prefix (eq(k, k) for k < p) and s the common suffix capped at m - p
// (eq(n_old - 1 - k, n_new - 1 - k) for k < s), new draw object j is matched to j when j < p, to j + n_old - n_new when
// j >= n_new - s, to j when p <= j < m - s and eq(j, j), and to nothing otherwise; old draw objects likewise from their side.
// It preserves order: the prefix pairs lie below m - s on both sides, the middle pairs are positional inside [p, m - s), and
// the suffix pairs lie at or above n_old - s and n_new - s, both at least m - s; inside each part the pairing is a shift. Every
// pair is equal by construction, and each index is paired at most once, from both sides alike. When n_old == n_new the suffix
// pass is the position pass, so only eq(k, k) is computed and j is matched to j exactly when eq(j, j).
//
// The tables this builds are k_recompose_damage's with one draw object per instance (identity draw prefixes), so that kernel
// ORs the damage unchanged: the boxes of unmatched draw objects (old boxes from the base frame, copied at the upload; new ones
// from this frame) and both boxes of matched ones whose clipped boxes differ. Nothing here depends on the arenas, so a re-run
// after an overflow builds the same tables.
#include "vb_device.cuh"
#include "vb_stages.h"

#define UD_THREADS 256u

// the byte at index i of a tag stream
__device__ __forceinline__ uint32_t ud_tag_byte(const uint32_t *__restrict__ tags, uint32_t i) {
    return (__ldg(tags + (i >> 2)) >> ((i & 3u) * 8u)) & 0xffu;
}

// The byte index of path p's TAG_PATH: the last tag word whose exclusive path count is at most p holds it.
__device__ __forceinline__ uint32_t ud_path_end(const uint32_t *__restrict__ tags, const VbTagMonoid *tm, uint32_t n_words, uint32_t p) {
    uint32_t lo = 0u, hi = n_words - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (tm[mid].path_ix <= p) lo = mid;
        else hi = mid - 1u;
    }
    const uint32_t word = __ldg(tags + lo);
    uint32_t k = p - tm[lo].path_ix, at = lo * 4u + 3u;
#pragma unroll
    for (uint32_t i = 0; i < 4u; i++) {
        const bool path = ((word >> (i * 8u)) & 0x10u) != 0u;
        if (path && k == 0u) at = min(at, lo * 4u + i);
        if (path) k--;
    }
    return at;
}

// The exclusive tag monoid at byte x (x up to 4 * n_words): transforms, path data words and style words before it.
__device__ __forceinline__ void ud_excl(const uint32_t *__restrict__ tags, const VbTagMonoid *tm, uint32_t n_words, uint32_t x, uint32_t &trans,
                                        uint32_t &off, uint32_t &style) {
    uint32_t wi = x >> 2, mask = (1u << ((x & 3u) * 8u)) - 1u;
    if (wi >= n_words) {
        wi = n_words - 1u;
        mask = 0xffffffffu;
    }
    const uint32_t w = __ldg(tags + wi) & mask;
    // reduce_tag (k_pathtag.cu) of the bytes below x in its word
    const uint32_t point_count = w & 0x3030303u;
    const uint32_t n_points = point_count + ((w >> 2) & 0x1010101u);
    uint32_t a = n_points + (n_points & (((w >> 3) & 0x1010101u) * 15u));
    a += a >> 8;
    a += a >> 16;
    const VbTagMonoid base = tm[wi];
    trans = base.trans_ix + __popc(w & (0x20u * 0x1010101u));
    off = base.pathseg_offset + (a & 0xffu);
    style = base.style_ix + __popc(w & (0x40u * 0x1010101u)) * 2u;
}

// One thread per draw object: its record (VbUdRec) from the scene's draw tags and its tag and draw monoids.
__global__ void __launch_bounds__(UD_THREADS)
k_upload_records(const uint32_t *__restrict__ scene, uint32_t path_tag_base, uint32_t draw_tag_base, uint32_t n_words, uint32_t n_draw,
                 const VbTagMonoid *tm, const VbDrawMonoid *dm, VbUdRec *out, uint32_t *init, uint32_t m) {
    const uint32_t i = blockIdx.x * UD_THREADS + threadIdx.x;
    if (init && i == 0u) {
        init[0] = m;
        init[1] = m;
    }
    if (i >= n_draw) return;
    VbUdRec r;
    r.dtag = __ldg(scene + draw_tag_base + i);
    const VbDrawMonoid d = dm[i];
    r.dd = d.scene_offset;
    r.tag0 = r.tag1 = r.pd0 = r.pd1 = r.t0 = r.t1 = r.s0 = r.s1 = 0u;
    if (r.dtag != VB_DRAWTAG_NOP && n_words != 0u) { // a NOP owns no path
        const uint32_t *tags = scene + path_tag_base, p = d.path_ix;
        const uint32_t b = ud_path_end(tags, tm, n_words, p);
        const uint32_t a = p ? min(ud_path_end(tags, tm, n_words, p - 1u) + 1u, b) : 0u;
        uint32_t ta, oa, sa, tb, ob, sb, te, oe, se;
        ud_excl(tags, tm, n_words, a, ta, oa, sa);
        ud_excl(tags, tm, n_words, b, tb, ob, sb);
        ud_excl(tags, tm, n_words, b + 1u, te, oe, se);
        // a tag at byte x reads transform (transforms before x) - 1 and style words from (style words before x) - 2
        r.tag0 = a;
        r.tag1 = b + 1u;
        r.pd0 = oa;
        r.pd1 = max(oe, oa);
        r.t0 = ta ? ta - 1u : 0u;
        r.t1 = max(tb, r.t0);
        r.s0 = sa >= 2u ? sa - 2u : 0u;
        r.s1 = max(sb, r.s0);
    }
    out[i] = r;
}

__device__ __forceinline__ bool ud_gradient(uint32_t tag) {
    return tag == VB_DRAWTAG_FILL_LIN_GRADIENT || tag == VB_DRAWTAG_FILL_RAD_GRADIENT || tag == VB_DRAWTAG_FILL_SWEEP_GRADIENT;
}

// eq(old a, new b) for the whole warp: every lane returns the same answer.
__device__ bool ud_eq(const VbUdSide &O, const VbUdSide &N, const VbUdRec &a, const VbUdRec &b, uint32_t lane) {
    if (a.dtag != b.dtag || a.tag1 - a.tag0 != b.tag1 - b.tag0 || a.pd1 - a.pd0 != b.pd1 - b.pd0 || a.t1 - a.t0 != b.t1 - b.t0 ||
        a.s1 - a.s0 != b.s1 - b.s0)
        return false;
    const uint32_t FULL = 0xffffffffu;
    const uint32_t *os = O.scene, *ns = N.scene;
    const uint32_t odd = O.layout.draw_data_base + a.dd, ndd = N.layout.draw_data_base + b.dd, n_dd = (a.dtag >> 2) & 7u;
    const bool grad = ud_gradient(a.dtag);
    bool ok = true;
    if (lane < n_dd) {
        const uint32_t x = __ldg(os + odd + lane), y = __ldg(ns + ndd + lane);
        ok = grad && lane == 0u ? (x & 3u) == (y & 3u) : x == y; // a gradient's ramp row may differ
    }
    if (!__all_sync(FULL, ok)) return false;
    if (grad) {
        const uint32_t ro = __ldg(os + odd) >> 2, rn = __ldg(ns + ndd) >> 2;
        if (ro >= O.n_ramps || rn >= N.n_ramps) return false;
        const uint32_t *po = O.ramps + (size_t)ro * 512u, *pn = N.ramps + (size_t)rn * 512u;
        for (uint32_t t = lane; t < 512u; t += 32u) ok &= __ldg(po + t) == __ldg(pn + t);
    } else if (a.dtag == VB_DRAWTAG_FILL_IMAGE && n_dd >= 2u) {
        const uint32_t xy = __ldg(os + odd), wh = __ldg(os + odd + 1u); // equal on both sides
        const uint32_t x = xy >> 16, y = xy & 0xffffu, w = wh >> 16, h = wh & 0xffffu;
        if (x + w > O.atlas_w || y + h > O.atlas_h || x + w > N.atlas_w || y + h > N.atlas_h) return false;
        const uint32_t *ao = (const uint32_t *)O.atlas, *an = (const uint32_t *)N.atlas;
        for (uint32_t k = lane; k < w * h; k += 32u) {
            const uint32_t row = y + k / w, col = x + k % w;
            ok &= __ldg(ao + (size_t)row * O.atlas_w + col) == __ldg(an + (size_t)row * N.atlas_w + col);
        }
    }
    if (!__all_sync(FULL, ok)) return false;
    for (uint32_t k = lane; k < a.tag1 - a.tag0; k += 32u)
        ok &= ud_tag_byte(os + O.layout.path_tag_base, a.tag0 + k) == ud_tag_byte(ns + N.layout.path_tag_base, b.tag0 + k);
    if (!__all_sync(FULL, ok)) return false;
    for (uint32_t k = lane; k < a.pd1 - a.pd0; k += 32u)
        ok &= __ldg(os + O.layout.path_data_base + a.pd0 + k) == __ldg(ns + N.layout.path_data_base + b.pd0 + k);
    if (!__all_sync(FULL, ok)) return false;
    for (uint32_t k = lane; k < (a.t1 - a.t0) * 6u; k += 32u)
        ok &= __ldg(os + O.layout.transform_base + a.t0 * 6u + k) == __ldg(ns + N.layout.transform_base + b.t0 * 6u + k);
    for (uint32_t k = lane; k < a.s1 - a.s0; k += 32u)
        ok &= __ldg(os + O.layout.style_base + a.s0 + k) == __ldg(ns + N.layout.style_base + b.s0 + k);
    return __all_sync(FULL, ok);
}

// One warp per pair: the m pairs by position, then (n_old != n_new) the m pairs from the end. eq[k] = eq(k, k); the first
// unequal pair of each pass bounds the prefix and the suffix.
__global__ void __launch_bounds__(UD_THREADS)
k_upload_eq(VbUdiff *h, const VbUdRec *__restrict__ old_rec, const VbUdRec *__restrict__ new_rec, uint32_t *eq, uint32_t n_old, uint32_t n_new) {
    const uint32_t w = blockIdx.x * (UD_THREADS / 32u) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    const uint32_t m = min(n_old, n_new), pairs = n_old != n_new ? 2u * m : m;
    if (w >= pairs) return;
    const bool pos = w < m;
    const uint32_t k = pos ? w : w - m, i = pos ? k : n_old - 1u - k, j = pos ? k : n_new - 1u - k;
    const bool e = ud_eq(h->old_side, h->new_side, old_rec[i], new_rec[j], lane);
    if (lane != 0u) return;
    if (pos) eq[k] = e ? 1u : 0u;
    if (!e) atomicMin(pos ? &h->prefix : &h->suffix, k);
}

// One thread per index up to max(n_old, n_new): k_recompose_damage's tables (vb_rcmp_tables).
__global__ void __launch_bounds__(UD_THREADS)
k_upload_tables(const VbUdiff *h, const uint32_t *__restrict__ eq, uint32_t *tables, uint32_t n_old, uint32_t n_new) {
    const uint32_t t = blockIdx.x * UD_THREADS + threadIdx.x;
    if (t > max(n_old, n_new)) return;
    const uint32_t m = min(n_old, n_new);
    uint32_t s = 0u; // n_old == n_new: the position pass decides alone
    if (n_old != n_new) {
        const uint32_t p = min(h->prefix, m);
        s = min(h->suffix, m - p);
    }
    const VbRcmpTables<uint32_t> T = vb_rcmp_tables(tables, n_old, n_new);
    if (t <= n_old) T.old_pre[t] = t;
    if (t <= n_new) T.new_pre[t] = t;
    // the prefix lies inside [0, m - s) with eq set, so the middle's rule covers it
    if (t < n_new) T.map[t] = t >= n_new - s ? t + n_old - n_new : t < m - s && eq[t] ? t : VB_RCMP_NONE;
    if (t < n_old) T.unmatched[t] = t >= n_old - s || (t < m - s && eq[t]) ? 0u : 1u;
}

extern "C" uint32_t vb_launch_upload_records(const uint32_t *scene, uint32_t path_tag_base, uint32_t draw_tag_base, uint32_t n_tag_words,
                                             uint32_t n_draw, const VbTagMonoid *tag_monoids, const VbDrawMonoid *draw_monoids, VbUdRec *out,
                                             uint32_t *init, uint32_t m, cudaStream_t st) {
    if (n_draw == 0u && !init) return 0u;
    const uint32_t blocks = n_draw ? (n_draw + UD_THREADS - 1u) / UD_THREADS : 1u;
    k_upload_records<<<blocks, UD_THREADS, 0, st>>>(scene, path_tag_base, draw_tag_base, n_tag_words, n_draw, tag_monoids, draw_monoids, out, init, m);
    return 1u;
}

extern "C" uint32_t vb_launch_upload_diff(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (!b.dmg.udiff) return 0u;
    const uint32_t n_old = b.dmg.n_old, n_new = b.dmg.n_new, m = n_old < n_new ? n_old : n_new;
    const VbUdLayout U = vb_udiff_layout(n_old, n_new);
    char *base = (char *)b.dmg.udiff;
    const VbUdRec *old_rec = (const VbUdRec *)(base + U.old_rec);
    VbUdRec *new_rec = (VbUdRec *)(base + U.new_rec);
    uint32_t *eq = (uint32_t *)(base + U.eq), *tables = (uint32_t *)(base + U.tables);
    uint32_t launches = vb_launch_upload_records(b.scene, cfg.layout.path_tag_base, cfg.layout.draw_tag_base, cfg.n_tag_words, n_new, b.tag_monoids,
                                                 b.draw_monoids, new_rec, &b.dmg.udiff->prefix, m, st);
    const uint32_t pairs = n_old != n_new ? 2u * m : m, per = UD_THREADS / 32u;
    if (pairs) {
        k_upload_eq<<<(pairs + per - 1u) / per, UD_THREADS, 0, st>>>(b.dmg.udiff, old_rec, new_rec, eq, n_old, n_new);
        launches++;
    }
    const uint32_t n = (n_old > n_new ? n_old : n_new) + 1u;
    k_upload_tables<<<(n + UD_THREADS - 1u) / UD_THREADS, UD_THREADS, 0, st>>>(b.dmg.udiff, eq, tables, n_old, n_new);
    return launches + 1u;
}
