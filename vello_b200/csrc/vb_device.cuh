// vb_device.cuh -- device-side building blocks shared by the stage kernels.
//
//  * warp-shuffle scans (32-wide warps; no shared-memory log-step scans as in the WGSL)
//  * single-pass "decoupled look-back" prefix over a K-field u32 monoid, a sum unless another is given (Merrill & Garland):
//    partitions take a ticket (so partition p only waits on partitions that already started),
//    publish {aggregate | inclusive prefix} descriptors, and warp 0 walks the predecessors 32 at
//    a time. This replaces the reference's 2-3 dispatch reduce/scan chains
//    (pathtag_reduce -> reduce2 -> scan1 -> scan, draw_reduce -> draw_leaf) with one pass and
//    makes bump allocation DETERMINISTIC where the reference uses atomicAdd order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vb_types.h"

#define VB_WARP 32
#define VB_FULL 0xffffffffu

__device__ __forceinline__ uint32_t vb_lane() { return threadIdx.x & 31u; }

__device__ __forceinline__ uint32_t vb_warp_incl_scan(uint32_t v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(VB_FULL, v, o);
        if ((int)vb_lane() >= o) v += t;
    }
    return v;
}
__device__ __forceinline__ uint32_t vb_warp_sum(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(VB_FULL, v, o);
    return v;
}

// Block-wide exclusive scan of one u32 per thread; returns the exclusive prefix, writes the block
// total to *total. `sh` must hold (blockDim.x / 32 + 1) words. All threads must call.
__device__ __forceinline__ uint32_t vb_block_excl_scan(uint32_t v, uint32_t *sh, uint32_t *total) {
    uint32_t incl = vb_warp_incl_scan(v);
    uint32_t w = threadIdx.x >> 5, nw = (blockDim.x + 31u) >> 5;
    if (vb_lane() == 31u) sh[w] = incl;
    __syncthreads();
    if (w == 0) {
        uint32_t x = vb_lane() < nw ? sh[vb_lane()] : 0u;
        uint32_t xi = vb_warp_incl_scan(x);
        if (vb_lane() < nw) sh[vb_lane()] = xi - x;
        if (vb_lane() == 31u) sh[nw] = xi;
    }
    __syncthreads();
    uint32_t r = sh[w] + incl - v;
    *total = sh[nw];
    __syncthreads();
    return r;
}

// ---- decoupled look-back ------------------------------------------------------------------
// Global state for one scan: [ticket][flags: n_parts][agg: n_parts*K][pref: n_parts*K].
// ticket + flags must be zero before the kernel starts (one cudaMemsetAsync per frame).
struct VbLookback {
    uint32_t *ticket, *flags, *agg, *pref;
};
__host__ __device__ inline size_t vb_lookback_words(uint32_t n_parts, int K) { return 1u + (size_t)n_parts * (1u + 2u * K); }
__host__ __device__ inline VbLookback vb_lookback_view(uint32_t *base, uint32_t n_parts, int K) {
    VbLookback s;
    s.ticket = base;
    s.flags = base + 1;
    s.agg = s.flags + n_parts;
    s.pref = s.agg + (size_t)n_parts * K;
    return s;
}
#define VB_LB_ZERO_WORDS(n_parts) (1u + (n_parts)) /* leading words that need zeroing */

__device__ __forceinline__ uint32_t vb_ld_flag(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void vb_st_flag(uint32_t *p, uint32_t v) {
    asm volatile("st.release.gpu.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Take the next partition index (call from all threads; `sh_ticket` is one shared word).
__device__ __forceinline__ uint32_t vb_take_ticket(const VbLookback &s, uint32_t *sh_ticket) {
    if (threadIdx.x == 0) *sh_ticket = atomicAdd(s.ticket, 1u);
    __syncthreads();
    uint32_t t = *sh_ticket;
    __syncthreads();
    return t;
}

// The monoid of a look-back: K u32 words whose identity is all zeros, and combine(a, b, r): r = a (+) b, where a is the
// earlier operand (r may alias a or b). The default is the field-wise sum.
struct VbSumOp {
    static constexpr bool commutative = true;
    template <int K> __device__ __forceinline__ static void combine(const uint32_t (&a)[K], const uint32_t (&b)[K], uint32_t (&r)[K]) {
#pragma unroll
        for (int k = 0; k < K; k++) r[k] = a[k] + b[k];
    }
};
// backdrop's look-back monoid (k_backdrop): [0] crossings, [1] a row starts in the range (0 / 1), [2] backdrop deltas summed
// from the range's last row start on (all of them without one). The last two form a segmented sum: associative, not
// commutative.
struct BdSegOp {
    static constexpr bool commutative = false;
    template <int K> __device__ __forceinline__ static void combine(const uint32_t (&a)[K], const uint32_t (&b)[K], uint32_t (&r)[K]) {
        static_assert(K == 3, "BdSegOp has three words");
        const uint32_t c = a[0] + b[0], f = a[1] | b[1], s = b[1] ? b[2] : a[2] + b[2];
        r[0] = c;
        r[1] = f;
        r[2] = s;
    }
};
// Warp reduction of a non-commutative monoid in which a HIGHER lane holds an EARLIER element: every lane ends with
// v[31] (+) v[30] (+) ... (+) v[0]. After the step of width o, a lane holds its aligned block of 2o lanes.
template <int K, class Op> __device__ __forceinline__ void vb_warp_reduce_rev(uint32_t (&v)[K]) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t p[K];
#pragma unroll
        for (int k = 0; k < K; k++) p[k] = __shfl_xor_sync(VB_FULL, v[k], o);
        if (vb_lane() & (uint32_t)o) Op::combine(v, p, v); // my block is the earlier one
        else Op::combine(p, v, v);
    }
}

// Must be called by ALL threads of warp 0 (other warps skip it). `agg` = this partition's
// aggregate (same value in every lane). On return `excl` = the combination of all earlier partitions, in partition order.
// A non-commutative Op is reduced in that order: lane 0 of a window holds the nearest predecessor, the cutoff lane the
// inclusive prefix of the earliest one.
template <int K, class Op = VbSumOp>
__device__ __forceinline__ void vb_lookback(const VbLookback &s, uint32_t part, const uint32_t (&agg)[K], uint32_t (&excl)[K]) {
    const uint32_t lane = vb_lane();
#pragma unroll
    for (int k = 0; k < K; k++) excl[k] = 0u;
    if (lane == 0) {
        uint32_t *dst = (part == 0 ? s.pref : s.agg) + (size_t)part * K;
#pragma unroll
        for (int k = 0; k < K; k++) dst[k] = agg[k];
        vb_st_flag(s.flags + part, part == 0 ? 2u : 1u);
    }
    if (part == 0) return;
    int idx = (int)part - 1;
    for (;;) {
        int my = idx - (int)lane;
        uint32_t f = 2u;
        if (my >= 0) {
            do { f = vb_ld_flag(s.flags + my); } while (f == 0u);
        }
        uint32_t pm = __ballot_sync(VB_FULL, f == 2u); // lanes holding an inclusive prefix (or before the start)
        int cutoff = pm ? (__ffs(pm) - 1) : 32;
        uint32_t v[K];
#pragma unroll
        for (int k = 0; k < K; k++) v[k] = 0u;
        if ((int)lane <= cutoff && my >= 0) {
            const uint32_t *src = ((int)lane == cutoff ? s.pref : s.agg) + (size_t)my * K;
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = src[k];
        }
        if constexpr (Op::commutative) {
#pragma unroll
            for (int k = 0; k < K; k++) excl[k] += vb_warp_sum(v[k]);
        } else {
            vb_warp_reduce_rev<K, Op>(v);
            Op::combine(v, excl, excl); // this window lies before the nearer ones already in excl
        }
        if (pm) break;
        idx -= 32;
    }
    if (lane == 0) {
        uint32_t *dst = s.pref + (size_t)part * K;
        uint32_t incl[K];
        Op::combine(excl, agg, incl);
#pragma unroll
        for (int k = 0; k < K; k++) dst[k] = incl[k];
        vb_st_flag(s.flags + part, 2u);
    }
}

// ---- misc -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t vb_f2u_sat(float f) { return __float2uint_rz(f); }  // saturating, NaN -> 0
__device__ __forceinline__ int32_t vb_f2i_sat(float f) { return __float2int_rz(f); }    // saturating, NaN -> 0
__device__ __forceinline__ float vb_signf(float x) { return (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f); }
__device__ __forceinline__ float vb_clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ int32_t vb_clampi(int32_t x, int32_t lo, int32_t hi) { return min(max(x, lo), hi); }
__device__ __forceinline__ uint32_t vb_span(float a, float b) {
    return vb_f2u_sat(fmaxf(ceilf(fmaxf(a, b)) - floorf(fminf(a, b)), 1.0f));
}
__device__ __forceinline__ uint32_t vb_scene(const uint32_t *__restrict__ scene, const VbConfig &cfg, uint32_t ix) {
    return ix < cfg.scene_words ? __ldg(scene + ix) : 0u;
}
// Batch: the cell of draw object `ix`, the last c with cell_draw[c] <= ix (empty cells are skipped: cell_draw[c + 1] > ix).
__device__ __forceinline__ uint32_t vb_cell_of(const VbConfig &cfg, uint32_t ix) {
    uint32_t lo = 0u, hi = cfg.n_cells; // cell_draw[lo] <= ix < cell_draw[hi]
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(cfg.cell_draw + mid) <= ix) lo = mid;
        else hi = mid;
    }
    return lo;
}
