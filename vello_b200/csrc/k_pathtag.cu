// k_pathtag.cu -- path tag monoid scan (replaces pathtag_reduce / reduce2 / scan1 / scan).
//
// Reference: vello_shaders/shader/pathtag_reduce.wgsl:21-42, pathtag_scan.wgsl:28-76,
// shared/pathtag.wgsl:58-71 (reduce_tag bit magic), vello_encoding/src/path.rs:334-364.
// Output: tag_monoids[w] = exclusive prefix of the 5-field monoid before tag word w (20 B each),
// bit-identical to the reference's.
//
// Design: ONE pass. A CTA takes a ticket, scans 1024 tag words (256 threads x 4 words) with
// warp shuffles, publishes its aggregate and resolves its prefix by decoupled look-back.
// Algorithmic traffic: 4 B read + 20 B written per tag word (HBM-bound, no tensor cores).
#include "vb_device.cuh"
#include "vb_stages.h"

#define PT_THREADS 256
#define PT_WORDS_PER_THREAD 4
#define PT_PART (PT_THREADS * PT_WORDS_PER_THREAD)

__device__ __forceinline__ void pt_reduce_tag(uint32_t tag_word, uint32_t (&m)[5]) {
    uint32_t point_count = tag_word & 0x3030303u;
    m[1] = __popc((point_count * 7u) & 0x4040404u);                 // pathseg_ix
    m[0] = __popc(tag_word & (0x20u * 0x1010101u));                 // trans_ix
    uint32_t n_points = point_count + ((tag_word >> 2) & 0x1010101u);
    uint32_t a = n_points + (n_points & (((tag_word >> 3) & 0x1010101u) * 15u));
    a += a >> 8;
    a += a >> 16;
    m[2] = a & 0xffu;                                               // pathseg_offset
    m[4] = __popc(tag_word & (0x10u * 0x1010101u));                 // path_ix
    m[3] = __popc(tag_word & (0x40u * 0x1010101u)) * 2u;            // style_ix
}

__global__ void __launch_bounds__(PT_THREADS)
k_pathtag_scan(VbConfig cfg, const uint32_t *__restrict__ scene, VbTagMonoid *__restrict__ tag_monoids, uint32_t *lb_mem,
               uint32_t n_parts) {
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_warp[5][PT_THREADS / 32];
    __shared__ uint32_t sh_prefix[5];
    VbLookback lb = vb_lookback_view(lb_mem, n_parts, 5);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t n_words = cfg.n_tag_words;
    const uint32_t w0 = part * PT_PART + threadIdx.x * PT_WORDS_PER_THREAD;

    uint32_t words[PT_WORDS_PER_THREAD];
    uint32_t local[PT_WORDS_PER_THREAD][5];
    uint32_t tsum[5] = {0, 0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < PT_WORDS_PER_THREAD; i++) {
        uint32_t w = w0 + i;
        words[i] = w < n_words ? __ldg(scene + cfg.layout.path_tag_base + w) : 0u;
        pt_reduce_tag(words[i], local[i]);
#pragma unroll
        for (int k = 0; k < 5; k++) tsum[k] += local[i][k];
    }
    // inclusive scan of the per-thread sums across the CTA (warp shuffles + 8 warp totals)
    uint32_t incl[5];
#pragma unroll
    for (int k = 0; k < 5; k++) incl[k] = vb_warp_incl_scan(tsum[k]);
    const uint32_t warp = threadIdx.x >> 5, lane = vb_lane();
    if (lane == 31) {
#pragma unroll
        for (int k = 0; k < 5; k++) sh_warp[k][warp] = incl[k];
    }
    __syncthreads();
    uint32_t woff[5], agg[5];
#pragma unroll
    for (int k = 0; k < 5; k++) {
        uint32_t o = 0, t = 0;
#pragma unroll
        for (int w = 0; w < PT_THREADS / 32; w++) {
            uint32_t x = sh_warp[k][w];
            if ((uint32_t)w < warp) o += x;
            t += x;
        }
        woff[k] = o;
        agg[k] = t;
    }
    if (warp == 0) {
        uint32_t excl[5];
        vb_lookback<5>(lb, part, agg, excl);
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 5; k++) sh_prefix[k] = excl[k];
        }
    }
    __syncthreads();
    uint32_t run[5];
#pragma unroll
    for (int k = 0; k < 5; k++) run[k] = sh_prefix[k] + woff[k] + incl[k] - tsum[k];
#pragma unroll
    for (int i = 0; i < PT_WORDS_PER_THREAD; i++) {
        uint32_t w = w0 + i;
        if (w < n_words) {
            VbTagMonoid m = {run[0], run[1], run[2], run[3], run[4]};
            tag_monoids[w] = m;
        }
#pragma unroll
        for (int k = 0; k < 5; k++) run[k] += local[i][k];
    }
}

extern "C" uint32_t vb_launch_pathtag(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (b.parts_pathtag == 0) return 0;
    k_pathtag_scan<<<b.parts_pathtag, PT_THREADS, 0, st>>>(cfg, b.scene, b.tag_monoids, b.lb_pathtag, b.parts_pathtag);
    return 1;
}
extern "C" uint32_t vb_pathtag_parts(uint32_t n_tag_words) { return (n_tag_words + PT_PART - 1) / PT_PART; }
