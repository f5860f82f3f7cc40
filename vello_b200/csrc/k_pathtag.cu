// k_pathtag.cu -- path tag monoid scan (replaces pathtag_reduce / reduce2 / scan1 / scan).
//
// Reference: vello_shaders/shader/pathtag_reduce.wgsl:21-42, pathtag_scan.wgsl:28-76,
// shared/pathtag.wgsl:58-71 (reduce_tag bit magic), vello_encoding/src/path.rs:334-364.
// Output: tag_monoids[w] = exclusive prefix of the 5-field monoid before tag word w (20 B each),
// bit-identical to the reference's.
//
// Design: ONE pass. A CTA takes a ticket, scans PT_PART tag words (256 threads x PT_WORDS_PER_THREAD words, loaded as
// 16-byte vectors) with warp shuffles, publishes its aggregate and resolves its prefix by decoupled look-back. The
// partition's monoids are staged in shared memory and stored as consecutive 16-byte words across the CTA: written straight
// from registers, a thread's consecutive 20-byte monoids put the 32 lanes of one store 20 * PT_WORDS_PER_THREAD bytes apart.
// Algorithmic traffic: 4 B read + 20 B written per tag word (HBM-bound, no tensor cores).
//
// It also writes the path table draw reads (path_draw[path_ix] = {style_ix, trans_ix} of every PATH tag: where draw finds
// the draw flags and transform that flatten's fl_open_path stores in the path's bbox), so that draw does not wait for
// flatten. Draw reads the style word itself: a load here would wait for the look-back, on the critical path.
#include "vb_device.cuh"
#include "vb_stages.h"

#define PT_THREADS 256
#ifndef PT_WORDS_PER_THREAD
#define PT_WORDS_PER_THREAD 8
#endif
#define PT_PART (PT_THREADS * PT_WORDS_PER_THREAD)
#define PT_VEC (PT_WORDS_PER_THREAD / 4)        // 16-byte tag loads per thread
#define PT_OUT_VEC (PT_PART * 5 / 4)             // 16-byte words of a partition's monoids
static_assert(PT_WORDS_PER_THREAD % 4 == 0, "a thread's tag words are loaded as whole 16-byte vectors");
static_assert(PT_PART * 20 <= 48 * 1024, "the staged monoids fit static shared memory");

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

// The path table entry of every PATH tag (bit 0x10) of `word`, whose exclusive prefix is `run`: its transform is the last one
// before it and its style the one the tag's path uses, as flatten's compute_tag_monoid / fl_open_path find them.
__device__ __forceinline__ void pt_open_paths(const VbConfig &cfg, uint2 *__restrict__ path_draw, uint32_t word, const uint32_t (&run)[5]) {
    uint32_t opens = word & (0x10u * 0x1010101u);
    while (opens != 0u) {
        const uint32_t shift = (uint32_t)(__ffs((int)opens) - 1) & ~7u;
        opens &= opens - 1u;
        const uint32_t below = word & ((1u << shift) - 1u);
        const uint32_t path_ix = run[4] + __popc(below & (0x10u * 0x1010101u));
        if (path_ix >= cfg.layout.n_paths) continue;
        const uint32_t trans_ix = run[0] + __popc(below & (0x20u * 0x1010101u)) - 1u;
        const uint32_t style_ix = run[3] + __popc(below & (0x40u * 0x1010101u)) * 2u - 2u;
        path_draw[path_ix] = make_uint2(style_ix, trans_ix);
    }
}

__global__ void __launch_bounds__(PT_THREADS)
k_pathtag_scan(VbConfig cfg, const uint32_t *__restrict__ scene, VbTagMonoid *__restrict__ tag_monoids, uint2 *__restrict__ path_draw,
               uint32_t *lb_mem, uint32_t n_parts) {
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_warp[5][PT_THREADS / 32];
    __shared__ uint32_t sh_prefix[5];
    __shared__ uint4 sh_out[PT_OUT_VEC];
    VbLookback lb = vb_lookback_view(lb_mem, n_parts, 5);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    const uint32_t n_words = cfg.n_tag_words;
    const uint32_t part_w0 = part * PT_PART;
    const uint32_t w0 = part_w0 + threadIdx.x * PT_WORDS_PER_THREAD;
    const uint32_t *tags = scene + cfg.layout.path_tag_base;

    uint32_t words[PT_WORDS_PER_THREAD];
    if ((cfg.layout.path_tag_base & 3u) == 0u && w0 + PT_WORDS_PER_THREAD <= n_words) {
#pragma unroll
        for (int v = 0; v < PT_VEC; v++) {
            const uint4 q = __ldg(reinterpret_cast<const uint4 *>(tags + w0) + v);
            words[4 * v] = q.x; words[4 * v + 1] = q.y; words[4 * v + 2] = q.z; words[4 * v + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < PT_WORDS_PER_THREAD; i++) words[i] = w0 + i < n_words ? __ldg(tags + w0 + i) : 0u;
    }
    uint32_t tsum[5] = {0, 0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < PT_WORDS_PER_THREAD; i++) {
        uint32_t m[5];
        pt_reduce_tag(words[i], m);
#pragma unroll
        for (int k = 0; k < 5; k++) tsum[k] += m[k];
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
    // this thread's monoids, 5 words each, as 16-byte words of the staging area (20 * PT_WORDS_PER_THREAD bytes apart)
    uint32_t out[PT_WORDS_PER_THREAD * 5];
#pragma unroll
    for (int i = 0; i < PT_WORDS_PER_THREAD; i++) {
#pragma unroll
        for (int k = 0; k < 5; k++) out[5 * i + k] = run[k];
        if ((words[i] & (0x10u * 0x1010101u)) != 0u) pt_open_paths(cfg, path_draw, words[i], run);
        uint32_t m[5];
        pt_reduce_tag(words[i], m);
#pragma unroll
        for (int k = 0; k < 5; k++) run[k] += m[k];
    }
    uint4 *mine = sh_out + threadIdx.x * (PT_WORDS_PER_THREAD * 5 / 4);
#pragma unroll
    for (int j = 0; j < PT_WORDS_PER_THREAD * 5 / 4; j++) mine[j] = make_uint4(out[4 * j], out[4 * j + 1], out[4 * j + 2], out[4 * j + 3]);
    __syncthreads();
    // the partition's monoids are 20 * n_valid bytes from tag_monoids + part_w0: whole 16-byte words, then 0..3 words
    const uint32_t n_valid = min(n_words - part_w0, (uint32_t)PT_PART);
    const uint32_t n_vec = n_valid * 5u / 4u;
    uint4 *dst = reinterpret_cast<uint4 *>(tag_monoids + part_w0);
    for (uint32_t j = threadIdx.x; j < n_vec; j += PT_THREADS) dst[j] = sh_out[j];
    const uint32_t n_tail = n_valid * 5u - n_vec * 4u;
    if (threadIdx.x < n_tail) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(sh_out) + n_vec * 4u;
        reinterpret_cast<uint32_t *>(dst + n_vec)[threadIdx.x] = src[threadIdx.x];
    }
}

extern "C" uint32_t vb_launch_pathtag(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    if (b.parts_pathtag == 0) return 0;
    k_pathtag_scan<<<b.parts_pathtag, PT_THREADS, 0, st>>>(cfg, b.scene, b.tag_monoids, b.path_draw, b.lb_pathtag, b.parts_pathtag);
    return 1;
}
extern "C" uint32_t vb_pathtag_parts(uint32_t n_tag_words) { return (n_tag_words + PT_PART - 1) / PT_PART; }
