// k_clip.cu -- clip stack resolution (replaces clip_reduce + clip_leaf).
//
// Reference: vello_shaders/shader/clip_reduce.wgsl:24-67, clip_leaf.wgsl:37-217 (bicyclic-semigroup
// tree search, stack depth <= 256: clip_leaf.wgsl:102 TODO), CPU twin cpu/clip_leaf.rs (sequential
// stack, unlimited depth). Outputs are the reference's: clip_bboxes[i] and the patched
// draw_monoids of EndClip objects (clip_leaf.wgsl:195-213).
//
// Design: the matching problem is restated as "nearest position to the left whose depth is
// <= v" on the depth sequence B (B[i] = number of open clips before op i):
//   * the BeginClip matching an EndClip at i is the last j < i with B[j] <= B[i] - 1;
//   * the enclosing BeginClip of a BeginClip at i is the last j < i with B[j] <= B[i] - 1.
// B comes from one CTA-wide scan; the query walks a 3-level min hierarchy (32 / 1024 / rest).
// Any nesting depth is supported (the reference's GPU path stops at 256), results identical
// to the CPU shader for every depth.
#include "vb_device.cuh"
#include "vb_stages.h"

#define CL_THREADS 1024

// Depth sequence B (exclusive scan of +1 / -1) and its 32 / 1024 minima. One CTA per 1024 clip ops; the carry between CTAs
// comes from the single-pass decoupled look-back of vb_device.cuh (K = 1), so a million clip ops are a thousand CTAs, not a
// thousand passes of one CTA (round 1: k_clip_depth<<<1, 1024>>>).
__global__ void __launch_bounds__(CL_THREADS)
k_clip_depth(uint32_t n_clips, const VbClipInp *__restrict__ clip_inp, int32_t *B, int32_t *min32, int32_t *min1024, uint32_t *lb_mem,
             uint32_t n_parts) {
    __shared__ uint32_t sh_scan[CL_THREADS / 32 + 2];
    __shared__ int32_t sh_min[CL_THREADS / 32];
    __shared__ uint32_t sh_ticket;
    __shared__ uint32_t sh_carry;
    const VbLookback lb = vb_lookback_view(lb_mem, n_parts, 1);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    if (part >= n_parts) return;
    const uint32_t base = part * CL_THREADS;
    const uint32_t i = base + threadIdx.x;
    uint32_t v = 0;
    if (i < n_clips) v = clip_inp[i].path_ix >= 0 ? 1u : 0xffffffffu;
    uint32_t total;
    const uint32_t ex = vb_block_excl_scan(v, sh_scan, &total);
    if (threadIdx.x < 32u) {
        uint32_t agg[1] = {total}, excl[1];
        vb_lookback<1>(lb, part, agg, excl);
        if (threadIdx.x == 0u) sh_carry = excl[0];
    }
    __syncthreads();
    const int32_t b = (int32_t)(sh_carry + ex);
    if (i < n_clips) B[i] = b;
    int32_t m = i < n_clips ? b : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(VB_FULL, m, o));
    if (vb_lane() == 0) {
        if (base + (threadIdx.x & ~31u) < n_clips) min32[(base + threadIdx.x) >> 5] = m;
        sh_min[threadIdx.x >> 5] = m;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        int32_t mm = sh_min[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mm = min(mm, __shfl_xor_sync(VB_FULL, mm, o));
        if (threadIdx.x == 0) min1024[part] = mm;
    }
}

__device__ __forceinline__ int cl_scan_group(const int32_t *__restrict__ B, int g, int n, int32_t v) {
    for (int j = min(g * 32 + 31, n - 1); j >= g * 32; j--)
        if (B[j] <= v) return j;
    return -1;
}
// max j < i with B[j] <= v, or -1
__device__ int cl_last_le(const int32_t *__restrict__ B, const int32_t *__restrict__ min32, const int32_t *__restrict__ min1024,
                          int n, int i, int32_t v) {
    int j = i - 1;
    while (j >= 0 && (j & 31) != 31) {
        if (B[j] <= v) return j;
        j--;
    }
    int g = j >> 5; // j == -1 -> g == -1
    while (g >= 0 && (g & 31) != 31) {
        if (min32[g] <= v) return cl_scan_group(B, g, n, v);
        g--;
    }
    int h = g >> 5;
    while (h >= 0) {
        if (min1024[h] <= v) {
            for (int g2 = h * 32 + 31; g2 >= h * 32; g2--)
                if (g2 * 32 < n && min32[g2] <= v) return cl_scan_group(B, g2, n, v);
        }
        h--;
    }
    return -1;
}

__global__ void k_clip_link(uint32_t n_clips, const VbClipInp *__restrict__ clip_inp, const int32_t *__restrict__ B,
                            const int32_t *__restrict__ min32, const int32_t *__restrict__ min1024, int32_t *link) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_clips) return;
    // push: enclosing push; pop: matching push. Both are "last j < i with B[j] <= B[i] - 1".
    int32_t b = B[i];
    link[i] = b > 0 ? cl_last_le(B, min32, min1024, (int)n_clips, (int)i, b - 1) : -1;
}

__device__ __forceinline__ VbBbox4 cl_path_bbox(const VbPathBbox *__restrict__ pbs, int32_t path_ix) {
    VbPathBbox pb = pbs[path_ix];
    VbBbox4 r = {(float)pb.x0, (float)pb.y0, (float)pb.x1, (float)pb.y1};
    return r;
}
__device__ __forceinline__ VbBbox4 cl_chain_bbox(const VbClipInp *__restrict__ clip_inp, const VbPathBbox *__restrict__ pbs,
                                                 const int32_t *__restrict__ link, int32_t i) {
    VbBbox4 b = cl_path_bbox(pbs, clip_inp[i].path_ix);
    for (int32_t p = link[i]; p >= 0; p = link[p]) {
        VbBbox4 q = cl_path_bbox(pbs, clip_inp[p].path_ix);
        b.x0 = fmaxf(b.x0, q.x0); b.y0 = fmaxf(b.y0, q.y0);
        b.x1 = fminf(b.x1, q.x1); b.y1 = fminf(b.y1, q.y1);
    }
    return b;
}

__global__ void k_clip_bbox(uint32_t n_clips, const VbClipInp *__restrict__ clip_inp, const VbPathBbox *__restrict__ pbs,
                            const int32_t *__restrict__ link, VbDrawMonoid *draw_monoids, VbBbox4 *clip_bboxes) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_clips) return;
    VbClipInp el = clip_inp[i];
    const VbBbox4 big = {-1e9f, -1e9f, 1e9f, 1e9f};
    if (el.path_ix >= 0) {
        clip_bboxes[i] = cl_chain_bbox(clip_inp, pbs, link, (int32_t)i);
    } else {
        int32_t j = link[i];
        if (j < 0) { clip_bboxes[i] = big; return; } // unbalanced pop: never produced by the encoder
        int32_t parent = link[j];
        clip_bboxes[i] = parent >= 0 ? cl_chain_bbox(clip_inp, pbs, link, parent) : big;
        VbClipInp begin = clip_inp[j];
        VbDrawMonoid bm = draw_monoids[begin.ix];
        draw_monoids[el.ix].path_ix = (uint32_t)begin.path_ix;
        draw_monoids[el.ix].scene_offset = bm.scene_offset;
        draw_monoids[el.ix].info_offset = bm.info_offset;
    }
}

extern "C" uint32_t vb_clip_parts(uint32_t n_clips) { return (n_clips + CL_THREADS - 1u) / CL_THREADS; }
extern "C" uint32_t vb_launch_clip(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const uint32_t n_clips = cfg.layout.n_clips;
    if (n_clips == 0) return 0;
    int32_t *B = b.clip_scratch; // B | min32 | min1024 | link
    int32_t *min32 = B + n_clips;
    int32_t *min1024 = min32 + (n_clips + 31) / 32;
    int32_t *link = min1024 + (n_clips + 1023) / 1024;
    const uint32_t n_parts = vb_clip_parts(n_clips);
    k_clip_depth<<<n_parts, CL_THREADS, 0, st>>>(n_clips, b.clip_inp, B, min32, min1024, b.lb_clip, n_parts);
    k_clip_link<<<(n_clips + 255) / 256, 256, 0, st>>>(n_clips, b.clip_inp, B, min32, min1024, link);
    k_clip_bbox<<<(n_clips + 255) / 256, 256, 0, st>>>(n_clips, b.clip_inp, b.path_bboxes, link, b.draw_monoids, b.clip_bboxes);
    return 3;
}
extern "C" size_t vb_clip_scratch_words(uint32_t n_clips) {
    return (size_t)n_clips * 2 + (n_clips + 31) / 32 + (n_clips + 1023) / 1024 + 8;
}
