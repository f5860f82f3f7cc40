// k_points.cu -- bound path points (vb_bind_path_points): every frame reads point k of the scene's path data, for k below the
// bound count, from row k of a device array, read when the frame runs.
//
// No pipeline kernel changes for it. Path data is read in one place, flatten's read_f32_point, through the frame's
// layout.path_data_base. prepare (vb_frame.cu) points that at a region past the scene's streams, and k_path_points writes the
// whole path-data stream there at the start of flatten's stage: the scene's words, with the words of each bound point replaced
// by its row's bits. Flatten then derives path boxes, culling, lines and everything after them from the bound points. The tags
// never change while rows are bound (every scene installation unbinds), so k_path_point_slots finds each path's first point
// once, at bind time, with a scan of the path tags (a composed or device-resolved scene's tags exist only on the device); damage
// tracking (k_damage.cu) maps a changed point to its path with it. The same walk finds each path's transform range for bound
// transforms (k_transforms.cu).
#include "vb_device.cuh"
#include "vb_stages.h"

#define PP_THREADS 256u
#define PP_SLOT_THREADS 1024u

// The path-data words of the tag bytes of `w`: the pathseg_offset field of the path tag monoid (k_pathtag.cu's pt_reduce_tag).
// A segment of type t reads t new points, one more when it ends a subpath, two words each for an F32 segment.
__device__ __forceinline__ uint32_t pp_words(uint32_t w) {
    const uint32_t n_points = (w & 0x3030303u) + ((w >> 2) & 0x1010101u);
    uint32_t a = n_points + (n_points & (((w >> 3) & 0x1010101u) * 15u));
    a += a >> 8;
    a += a >> 16;
    return a & 0xffu;
}

// One CTA walks the tag words a chunk at a time: the exclusive scans of their path-data words, TAG_PATH bytes and TRANSFORM
// bytes give, at each tag byte, the point, path and transform it is at. At the TAG_PATH byte that ends path p:
//  - with `first`, the first point of path p + 1. first[0] = 0 and first[n_paths] is the scene's point count, so path p owns
//    points first[p] .. first[p + 1]. *i16 is 1 when a segment tag lacks the F32 bit (its points are not f32 pairs).
//  - with `xf_range` (bound transforms), xf_range[p].y = t_hi(p), the transform in effect there: the one draw reads for the
//    path's brush (pathtag's path_draw). xf_range[p].x = t_lo(p) is the transform in effect at the path's first segment tag,
//    the least one flatten reads for its segments (transforms only grow along the tags, so it is the least over the segment
//    bytes: the first segment byte of each path in each tag word takes an atomicMin). A path with no segment gets t_lo = t_hi.
//    The caller sets xf_range to all ones first. The transform in effect at a byte is the TRANSFORM bytes before it, minus 1,
//    as flatten's compute_tag_monoid counts it.
__global__ void __launch_bounds__(PP_SLOT_THREADS) k_path_point_slots(const uint32_t *__restrict__ tags, uint32_t n_words, uint32_t n_paths,
                                                                      uint32_t *first, uint32_t *i16, uint2 *xf_range) {
    __shared__ uint32_t sh[PP_SLOT_THREADS / 32u + 1u];
    uint32_t off0 = 0u, path0 = 0u, xf0 = 0u;
    int any_i16 = 0;
    for (uint32_t c = 0u; c < n_words; c += PP_SLOT_THREADS) {
        const uint32_t k = c + threadIdx.x;
        const uint32_t w = k < n_words ? __ldg(tags + k) : 0u;
        uint32_t off_total = 0u, path_total, xf_total = 0u;
        const uint32_t path = path0 + vb_block_excl_scan(__popc(w & 0x10101010u), sh, &path_total);
        if (first) {
            const uint32_t off = off0 + vb_block_excl_scan(pp_words(w), sh, &off_total);
            const uint32_t seg = (w | (w >> 1)) & 0x1010101u; // bytes with a segment type
            any_i16 |= __syncthreads_or((seg & ~(w >> 3)) != 0u);
            uint32_t opens = w & 0x10101010u;
            while (opens != 0u) {
                const uint32_t shift = (uint32_t)(__ffs((int)opens) - 1) & ~7u;
                opens &= opens - 1u;
                const uint32_t p = path + __popc(w & ((1u << shift) - 1u) & 0x10101010u);
                const uint32_t upto = shift == 24u ? 0xffffffffu : (1u << (shift + 8u)) - 1u; // the bytes through this TAG_PATH
                if (p < n_paths) first[p + 1u] = (off + pp_words(w & upto)) >> 1;
            }
        }
        if (xf_range) {
            uint32_t t = xf0 + vb_block_excl_scan(__popc(w & 0x20202020u), sh, &xf_total), p = path;
            bool seen = false; // a segment byte of path p earlier in this word
#pragma unroll
            for (uint32_t b = 0u; b < 4u; b++) {
                const uint32_t tag = (w >> (8u * b)) & 0xffu;
                if ((tag & 3u) != 0u && !seen) {
                    if (p < n_paths) atomicMin(&xf_range[p].x, t - 1u);
                    seen = true;
                }
                if (tag & 0x10u) {
                    if (p < n_paths) xf_range[p].y = t - 1u;
                    p++;
                    seen = false;
                }
                if (tag & 0x20u) t++;
            }
        }
        off0 += off_total;
        path0 += path_total;
        xf0 += xf_total;
    }
    if (first && threadIdx.x == 0u) {
        first[0] = 0u;
        *i16 = any_i16 ? 1u : 0u;
    }
    if (xf_range) {
        __syncthreads();
        for (uint32_t p = threadIdx.x; p < n_paths; p += PP_SLOT_THREADS) {
            const uint2 r = xf_range[p];
            if (r.x > r.y) xf_range[p].x = r.y;
        }
    }
}

// One thread per point k of the path data: the scene's two words, or below n the row's bits when both are finite, so that no
// NaN or infinity reaches flatten. Bits are copied, never converted: a bound frame reads exactly the words a host-patched
// upload holds.
__global__ void __launch_bounds__(PP_THREADS) k_path_points(const uint8_t *__restrict__ rows, uint32_t pitch, uint32_t n, const uint32_t *__restrict__ src,
                                                            uint32_t *dst, uint32_t n_words) {
    const uint32_t k = blockIdx.x * PP_THREADS + threadIdx.x;
    const uint32_t u = 2u * k;
    if (u >= n_words) return;
    uint32_t x = __ldg(src + u), y = u + 1u < n_words ? __ldg(src + u + 1u) : 0u;
    if (k < n) {
        const uint32_t *row = reinterpret_cast<const uint32_t *>(rows + (size_t)k * pitch);
        const uint32_t rx = __ldg(row), ry = __ldg(row + 1);
        const uint32_t E = 0x7f800000u; // an all-ones exponent: infinity or NaN
        if ((rx & E) != E && (ry & E) != E) {
            x = rx;
            y = ry;
        }
    }
    dst[u] = x;
    if (u + 1u < n_words) dst[u + 1u] = y;
}

extern "C" uint32_t vb_launch_path_point_slots(const uint32_t *tags, uint32_t n_words, uint32_t n_paths, uint32_t *first, uint32_t *i16,
                                               uint2 *xf_range, cudaStream_t st) {
    k_path_point_slots<<<1, PP_SLOT_THREADS, 0, st>>>(tags, n_words, n_paths, first, i16, xf_range);
    return 1u;
}

extern "C" uint32_t vb_launch_path_points(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbRows &rows = b.bound.rows[VB_BIND_POINTS];
    if (!rows.rows) return 0u;
    // the region prepare reserved past the scene's streams, the last one
    const uint32_t n_words = b.pd_len;
    if (n_words == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + cfg.layout.path_data_base;
    const uint32_t n_points = (n_words + 1u) / 2u;
    k_path_points<<<(n_points + PP_THREADS - 1u) / PP_THREADS, PP_THREADS, 0, st>>>(rows.rows, rows.pitch, rows.n, b.pt_src, dst, n_words);
    return 1u;
}
