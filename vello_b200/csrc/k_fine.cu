// k_fine.cu -- fine rasterisation: interpret each tile's PTCL and write RGBA8 pixels.
//
// Reference: vello_shaders/shader/fine.wgsl (area coverage :1005-1059, MSAA :146-709, interpreter
// :1064-1398), shared/blend.wgsl, mask LUTs vello_encoding/src/mask.rs. The reference has no CPU
// fine; our oracle (oracle/vbo_fine.c) restates the WGSL and this kernel must match it bit for bit
// (MSAA: integer sample counts -> exact; area: float sums in slice order).
//
// Design (v3): PERSISTENT WARPS, ONE WARP PER TILE, TMA-STAGED COMMAND WINDOWS.
//  * The grid is sized to the machine (2 CTAs of FI_MAX_WARPS warps per SM) and every warp pulls tile indices from a
//    global queue (one atomic per tile, issued two tiles ahead), so a long tile no longer idles the other warp
//    slots of its CTA (v2 launched one two-warp CTA per pair of tiles).
//  * The half-plane mask LUT (8 KB for MSAA16) is copied ONCE per CTA into shared memory with one bulk copy
//    (cp.async.bulk + mbarrier, the TMA path; v2 fetched it with __ldg per pixel touch).
//  * Each warp owns two 256-byte command windows in shared memory. A window is filled by one bulk copy signalled on
//    the warp's mbarrier; while a tile is being painted the NEXT tile's window is already in flight, so the
//    interpreter reads its commands from shared memory (v2: one dependent global round trip per command).
//    A window is re-staged when the command pointer leaves it (lists longer than ~60 words, CMD_JUMP).
//  * A warp owns the tile (lane = 8 horizontally adjacent pixels = two of the WGSL's 4-pixel groups, so every
//    per-group float expression is unchanged); all synchronisation is __syncwarp / shuffles / ballots. The MSAA
//    state stays CLEAN between fills and is initialised once per warp, not per tile. Pixels that receive sample
//    masks are appended to a per-fill list by the first lane that touches them (atomicOr on a 256-bit map returns
//    the old word); the resolve then handles ONE TOUCHED PIXEL PER LANE -- instead of every lane walking its 8
//    pixels through a divergent branch -- and untouched pixels are decided 4 at a time with SWAR byte compares on
//    the winding words. The integer arithmetic per touched pixel is the WGSL's, word for word.
//  * Each tile starts at its occlusion start (the last opaque full-tile cover, noted by coarse).
//  * The lane's 8 pixels (rgba[8], area[8]: 40 registers) are only ever indexed by compile-time constants, so they live in
//    registers for the whole tile; the rarely used brushes that loop over them without unrolling work on a copy. (A dynamically
//    indexed loop once kept them in local memory, and that local traffic was the top stall of the kernel.)
// Conventions fixed where WGSL leaves latitude: see oracle/vbo_fine.c.
// Algorithmic bytes: 4 B/pixel stored + 4 B per PTCL word + 24 B per segment referenced.
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "vb_detmath.h"
#include "vb_device.cuh"
#include "vb_stages.h"

#ifndef FI_MAX_WARPS
#define FI_MAX_WARPS 10 // warps (= tiles in flight) per CTA; the launcher picks 2..FI_MAX_WARPS by frame size. 2 CTAs x 10 warps leave
                        // 102 registers per thread: the 8 pixels of a lane (32 colour + 8 coverage registers) stay in registers
#endif
#ifndef FI_MINB
#define FI_MINB 2
#endif
#define FI_MAX_THREADS (32 * FI_MAX_WARPS)
// k_fine_solid: FI_SOLID_MINB CTAs of FI_SOLID_WARPS warps per SM, 24 resident warps at 80 registers. Measured on the headline
// frame (H100 SXM, 700 W): 16 warps at 64 registers and 14 at 72 hold more warps but spill the pixels around the fill, and
// paint slower (DESIGN §8).
#ifndef FI_SOLID_WARPS
#define FI_SOLID_WARPS 12
#endif
#ifndef FI_SOLID_MINB
#define FI_SOLID_MINB 2
#endif
#define PX 8                       // pixels per lane
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define GRADIENT_WIDTH 512
#define WIN_WORDS 64u              // command window: 256 bytes

struct rgba_t { float r, g, b, a; };
__device__ __forceinline__ rgba_t RG(float r, float g, float b, float a) { rgba_t c; c.r = r; c.g = g; c.b = b; c.a = a; return c; }
__device__ __forceinline__ rgba_t rg_scale(rgba_t c, float s) { return RG(c.r * s, c.g * s, c.b * s, c.a * s); }
__device__ __forceinline__ rgba_t unpack4x8unorm(uint32_t u) {
    return RG((float)(u & 0xffu) / 255.0f, (float)((u >> 8) & 0xffu) / 255.0f, (float)((u >> 16) & 0xffu) / 255.0f,
              (float)(u >> 24) / 255.0f);
}
__device__ __forceinline__ uint32_t unorm8(float x) { return (uint32_t)floorf(0.5f + 255.0f * fminf(1.0f, fmaxf(0.0f, x))); }
__device__ __forceinline__ uint32_t pack4x8unorm(rgba_t c) {
    return unorm8(c.r) | (unorm8(c.g) << 8) | (unorm8(c.b) << 16) | (unorm8(c.a) << 24);
}
__device__ __forceinline__ rgba_t over(rgba_t bg, rgba_t fg) {
    float k = 1.0f - fg.a;
    return RG(fmaf(bg.r, k, fg.r), fmaf(bg.g, k, fg.g), fmaf(bg.b, k, fg.b), fmaf(bg.a, k, fg.a)); // explicit FMA (see oracle)
}

// byte / 255.0f for the warp-uniform unpacks (CMD_COLOR, base colour): filled on the host with the same IEEE
// division, so values are identical to unpack4x8unorm()'s.
__constant__ float c_unorm[256];
__device__ __forceinline__ rgba_t unpack4x8unorm_uniform(uint32_t u) {
    return RG(c_unorm[u & 0xffu], c_unorm[(u >> 8) & 0xffu], c_unorm[(u >> 16) & 0xffu], c_unorm[u >> 24]);
}

struct FineArgs {
    const VbSegment *segments;
    const uint32_t *ptcl;
    const uint32_t *info;
    uint32_t *blend_spill;
    uint32_t *out; // RGBA8 packed, r in the low byte
    const uint32_t *ramps;
    const uint8_t *atlas;
    const uint32_t *mask_lut;
    const VbBump *bump;         // bump.failed != 0: an upstream stage overflowed an arena, nothing to paint (fine.wgsl:1070)
    const uint32_t *tile_start; // per tile: PTCL offset of its last opaque full-tile cover, or 0 (written by coarse)
    uint32_t *queue;            // tile queue of this launch (zero at launch; see the tile loop)
    const uint2 *cls_list;      // cost-ordered tile lists written by coarse: VB_FINE_CLASSES x cls_stride entries {tile, start}
    const uint32_t *cls_count;  // their fill counts (control block); NULL: natural tile order
    uint32_t cls_stride;
    uint32_t cull;              // 1: start each tile there
    uint32_t lists;             // FI_LISTS_*: which of those lists the launch walks
};
// The arguments of the FI_DST instantiations: FineArgs, then a registered destination's (vb_launch_fine's VbFineOut): the
// __byte_perm selector of the stored byte order, the texel size (4: 8-bit, 8: RGBA16F, 16: RGBA32F), premultiplied or straight
// alpha, and either linear memory at `out` or, with `array`, the surface of a CUDA array, pixel (x, y) of the frame at texel
// (x0 + x, y0 + y). The other instantiations take FineArgs alone, so that their code is exactly what it was before destinations
// existed (a larger parameter block alone changes ptxas's register assignment).
struct FineDstArgs : FineArgs {
    cudaSurfaceObject_t surf;
    uint32_t swz, array, x0, y0, texel, premul;
};
// The arguments of the FI_BG instantiations: FineDstArgs, then the background every tile starts from (vb_set_background).
struct FineBgArgs : FineDstArgs {
    VbFineBg bg;
};

// The store of a float destination (FI_DST, texel 8 or 16), for a lane's PX pixels at frame row gy, columns gx..gx+7 (gx a
// multiple of 8). Each texel is clamp01 (unorm8's clamp, NaN to 0) of the premultiplied pixel, or of its straight colour
// rgb * (1 / max(a, 1e-6)) and alpha: the values the 8-bit store rounds. When every pixel of the warp is opaque the factor is
// exactly 1 and is skipped, as there. RGBA16F rounds them to nearest even halves. cfg.out_pitch_px is the pitch in texels.
__device__ __forceinline__ float clamp01(float x) { return fminf(1.0f, fmaxf(0.0f, x)); }
__device__ __forceinline__ uint32_t half2_bits(float lo, float hi) {
    return (uint32_t)__half_as_ushort(__float2half_rn(lo)) | ((uint32_t)__half_as_ushort(__float2half_rn(hi)) << 16);
}
__device__ __forceinline__ void store_float(const FineDstArgs &A, const VbConfig &cfg, rgba_t (&rgba)[PX], uint32_t gx, uint32_t gy,
                                            bool all_opaque) {
    const bool straight = A.premul == 0u && !all_opaque;
#pragma unroll
    for (int i = 0; i < PX; i++) {
        const rgba_t c = rgba[i];
        const float k = straight ? 1.0f / fmaxf(c.a, 1e-6f) : 1.0f;
        rgba[i] = straight ? RG(clamp01(c.r * k), clamp01(c.g * k), clamp01(c.b * k), clamp01(c.a))
                           : RG(clamp01(c.r), clamp01(c.g), clamp01(c.b), clamp01(c.a));
    }
    const bool full = gx + 7u < cfg.target_width;
    const uint32_t x = A.x0 + gx, y = A.y0 + gy;
    char *row = (char *)A.out + (size_t)(gy - cfg.out_row0) * cfg.out_pitch_px * A.texel;
    if (A.texel == 16u) {
        // one 128-bit store per texel: the registered pointer and pitch are multiples of 16
#pragma unroll
        for (int i = 0; i < PX; i++) {
            if (!full && gx + i >= cfg.target_width) continue;
            const float4 v = make_float4(rgba[i].r, rgba[i].g, rgba[i].b, rgba[i].a);
            if (A.array) surf2Dwrite(v, A.surf, (int)((x + i) * 16u), (int)y, cudaBoundaryModeZero);
            else reinterpret_cast<float4 *>(row)[gx + i] = v;
        }
        return;
    }
    uint2 t[PX];
#pragma unroll
    for (int i = 0; i < PX; i++) t[i] = make_uint2(half2_bits(rgba[i].r, rgba[i].g), half2_bits(rgba[i].b, rgba[i].a));
    if (full && (A.array ? (x & 1u) == 0u : (cfg.out_pitch_px & 1u) == 0u && ((uintptr_t)A.out & 15u) == 0u)) {
        // four 128-bit stores of two texels each: the lane's 64 contiguous bytes
#pragma unroll
        for (int i = 0; i < PX; i += 2) {
            const uint4 v = make_uint4(t[i].x, t[i].y, t[i + 1].x, t[i + 1].y);
            if (A.array) surf2Dwrite(v, A.surf, (int)((x + i) * 8u), (int)y, cudaBoundaryModeZero);
            else reinterpret_cast<uint4 *>(row)[(gx + i) / 2u] = v;
        }
    } else {
#pragma unroll
        for (int i = 0; i < PX; i++) {
            if (gx + i >= cfg.target_width) continue;
            if (A.array) surf2Dwrite(t[i], A.surf, (int)((x + i) * 8u), (int)y, cudaBoundaryModeZero);
            else reinterpret_cast<uint2 *>(row)[gx + i] = t[i];
        }
    }
}

// The background's texels of a lane's PX pixels (FI_BG), frame row gy of cell `cell`, columns gx..gx+7, as stored: pixel i's in
// w[i] (8-bit formats), w[2i..2i+1] (RGBA16F) or w[4i..4i+3] (RGBA32F). A pixel right of the frame reads nothing and stays 0.
// Plain (coherent) loads, never the non-coherent path: the background may be the destination, which this kernel writes. A lane
// reads its 8 pixels with 128-bit loads where the row is 16-byte aligned, or through the array's surface in 16-byte texel groups.
__device__ __forceinline__ void load_bg_texels(const VbFineBg &B, const VbConfig &cfg, uint32_t cell, uint32_t gx, uint32_t gy,
                                               uint32_t (&w)[4 * PX]) {
#pragma unroll
    for (int k = 0; k < 4 * PX; k++) w[k] = 0u;
    const bool full = gx + 7u < cfg.target_width;
    const uint32_t T = B.texel;
    if (B.array) {
        const uint32_t x = B.x0 + gx;
        const int y = (int)(B.y0 + gy);
        if (full && (x & (16u / T - 1u)) == 0u) {
#pragma unroll
            for (int k = 0; k < 8; k++) {
                if ((uint32_t)k * 16u >= PX * T) break;
                const uint4 v = surf2Dread<uint4>(B.surf, (int)(x * T + (uint32_t)k * 16u), y, cudaBoundaryModeZero);
                w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < PX; i++) {
                if (gx + i >= cfg.target_width) continue;
                const int bx = (int)((x + i) * T);
                if (T == 16u) {
                    const uint4 v = surf2Dread<uint4>(B.surf, bx, y, cudaBoundaryModeZero);
                    w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
                } else if (T == 8u) {
                    const uint2 v = surf2Dread<uint2>(B.surf, bx, y, cudaBoundaryModeZero);
                    w[2 * i] = v.x; w[2 * i + 1] = v.y;
                } else {
                    w[i] = surf2Dread<uint32_t>(B.surf, bx, y, cudaBoundaryModeZero);
                }
            }
        }
        return;
    }
    const uint8_t *row = B.ptr + ((size_t)cell * cfg.target_height + gy) * B.pitch + (size_t)gx * T;
    if (full && ((uintptr_t)row & 15u) == 0u) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if ((uint32_t)k * 16u >= PX * T) break;
            const uint4 v = __ldcg(reinterpret_cast<const uint4 *>(row) + k);
            w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < PX; i++) {
            if (gx + i >= cfg.target_width) continue;
            if (T == 16u) {
                const uint4 v = __ldcg(reinterpret_cast<const uint4 *>(row) + i);
                w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
            } else if (T == 8u) {
                const uint2 v = __ldcg(reinterpret_cast<const uint2 *>(row) + i);
                w[2 * i] = v.x; w[2 * i + 1] = v.y;
            } else {
                w[i] = __ldcg(reinterpret_cast<const unsigned int *>(row) + i);
            }
        }
    }
}
// The background's pixels as fine's starting pixels: each channel as f32 (byte / 255.0f with r and b swapped back for BGRA8, the
// half converted exactly, the float as stored), clamp01 of it (the store's clamp: NaN gives 0, and nothing outside [0, 1] enters
// the blend arithmetic), then for straight alpha (r * a, g * a, b * a, a), each product rounded on its own.
__device__ __forceinline__ void load_bg(const VbFineBg &B, const VbConfig &cfg, uint32_t cell, uint32_t gx, uint32_t gy, rgba_t (&rgba)[PX]) {
    uint32_t w[4 * PX];
    load_bg_texels(B, cfg, cell, gx, gy, w);
#pragma unroll
    for (int i = 0; i < PX; i++) {
        rgba_t c;
        if (B.texel == 16u) {
            c = RG(__uint_as_float(w[4 * i]), __uint_as_float(w[4 * i + 1]), __uint_as_float(w[4 * i + 2]), __uint_as_float(w[4 * i + 3]));
        } else if (B.texel == 8u) {
            c = RG(__half2float(__ushort_as_half((unsigned short)(w[2 * i] & 0xffffu))), __half2float(__ushort_as_half((unsigned short)(w[2 * i] >> 16))),
                   __half2float(__ushort_as_half((unsigned short)(w[2 * i + 1] & 0xffffu))),
                   __half2float(__ushort_as_half((unsigned short)(w[2 * i + 1] >> 16))));
        } else {
            c = unpack4x8unorm(w[i]);
            if (B.bgra) c = RG(c.b, c.g, c.r, c.a);
        }
        c = RG(clamp01(c.r), clamp01(c.g), clamp01(c.b), clamp01(c.a));
        rgba[i] = B.premul ? c : RG(c.r * c.a, c.g * c.a, c.b * c.a, c.a);
    }
}

// ---------------- mbarrier + bulk-copy (TMA) primitives: PTX as in cute/arch/copy_sm90_tma.hpp, cutlass/arch/barrier.h ----------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0u;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// global -> shared bulk copy (16-byte aligned addresses, size a multiple of 16), completion counted on `bar`
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ VbSegment ld_segment(const VbSegment *__restrict__ segs, uint32_t ix) {
    const uint2 *p = reinterpret_cast<const uint2 *>(segs + ix);
    uint2 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2);
    VbSegment s;
    s.p0[0] = __uint_as_float(a.x); s.p0[1] = __uint_as_float(a.y);
    s.p1[0] = __uint_as_float(b.x); s.p1[1] = __uint_as_float(b.y);
    s.y_edge = __uint_as_float(c.x);
    s._pad = 0;
    return s;
}
// ---------------- area coverage: fine.wgsl:1005-1059 ----------------
// lane = row `ly`, pixels 8*h .. 8*h+7 = WGSL thread groups (2h, ly) and (2h+1, ly): xy.x = 4 * group.
__device__ void fill_path_area(const FineArgs &A, uint32_t size_and_rule, uint32_t seg_data, int32_t backdrop, float lx0, float xyy,
                               float (&area)[PX]) {
    const uint32_t n_segs = size_and_rule >> 1;
    const bool even_odd = (size_and_rule & 1u) != 0u;
    const float backdrop_f = (float)backdrop;
#pragma unroll
    for (int i = 0; i < PX; i++) area[i] = backdrop_f;
    for (uint32_t s = 0; s < n_segs; s++) {
        const VbSegment seg = ld_segment(A.segments, seg_data + s);
        const float y = seg.p0[1] - xyy;
        const float deltax = seg.p1[0] - seg.p0[0], deltay = seg.p1[1] - seg.p0[1];
        const float y0 = vb_clampf(y, 0.0f, 1.0f);
        const float y1 = vb_clampf(y + deltay, 0.0f, 1.0f);
        const float dy = y0 - y1;
        if (dy != 0.0f) {
            const float vec_y_recip = 1.0f / deltay;
            const float t0 = (y0 - y) * vec_y_recip;
            const float t1 = (y1 - y) * vec_y_recip;
#pragma unroll
            for (int q = 0; q < 2; q++) {
                const float startx = seg.p0[0] - (lx0 + 4.0f * (float)q);
                const float x0 = startx + t0 * deltax;
                const float x1 = startx + t1 * deltax;
                const float xmin0 = fminf(x0, x1);
                const float xmax0 = fmaxf(x0, x1);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const float i_f = (float)i;
                    const float xmin = fminf(xmin0 - i_f, 1.0f) - 1.0e-6f;
                    const float xmax = xmax0 - i_f;
                    const float b = fminf(xmax, 1.0f);
                    const float c = fmaxf(b, 0.0f);
                    const float d = fmaxf(xmin, 0.0f);
                    const float a = (b + 0.5f * (d * d - c * c) - xmin) / (xmax - xmin);
                    area[q * 4 + i] += a * dy;
                }
            }
        }
        const float y_edge = vb_signf(deltax) * vb_clampf(xyy - seg.y_edge + 1.0f, 0.0f, 1.0f);
#pragma unroll
        for (int i = 0; i < PX; i++) area[i] += y_edge;
    }
    if (even_odd) {
#pragma unroll
        for (int i = 0; i < PX; i++) {
            const float a = area[i];
            area[i] = fabsf(a - 2.0f * rintf(0.5f * a));
        }
    } else {
#pragma unroll
        for (int i = 0; i < PX; i++) area[i] = fminf(fabsf(area[i]), 1.0f);
    }
}

// ---------------- MSAA coverage: fine.wgsl:146-709, one warp per tile ----------------
// Per-warp shared state. INVARIANT between fills (established once per warp by ms_init, restored by every fill):
// samples == 0x80808080 (biased zero), winding == 0x80808080, winding_y == 0x80808080, eo_* == 0, touched == 0.
// The even-odd rule keeps its 16 (8) sample parities in the first word of a pixel's sample group, XORed onto the
// same biased-zero pattern, so the two rules share one array.
template <int AA>
struct WarpMs {
    static constexpr uint32_t WPP = AA == 2 ? 4u : 2u; // sample words per pixel
    uint32_t samples[256 * (AA == 2 ? 4 : 2)];
    uint32_t winding[64];
    uint32_t eo_winding[16];
    uint32_t winding_y[4];
    uint32_t eo_winding_y[4];
    uint32_t touched[8];   // 256-bit map of pixels that received sample masks in the current fill
    uint32_t counts[32];
    uint32_t tb[64];       // one byte per pixel: winding byte (parity) of the pixel, then its resolved sample count
    uint8_t list[256];     // the touched pixels of the current fill, in first-touch order
};
// Per-warp command windows (all AA modes)
struct WarpIo {
    uint32_t ptcl[2][WIN_WORDS];
    uint64_t mbar[2];
};

template <int AA>
__device__ __forceinline__ void ms_init(WarpMs<AA> &S, uint32_t lane) {
    for (uint32_t i = lane; i < 256u * WarpMs<AA>::WPP; i += 32u) S.samples[i] = 0x80808080u;
    S.winding[lane] = 0x80808080u;
    S.winding[lane + 32u] = 0x80808080u;
    if (lane < 16u) S.eo_winding[lane] = 0u;
    if (lane < 4u) { S.winding_y[lane] = 0x80808080u; S.eo_winding_y[lane] = 0u; }
    if (lane < 8u) S.touched[lane] = 0u;
    __syncwarp();
}

// bits 0..3 of `b` -> bytes 0x01 / 0x00 (bit k lands on bit 8k: k + 7k, no two partial products collide)
__device__ __forceinline__ uint32_t bits4_to_bytes(uint32_t b) { return ((b & 0xfu) * 0x00204081u) & 0x01010101u; }
// byte-wise a + b (mod 256 per byte, no carries across bytes)
__device__ __forceinline__ uint32_t byte_add(uint32_t a, uint32_t b) {
    return ((a & 0x7f7f7f7fu) + (b & 0x7f7f7f7fu)) ^ ((a ^ b) & 0x80808080u);
}
// 0x80 in every byte of x that is zero, 0 elsewhere (exact per byte)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu); }

template <int AA> // 1 = msaa8, 2 = msaa16
__device__ void fill_path_ms(const FineArgs &A, WarpMs<AA> &S, const uint32_t *__restrict__ lut, uint32_t size_and_rule, uint32_t seg_data,
                             int32_t backdrop, uint32_t lane, float (&area)[PX]) {
    constexpr uint32_t MASK_WIDTH = AA == 2 ? 64u : 32u;
    constexpr uint32_t MASK_HEIGHT = MASK_WIDTH;
    constexpr uint32_t WPP = WarpMs<AA>::WPP;
    constexpr uint32_t FULL_COUNT = AA == 2 ? 16u : 8u;
    const uint32_t n_segs = size_and_rule >> 1;
    const bool even_odd = (size_and_rule & 1u) != 0u;
    const uint32_t ly = lane >> 1, h = lane & 1u;
    const uint32_t lanemask_lt = (1u << lane) - 1u;
    uint32_t n_touched = 0u; // warp-uniform: pixels in S.list

    // ---- accumulate: batches of 32 segments; every lane first counts its segment's pixel touches, then the
    // touches are spread over the lanes (prefix sum + binary search, as fine.wgsl:196-224)
    for (uint32_t batch_start = 0u; batch_start < n_segs; batch_start += 32u) {
        const uint32_t slice_size = min(n_segs - batch_start, 32u);
        // per-segment line setup, computed ONCE by the owning lane (the WGSL recomputes it for every pixel touch)
        float s_a = 0.f, s_b = 0.f, s_y0i = 0.f, s_xy0y = 0.f, s_xy1y = 0.f;
        int32_t s_x0i = 0;
        uint32_t s_flags = 0u; // bit0 is_down, bit1 is_positive_slope, bit2 xy0.x == 0, bit3 xy1.x != 0, bit4 y0i == xy0.y
        uint32_t count = 0u;
        if (lane < slice_size) {
            const VbSegment seg = ld_segment(A.segments, seg_data + batch_start + lane);
            const float sx0 = seg.p0[0], sy0 = seg.p0[1], sx1 = seg.p1[0], sy1 = seg.p1[1];
            float y_edge_f = 16.0f;
            const int32_t delta = (sx1 <= sx0) ? 1 : -1;
            if (sx0 == 0.0f) y_edge_f = sy0;
            else if (sx1 == 0.0f) y_edge_f = sy1;
            if (!(sy0 == sy1 && sy0 == floorf(sy0))) count = vb_span(sx0, sx1) + vb_span(sy0, sy1) - 1u;
            const uint32_t y_edge = vb_f2u_sat(ceilf(y_edge_f));
            if (y_edge < 16u) {
                if (even_odd) atomicXor(&S.eo_winding_y[0], 1u << y_edge);
                else atomicAdd(&S.winding_y[y_edge >> 2], ((uint32_t)delta) << ((y_edge & 3u) << 3));
            }
            const bool is_down = sy1 >= sy0;
            const float xy0x = is_down ? sx0 : sx1, xy0y = is_down ? sy0 : sy1;
            const float xy1x = is_down ? sx1 : sx0, xy1y = is_down ? sy1 : sy0;
            const float dx = fabsf(xy1x - xy0x);
            const float dy = xy1y - xy0y;
            const float idxdy = 1.0f / (dx + dy);
            float a = dx * idxdy;
            const bool is_positive_slope = xy1x >= xy0x;
            const float x_sign = is_positive_slope ? 1.0f : -1.0f;
            const float xt0 = floorf(xy0x * x_sign);
            const float c = xy0x * x_sign - xt0;
            const float y0i = floorf(xy0y);
            const float ytop = y0i + 1.0f;
            const float b = fminf((dy * c + dx * (ytop - xy0y)) * idxdy, ONE_MINUS_ULP);
            const uint32_t count_x = vb_span(xy0x, xy1x) - 1u;
            const uint32_t count_full = count_x + vb_span(xy0y, xy1y);
            const float robust_err = floorf(a * ((float)count_full - 1.0f) + b) - (float)count_x;
            if (robust_err != 0.0f) a -= ROBUST_EPSILON * vb_signf(robust_err);
            s_a = a; s_b = b; s_y0i = y0i; s_xy0y = xy0y; s_xy1y = xy1y;
            s_x0i = vb_f2i_sat(xt0 * x_sign + 0.5f * (x_sign - 1.0f));
            s_flags = (is_down ? 1u : 0u) | (is_positive_slope ? 2u : 0u) | (xy0x == 0.0f ? 4u : 0u) | (xy1x != 0.0f ? 8u : 0u) |
                      (y0i == xy0y ? 16u : 0u);
        }
        const uint32_t incl = vb_warp_incl_scan(count);
        const uint32_t total = __shfl_sync(VB_FULL, incl, 31);
        S.counts[lane] = incl;
        __syncwarp();
        for (uint32_t base = 0u; base < total; base += 32u) {
            const uint32_t i = base + lane;
            const bool active = i < total;
            uint32_t lo = 0u;
            if (active) {
                uint32_t hi = slice_size;
                while (hi > lo + 1u) {
                    const uint32_t m = (lo + hi) >> 1;
                    if (i >= S.counts[m - 1u]) lo = m; else hi = m;
                }
            }
            const uint32_t el_ix = lo;
            // fetch the owning lane's setup (all lanes take part in the shuffles; inactive lanes compute on lane 0's
            // values and touch no memory)
            const float a = __shfl_sync(VB_FULL, s_a, el_ix), b = __shfl_sync(VB_FULL, s_b, el_ix);
            const float y0i = __shfl_sync(VB_FULL, s_y0i, el_ix);
            const float xy0y = __shfl_sync(VB_FULL, s_xy0y, el_ix), xy1y = __shfl_sync(VB_FULL, s_xy1y, el_ix);
            const int32_t x0i = __shfl_sync(VB_FULL, s_x0i, el_ix);
            const uint32_t fl = __shfl_sync(VB_FULL, s_flags, el_ix);
            const bool is_down = (fl & 1u) != 0u, is_positive_slope = (fl & 2u) != 0u;
            const bool xy0x_zero = (fl & 4u) != 0u, xy1x_nonzero = (fl & 8u) != 0u, y0i_eq = (fl & 16u) != 0u;
            const float x_sign = is_positive_slope ? 1.0f : -1.0f;
            const uint32_t seg_end = S.counts[el_ix];
            const bool last_pixel = i + 1u == seg_end;
            const uint32_t sub_ix = i - (el_ix > 0u ? S.counts[el_ix - 1u] : 0u);
            const float zf = a * (float)sub_ix + b;
            const float z = floorf(zf);
            const int32_t x = x0i + vb_f2i_sat(x_sign * z);
            const int32_t y = vb_f2i_sat(y0i) + (int32_t)sub_ix - vb_f2i_sat(z);
            bool is_delta, is_bump = false;
            if (sub_ix == 0u) {
                is_delta = y0i_eq;
                is_bump = even_odd ? xy0x_zero : (xy0x_zero && !y0i_eq);
            } else {
                const float zp = floorf(a * (float)(sub_ix - 1u) + b);
                is_delta = z == zp;
                is_bump = is_positive_slope && !is_delta;
            }
            const uint32_t pix_ix = (uint32_t)y * 16u + (uint32_t)x;
            if (active && (uint32_t)x < 15u && (uint32_t)y < 16u && is_delta) {
                if (even_odd) {
                    atomicXor(&S.eo_winding[y], 2u << (uint32_t)x);
                } else {
                    const uint32_t delta_pix = pix_ix + 1u;
                    atomicAdd(&S.winding[delta_pix >> 2], (is_down ? 1u : 0xffffffffu) << ((delta_pix & 3u) << 3));
                }
            }
            const uint32_t mask_block = (uint32_t)is_positive_slope * (MASK_WIDTH * MASK_HEIGHT / 2u);
            const float half_height = (float)(MASK_HEIGHT / 2u);
            const float mask_row = floorf(fminf(a * half_height, half_height - 1.0f)) * (float)MASK_WIDTH;
            const float mask_col = floorf((zf - z) * (float)MASK_WIDTH);
            const uint32_t mask_ix = mask_block + vb_f2u_sat(mask_row + mask_col);
            const bool in_tile = active && pix_ix < 256u;
            uint32_t mask;
            if (AA == 1) {
                mask = (lut[(mask_ix / 4u) & 255u] >> ((mask_ix % 4u) * 8u)) & 0xffu;
                if (sub_ix == 0u && !is_bump) {
                    const uint32_t sh = vb_f2u_sat(rintf(8.0f * (xy0y - (float)y)));
                    mask &= sh < 32u ? (0xffu << sh) : 0u;
                }
                if (last_pixel && xy1x_nonzero) {
                    const uint32_t sh = vb_f2u_sat(rintf(8.0f * (xy1y - (float)y)));
                    mask &= ~(sh < 32u ? (0xffu << sh) : 0u);
                }
            } else {
                mask = (lut[(mask_ix / 2u) & 2047u] >> ((mask_ix % 2u) * 16u)) & 0xffffu;
                if (sub_ix == 0u && !is_bump) {
                    const uint32_t sh = vb_f2u_sat(rintf(16.0f * (xy0y - (float)y)));
                    mask &= sh < 32u ? (0xffffu << sh) : 0u;
                }
                if (last_pixel && xy1x_nonzero) {
                    const uint32_t sh = vb_f2u_sat(rintf(16.0f * (xy1y - (float)y)));
                    mask &= ~(sh < 32u ? (0xffffu << sh) : 0u);
                }
            }
            // first lane to touch a pixel appends it to the list (the atomicOr returns the word before this lane's bit)
            const uint32_t bit = 1u << (pix_ix & 31u);
            uint32_t old = ~0u;
            if (in_tile) old = atomicOr(&S.touched[pix_ix >> 5], bit);
            const bool first = (old & bit) == 0u;
            const uint32_t fm = __ballot_sync(VB_FULL, first);
            if (first) S.list[n_touched + __popc(fm & lanemask_lt)] = (uint8_t)pix_ix;
            n_touched += __popc(fm);
            if (in_tile) {
                if (even_odd) {
                    if (is_bump) mask ^= (AA == 1 ? 0xffu : 0xffffu);
                    atomicXor(&S.samples[pix_ix * WPP], mask);
                } else if (AA == 1) {
                    const uint32_t mask_a = mask ^ (mask << 7);
                    const uint32_t mask_b = mask_a ^ (mask_a << 14);
                    const uint32_t m0 = mask_b & 0x1010101u, m1 = (mask_b >> 4) & 0x1010101u;
                    uint32_t m0s = is_down ? (0u - m0) : m0;
                    uint32_t m1s = is_down ? (0u - m1) : m1;
                    if (is_bump) {
                        const uint32_t bd = is_down ? 0x1010101u : (0u - 0x1010101u);
                        m0s += bd; m1s += bd;
                    }
                    atomicAdd(&S.samples[pix_ix * 2u], m0s);
                    atomicAdd(&S.samples[pix_ix * 2u + 1u], m1s);
                } else {
                    const uint32_t mask0 = mask & 0xffu;
                    const uint32_t mask0_a = mask0 ^ (mask0 << 7);
                    const uint32_t mask0_b = mask0_a ^ (mask0_a << 14);
                    const uint32_t e0 = mask0_b & 0x1010101u, e1 = (mask0_b >> 4) & 0x1010101u;
                    const uint32_t mask1 = (mask >> 8) & 0xffu;
                    const uint32_t mask1_a = mask1 ^ (mask1 << 7);
                    const uint32_t mask1_b = mask1_a ^ (mask1_a << 14);
                    const uint32_t e2 = mask1_b & 0x1010101u, e3 = (mask1_b >> 4) & 0x1010101u;
                    uint32_t s0 = is_down ? (0u - e0) : e0, s1 = is_down ? (0u - e1) : e1;
                    uint32_t s2 = is_down ? (0u - e2) : e2, s3 = is_down ? (0u - e3) : e3;
                    if (is_bump) {
                        const uint32_t bd = is_down ? 0x1010101u : (0u - 0x1010101u);
                        s0 += bd; s1 += bd; s2 += bd; s3 += bd;
                    }
                    atomicAdd(&S.samples[pix_ix * 4u], s0);
                    atomicAdd(&S.samples[pix_ix * 4u + 1u], s1);
                    atomicAdd(&S.samples[pix_ix * 4u + 2u], s2);
                    atomicAdd(&S.samples[pix_ix * 4u + 3u], s3);
                }
            }
        }
        __syncwarp();
    }

    // ---- resolve. Row owners (lane = row ly, pixels 8h..8h+7) work out the winding byte / parity of their 8 pixels and
    // the coverage those pixels have if untouched (0 or all samples); touched pixels are then resolved one per lane from
    // the list, and the owners merge the counts back in. cov[q] holds the sample counts of pixels 4q..4q+3, one per byte.
    const uint32_t tbits = (S.touched[ly >> 1] >> ((ly & 1u) * 16u + h * 8u)) & 0xffu;
    uint32_t cov[2];
    uint8_t *tb8 = reinterpret_cast<uint8_t *>(S.tb);
    if (even_odd) {
        uint32_t scan_x = S.eo_winding[ly];
        scan_x ^= scan_x << 1; scan_x ^= scan_x << 2; scan_x ^= scan_x << 4; scan_x ^= scan_x << 8;
        uint32_t scan_y = S.eo_winding_y[0];
        scan_y ^= scan_y << 1; scan_y ^= scan_y << 2; scan_y ^= scan_y << 4; scan_y ^= scan_y << 8;
        const uint32_t row_parity = ((scan_y >> ly) ^ (uint32_t)backdrop) & 1u;
        const uint32_t par8 = ((scan_x >> (h * 8u)) ^ (0u - row_parity)) & 0xffu; // pix_parity of my 8 pixels (fine.wgsl:693)
        const uint32_t pb0 = bits4_to_bytes(par8), pb1 = bits4_to_bytes(par8 >> 4);
        cov[0] = pb0 * FULL_COUNT; // untouched: samples == 0 -> popcount(pix_mask) = all or none
        cov[1] = pb1 * FULL_COUNT;
        if (n_touched != 0u) {
            *reinterpret_cast<uint2 *>(&S.tb[lane * 2u]) = make_uint2(pb0, pb1);
            __syncwarp();
            for (uint32_t j = lane; j < n_touched; j += 32u) {
                const uint32_t pix = S.list[j];
                const uint32_t p = tb8[pix];
                const uint32_t samples = S.samples[pix * WPP] ^ 0x80808080u;
                S.samples[pix * WPP] = 0x80808080u;
                tb8[pix] = (uint8_t)__popc((samples ^ (0u - p)) & (AA == 2 ? 0xffffu : 0xffu));
            }
            __syncwarp();
            if (tbits != 0u) {
                const uint2 c = *reinterpret_cast<const uint2 *>(&S.tb[lane * 2u]);
                const uint32_t m0 = bits4_to_bytes(tbits) * 0xffu, m1 = bits4_to_bytes(tbits >> 4) * 0xffu;
                cov[0] = (cov[0] & ~m0) | (c.x & m0);
                cov[1] = (cov[1] & ~m1) | (c.y & m1);
            }
        }
        __syncwarp();
        if (lane < 16u) S.eo_winding[lane] = 0u;
        if (lane == 0u) S.eo_winding_y[0] = 0u;
        if (lane < 8u) S.touched[lane] = 0u;
    } else {
        // winding of the 4 words of this row, exactly as fine.wgsl:399-425
        uint32_t pw[4], pfx[4];
        {
            const uint4 wr = *reinterpret_cast<const uint4 *>(&S.winding[ly * 4u]);
            const uint32_t wv[4] = {wr.x, wr.y, wr.z, wr.w};
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                uint32_t w = wv[k];
                w += (w - 0x808080u) << 8;
                w += (w - 0x8080u) << 16;
                pw[k] = w;
                pfx[k] = ((w >> 24) - 0x80u) * 0x1010101u;
            }
        }
        uint32_t packed_w[2];
        packed_w[0] = h == 1u ? pw[2] : pw[0]; // selects, not pw[h * 2]: a dynamically indexed array would live in local memory
        packed_w[1] = h == 1u ? pw[3] : pw[1];
        if (h == 1u) { packed_w[0] += pfx[0]; packed_w[0] += pfx[1]; packed_w[1] += pfx[0]; packed_w[1] += pfx[1]; packed_w[1] += pfx[2]; }
        else { packed_w[1] += pfx[0]; }
        uint32_t wind_y;
        {
            const uint4 yr = *reinterpret_cast<const uint4 *>(&S.winding_y[0]);
            const uint32_t yv[4] = {yr.x, yr.y, yr.z, yr.w};
            uint32_t py[4];
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                uint32_t w = yv[k];
                w += (w - 0x808080u) << 8;
                w += (w - 0x8080u) << 16;
                py[k] = w;
            }
            const uint32_t yq = ly >> 2;
            const uint32_t py_sel = yq == 0u ? py[0] : (yq == 1u ? py[1] : (yq == 2u ? py[2] : py[3]));
            wind_y = (py_sel >> ((ly & 3u) << 3)) - 0x80u;
            if (yq > 0u) wind_y += (py[0] >> 24) - 0x80u;
            if (yq > 1u) wind_y += (py[1] >> 24) - 0x80u;
            if (yq > 2u) wind_y += (py[2] >> 24) - 0x80u;
        }
        // t = ((packed_w >> 8i) + wind_y) & 0xff for my 8 pixels (fine.wgsl:447); expected_zero = t - backdrop
        const uint32_t wy = (wind_y & 0xffu) * 0x1010101u;
        const uint32_t tw0 = byte_add(packed_w[0], wy), tw1 = byte_add(packed_w[1], wy);
        // untouched pixel: every sample is the biased zero 0x80, so all samples differ from `expected_zero` unless it IS
        // 0x80 (this includes expected_zero >= 256, which the WGSL maps to full coverage)
        uint32_t z0 = 0u, z1 = 0u;
        if (backdrop >= -128 && backdrop <= 127) {
            const uint32_t tgt = ((uint32_t)(0x80 + backdrop) & 0xffu) * 0x1010101u;
            z0 = zero_bytes(tw0 ^ tgt);
            z1 = zero_bytes(tw1 ^ tgt);
        }
        cov[0] = (~z0 & 0x80808080u) >> (AA == 2 ? 3 : 4);
        cov[1] = (~z1 & 0x80808080u) >> (AA == 2 ? 3 : 4);
        if (n_touched != 0u) {
            *reinterpret_cast<uint2 *>(&S.tb[lane * 2u]) = make_uint2(tw0, tw1);
            __syncwarp();
            for (uint32_t j = lane; j < n_touched; j += 32u) {
                const uint32_t pix = S.list[j];
                const uint32_t expected_zero = (uint32_t)tb8[pix] - (uint32_t)backdrop;
                uint32_t cnt = FULL_COUNT;
                if (AA == 1) {
                    const uint2 sm = *reinterpret_cast<const uint2 *>(&S.samples[pix * 2u]);
                    *reinterpret_cast<uint2 *>(&S.samples[pix * 2u]) = make_uint2(0x80808080u, 0x80808080u);
                    if (expected_zero < 256u) {
                        const uint32_t ez = expected_zero * 0x1010101u;
                        const uint32_t xored0 = ez ^ sm.x;
                        const uint32_t xored0_2 = xored0 | (xored0 * 2u);
                        const uint32_t xored1 = ez ^ sm.y;
                        const uint32_t xored1_2 = xored1 | (xored1 >> 1);
                        const uint32_t xored2 = (xored0_2 & 0xAAAAAAAAu) | (xored1_2 & 0x55555555u);
                        const uint32_t xored4 = xored2 | (xored2 * 4u);
                        const uint32_t xored8 = xored4 | (xored4 * 16u);
                        cnt = __popc(xored8 & 0xC0C0C0C0u);
                    }
                } else {
                    const uint4 sm = *reinterpret_cast<const uint4 *>(&S.samples[pix * 4u]);
                    *reinterpret_cast<uint4 *>(&S.samples[pix * 4u]) = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
                    if (expected_zero < 256u) {
                        const uint32_t ez = expected_zero * 0x1010101u;
                        const uint32_t xored0 = ez ^ sm.x;
                        const uint32_t xored0_2 = xored0 | (xored0 * 2u);
                        const uint32_t xored1 = ez ^ sm.y;
                        const uint32_t xored1_2 = xored1 | (xored1 >> 1);
                        const uint32_t xored01 = (xored0_2 & 0xAAAAAAAAu) | (xored1_2 & 0x55555555u);
                        const uint32_t xored01_4 = xored01 | (xored01 * 4u);
                        const uint32_t xored2 = ez ^ sm.z;
                        const uint32_t xored2_2 = xored2 | (xored2 * 2u);
                        const uint32_t xored3 = ez ^ sm.w;
                        const uint32_t xored3_2 = xored3 | (xored3 >> 1);
                        const uint32_t xored23 = (xored2_2 & 0xAAAAAAAAu) | (xored3_2 & 0x55555555u);
                        const uint32_t xored23_4 = xored23 | (xored23 >> 2);
                        const uint32_t xored4 = (xored01_4 & 0xCCCCCCCCu) | (xored23_4 & 0x33333333u);
                        const uint32_t xored8 = xored4 | (xored4 * 16u);
                        cnt = __popc(xored8 & 0xF0F0F0F0u);
                    }
                }
                tb8[pix] = (uint8_t)cnt;
            }
            __syncwarp();
            if (tbits != 0u) {
                const uint2 c = *reinterpret_cast<const uint2 *>(&S.tb[lane * 2u]);
                const uint32_t m0 = bits4_to_bytes(tbits) * 0xffu, m1 = bits4_to_bytes(tbits >> 4) * 0xffu;
                cov[0] = (cov[0] & ~m0) | (c.x & m0);
                cov[1] = (cov[1] & ~m1) | (c.y & m1);
            }
        }
        __syncwarp();
        S.winding[lane] = 0x80808080u;
        S.winding[lane + 32u] = 0x80808080u;
        if (lane < 4u) S.winding_y[lane] = 0x80808080u;
        if (lane < 8u) S.touched[lane] = 0u;
    }
    __syncwarp();
#pragma unroll
    for (uint32_t i = 0; i < PX; i++)
        area[i] = (float)((cov[i >> 2] >> ((i & 3u) * 8u)) & 0xffu) * (AA == 2 ? 0.0625f : 0.125f);
}

// ---------------- CMD_FILL, CMD_SOLID, CMD_COLOR: the commands both interpreters run (k_fine and k_fine_solid) ----------------
template <int AA>
__device__ __forceinline__ void fine_cmd_fill(const FineArgs &A, WarpMs<AA == 0 ? 1 : AA> &S, const uint32_t *__restrict__ lut, uint32_t sr,
                                              uint32_t sd, int32_t bd, uint32_t lane, float (&area)[PX]) {
    if (AA == 0) fill_path_area(A, sr, sd, bd, (float)((lane & 1u) * 8u), (float)(lane >> 1), area);
    else fill_path_ms<AA == 0 ? 1 : AA>(A, S, lut, sr, sd, bd, lane, area);
}
__device__ __forceinline__ void fine_cmd_solid(float (&area)[PX]) {
#pragma unroll
    for (int i = 0; i < PX; i++) area[i] = 1.0f;
}
__device__ __forceinline__ void fine_cmd_color(uint32_t rgba8, rgba_t (&rgba)[PX], const float (&area)[PX]) {
    const rgba_t fg = unpack4x8unorm_uniform(rgba8);
#pragma unroll
    for (int i = 0; i < PX; i++) rgba[i] = over(rgba[i], rg_scale(fg, area[i]));
}

// ---------------- blend.wgsl ----------------
struct v3 { float x, y, z; };
__device__ __forceinline__ v3 V3(float x, float y, float z) { v3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ float color_dodge(float cb, float cs) {
    if (cb == 0.0f) return 0.0f;
    if (cs == 1.0f) return 1.0f;
    return fminf(1.0f, cb / (1.0f - cs));
}
__device__ float color_burn(float cb, float cs) {
    if (cb == 1.0f) return 1.0f;
    if (cs == 0.0f) return 0.0f;
    return 1.0f - fminf(1.0f, (1.0f - cb) / cs);
}
__device__ __forceinline__ float screen1(float cb, float cs) { return cb + cs - (cb * cs); }
__device__ float hard_light1(float cb, float cs) { return cs <= 0.5f ? cb * 2.0f * cs : screen1(cb, 2.0f * cs - 1.0f); }
__device__ float soft_light1(float cb, float cs) {
    float d = cb <= 0.25f ? ((16.0f * cb - 12.0f) * cb + 4.0f) * cb : sqrtf(cb);
    return cs <= 0.5f ? cb - (1.0f - 2.0f * cs) * cb * (1.0f - cb) : cb + (2.0f * cs - 1.0f) * (d - cb);
}
__device__ __forceinline__ float sat3(v3 c) { return fmaxf(c.x, fmaxf(c.y, c.z)) - fminf(c.x, fminf(c.y, c.z)); }
__device__ __forceinline__ float dot3(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float lum(v3 c) { return dot3(c, V3(0.3f, 0.59f, 0.11f)); }
__device__ __forceinline__ float svg_lum(v3 c) { return dot3(c, V3(0.2125f, 0.7154f, 0.0721f)); }
__device__ v3 clip_color(v3 c) {
    float l = lum(c);
    float n = fminf(c.x, fminf(c.y, c.z));
    float x = fmaxf(c.x, fmaxf(c.y, c.z));
    if (n < 0.0f) c = V3(l + (((c.x - l) * l) / (l - n)), l + (((c.y - l) * l) / (l - n)), l + (((c.z - l) * l) / (l - n)));
    if (x > 1.0f)
        c = V3(l + (((c.x - l) * (1.0f - l)) / (x - l)), l + (((c.y - l) * (1.0f - l)) / (x - l)),
               l + (((c.z - l) * (1.0f - l)) / (x - l)));
    return c;
}
__device__ v3 set_lum(v3 c, float l) {
    float d = l - lum(c);
    return clip_color(V3(c.x + d, c.y + d, c.z + d));
}
__device__ void set_sat_inner(float &cmin, float &cmid, float &cmax, float s) {
    if (cmax > cmin) {
        cmid = ((cmid - cmin) * s) / (cmax - cmin);
        cmax = s;
    } else {
        cmid = 0.0f;
        cmax = 0.0f;
    }
    cmin = 0.0f;
}
__device__ v3 set_sat(v3 c, float s) {
    float r = c.x, g = c.y, b = c.z;
    if (r <= g) {
        if (g <= b) set_sat_inner(r, g, b, s);
        else if (r <= b) set_sat_inner(r, b, g, s);
        else set_sat_inner(b, r, g, s);
    } else {
        if (r <= b) set_sat_inner(g, r, b, s);
        else if (g <= b) set_sat_inner(g, b, r, s);
        else set_sat_inner(b, g, r, s);
    }
    return V3(r, g, b);
}
__device__ v3 blend_mix(v3 cb, v3 cs, uint32_t mode) {
    switch (mode) {
    case 1: return V3(cb.x * cs.x, cb.y * cs.y, cb.z * cs.z);
    case 2: return V3(screen1(cb.x, cs.x), screen1(cb.y, cs.y), screen1(cb.z, cs.z));
    case 3: return V3(hard_light1(cs.x, cb.x), hard_light1(cs.y, cb.y), hard_light1(cs.z, cb.z));
    case 4: return V3(fminf(cb.x, cs.x), fminf(cb.y, cs.y), fminf(cb.z, cs.z));
    case 5: return V3(fmaxf(cb.x, cs.x), fmaxf(cb.y, cs.y), fmaxf(cb.z, cs.z));
    case 6: return V3(color_dodge(cb.x, cs.x), color_dodge(cb.y, cs.y), color_dodge(cb.z, cs.z));
    case 7: return V3(color_burn(cb.x, cs.x), color_burn(cb.y, cs.y), color_burn(cb.z, cs.z));
    case 8: return V3(hard_light1(cb.x, cs.x), hard_light1(cb.y, cs.y), hard_light1(cb.z, cs.z));
    case 9: return V3(soft_light1(cb.x, cs.x), soft_light1(cb.y, cs.y), soft_light1(cb.z, cs.z));
    case 10: return V3(fabsf(cb.x - cs.x), fabsf(cb.y - cs.y), fabsf(cb.z - cs.z));
    case 11: return V3(cb.x + cs.x - 2.0f * cb.x * cs.x, cb.y + cs.y - 2.0f * cb.y * cs.y, cb.z + cs.z - 2.0f * cb.z * cs.z);
    case 12: return set_lum(set_sat(cs, sat3(cb)), lum(cb));
    case 13: return set_lum(set_sat(cb, sat3(cs)), lum(cb));
    case 14: return set_lum(cs, lum(cb));
    case 15: return set_lum(cb, lum(cs));
    default: return cs;
    }
}
__device__ rgba_t blend_compose(v3 cb, v3 cs, float ab, float as_, uint32_t mode) {
    float fa = 0.0f, fb = 0.0f;
    switch (mode) {
    case 1: fa = 1.0f; fb = 0.0f; break;
    case 2: fa = 0.0f; fb = 1.0f; break;
    case 3: fa = 1.0f; fb = 1.0f - as_; break;
    case 4: fa = 1.0f - ab; fb = 1.0f; break;
    case 5: fa = ab; fb = 0.0f; break;
    case 6: fa = 0.0f; fb = as_; break;
    case 7: fa = 1.0f - ab; fb = 0.0f; break;
    case 8: fa = 0.0f; fb = 1.0f - as_; break;
    case 9: fa = ab; fb = 1.0f - as_; break;
    case 10: fa = 1.0f - ab; fb = as_; break;
    case 11: fa = 1.0f - ab; fb = 1.0f - as_; break;
    case 12: fa = 1.0f; fb = 1.0f; break;
    case 13:
        return RG(fminf(1.0f, as_ * cs.x + ab * cb.x), fminf(1.0f, as_ * cs.y + ab * cb.y), fminf(1.0f, as_ * cs.z + ab * cb.z),
                  fminf(1.0f, as_ + ab));
    default: break;
    }
    float as_fa = as_ * fa, ab_fb = ab * fb;
    return RG(as_fa * cs.x + ab_fb * cb.x, as_fa * cs.y + ab_fb * cb.y, as_fa * cs.z + ab_fb * cb.z, fminf(as_fa + ab_fb, 1.0f));
}
__device__ __forceinline__ v3 unpremultiply(rgba_t c) {
    float inv = 1.0f / fmaxf(c.a, 1e-15f);
    return V3(c.r * inv, c.g * inv, c.b * inv);
}
__device__ __forceinline__ float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; }
__device__ rgba_t blend_mix_compose(rgba_t backdrop, rgba_t src, uint32_t mode) {
    if ((mode & 0x7fffu) == 3u) return over(backdrop, src);
    v3 cs = unpremultiply(src);
    v3 cb = unpremultiply(backdrop);
    v3 mixed = blend_mix(cb, cs, mode >> 8);
    cs = V3(mixf(cs.x, mixed.x, backdrop.a), mixf(cs.y, mixed.y, backdrop.a), mixf(cs.z, mixed.z, backdrop.a));
    uint32_t compose_mode = mode & 0xffu;
    if (compose_mode == 3u) {
        return RG(mixf(backdrop.r, cs.x, src.a), mixf(backdrop.g, cs.y, src.a), mixf(backdrop.b, cs.z, src.a),
                  src.a + backdrop.a * (1.0f - src.a));
    }
    return blend_compose(cb, cs, backdrop.a, src.a, compose_mode);
}

// ---------------- gradients / images ----------------
__device__ __forceinline__ float extend_mode_normalized(float t, uint32_t mode) {
    if (mode == 0u) return vb_clampf(t, 0.0f, 1.0f);
    if (mode == 1u) return t - floorf(t);
    return fabsf(t - 2.0f * rintf(0.5f * t));
}
__device__ __forceinline__ float extend_mode(float t, uint32_t mode, float mx) {
    if (mode == 0u) return vb_clampf(t, 0.0f, mx);
    return extend_mode_normalized(t / mx, mode) * mx;
}
__device__ __forceinline__ rgba_t ramp_load(const FineArgs &A, const VbConfig &cfg, int32_t x, uint32_t index) {
    if (index >= cfg.n_ramps || x < 0 || x >= GRADIENT_WIDTH) return RG(0, 0, 0, 0);
    return unpack4x8unorm(__ldg(A.ramps + (size_t)index * GRADIENT_WIDTH + (uint32_t)x));
}
__device__ __forceinline__ rgba_t atlas_load(const FineArgs &A, const VbConfig &cfg, float fx, float fy) {
    int32_t x = vb_f2i_sat(fx), y = vb_f2i_sat(fy);
    if (x < 0 || y < 0 || (uint32_t)x >= cfg.atlas_w || (uint32_t)y >= cfg.atlas_h) return RG(0, 0, 0, 0);
    uint32_t p = __ldg(reinterpret_cast<const uint32_t *>(A.atlas) + (size_t)y * cfg.atlas_w + (uint32_t)x);
    return unpack4x8unorm(p);
}
__device__ __forceinline__ rgba_t maybe_premul(rgba_t p, uint32_t alpha_type) {
    if (alpha_type == 1u) return p;
    return RG(p.r * p.a, p.g * p.a, p.b * p.a, p.a);
}
__device__ __forceinline__ rgba_t pixel_format(rgba_t p, uint32_t format) { return format == 1u ? RG(p.b, p.g, p.r, p.a) : p; }
__device__ float erf7(float x) {
    float y = vb_clampf(x * 1.1283791671f, -100.0f, 100.0f);
    float yy = y * y;
    float z = y + (0.24295f + (0.03395f + 0.0104f * yy) * yy) * (y * yy);
    return z / sqrtf(1.0f + z * z);
}
__device__ __forceinline__ float hypot_w(float a, float b) { return sqrtf(a * a + b * b); }
__device__ __forceinline__ float single_weight(float t, float a, float b, float c, float d) { return t * (t * (t * d + c) + b) + a; }
__device__ void cubic_weights(float fr, float (&w)[4]) {
    w[0] = single_weight(fr, (1.0f / 6.0f) / 3.0f, -(3.0f / 6.0f) / 3.0f - 1.0f / 3.0f, (3.0f / 6.0f) / 3.0f + 2.0f * 1.0f / 3.0f,
                         -(1.0f / 6.0f) / 3.0f - 1.0f / 3.0f);
    w[1] = single_weight(fr, 1.0f - (2.0f / 6.0f) / 3.0f, 0.0f, -3.0f + (12.0f / 6.0f) / 3.0f + 1.0f / 3.0f,
                         2.0f - (9.0f / 6.0f) / 3.0f - 1.0f / 3.0f);
    w[2] = single_weight(fr, (1.0f / 6.0f) / 3.0f, (3.0f / 6.0f) / 3.0f + 1.0f / 3.0f, 3.0f - (15.0f / 6.0f) / 3.0f - 2.0f * 1.0f / 3.0f,
                         -2.0f + (9.0f / 6.0f) / 3.0f + 1.0f / 3.0f);
    w[3] = single_weight(fr, 0.0f, 0.0f, -1.0f / 3.0f, (1.0f / 6.0f) / 3.0f + 1.0f / 3.0f);
}
__device__ rgba_t bicubic_sample(const FineArgs &A, const VbConfig &cfg, float cx, float cy, float ox, float oy, float mx, float my,
                                 uint32_t alpha_type) {
    float fxx = (cx + 0.5f) - floorf(cx + 0.5f), fyy = (cy + 0.5f) - floorf(cy + 0.5f);
    float wx[4], wy[4];
    cubic_weights(fxx, wx);
    cubic_weights(fyy, wy);
    const float offs[4] = {-1.5f, -0.5f, 0.5f, 1.5f};
    rgba_t r = RG(0, 0, 0, 0);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        rgba_t acc = RG(0, 0, 0, 0);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            rgba_t s = maybe_premul(atlas_load(A, cfg, vb_clampf(cx + offs[i], ox, mx), vb_clampf(cy + offs[j], oy, my)), alpha_type);
            if (i == 0) acc = rg_scale(s, wx[0]);
            else acc = RG(acc.r + wx[i] * s.r, acc.g + wx[i] * s.g, acc.b + wx[i] * s.b, acc.a + wx[i] * s.a);
        }
        if (j == 0) r = rg_scale(acc, wy[0]);
        else r = RG(r.r + wy[j] * acc.r, r.g + wy[j] * acc.g, r.b + wy[j] * acc.b, r.a + wy[j] * acc.a);
    }
    float a = vb_clampf(r.a, 0.0f, 1.0f);
    return RG(vb_clampf(r.r, 0.0f, a), vb_clampf(r.g, 0.0f, a), vb_clampf(r.b, 0.0f, a), a);
}

// Occlusion start. A tile's command list is painted back to front; `CMD_SOLID, CMD_COLOR` with alpha 255 outside any
// clip replaces every pixel of the tile (over(bg, fg) = fg + bg * (1 - 1) = fg exactly), so nothing before the LAST such
// pair can reach the output. coarse notes the offset of that CMD_SOLID per tile while it writes the list
// (k_coarse.cu, tile_start) and fine starts there: identical pixels, and on map-like scenes with opaque area fills most
// of a tile's commands are never executed. The reference executes the whole list (fine.wgsl:1064); the PTCL is unchanged.

// ---------------- the interpreter: fine.wgsl:1064-1398 ----------------
// Dynamic shared memory of a CTA of W warps:  [mask LUT (AA != 0)] [LUT mbarrier, 16 B] [W x WarpIo] [W x WarpMs (AA != 0)]
template <int AA>
struct FineSmem {
    static constexpr uint32_t LUT_WORDS = AA == 2 ? 2048u : (AA == 1 ? 256u : 0u);
    static constexpr uint32_t MS_BYTES = AA == 0 ? 0u : (uint32_t)sizeof(WarpMs<AA == 0 ? 1 : AA>);
    static constexpr uint32_t PER_WARP = (uint32_t)sizeof(WarpIo) + MS_BYTES;
    __host__ __device__ static constexpr uint32_t bytes(uint32_t warps) { return LUT_WORDS * 4u + 16u + warps * PER_WARP; }
};
static_assert(sizeof(WarpIo) % 16 == 0 && sizeof(WarpMs<1>) % 16 == 0 && sizeof(WarpMs<2>) % 16 == 0, "16-byte aligned smem blocks");

// MODE: the AA mode (0 area, 1 MSAA8, 2 MSAA16), plus FI_DMG for damage tracking (k_damage.cu): coarse listed only the
// damaged tiles, and those lists are the whole queue, so no other pixel is written. FI_DST: a registered destination
// (vb_register_destination) in BGRA8 order, with premultiplied alpha, in a float format or in a CUDA array; only the store
// differs. FI_BG (always with FI_DST, never with FI_DMG): every tile starts from a background's pixels (vb_set_background)
// instead of the base colour. These three instantiations are compiled into k_fine_bg.o (VB_FINE_BG), so that k_fine.o holds
// exactly the others.
#define FI_DMG 16
#define FI_DST 32
#define FI_BG 64
template <int MODE>
using FineArgsOf = typename std::conditional<(MODE & FI_BG) != 0, FineBgArgs,
                                             typename std::conditional<(MODE & FI_DST) != 0, FineDstArgs, FineArgs>::type>::type;

// Which of coarse's tile lists a launch walks (FineArgs::lists). coarse puts each tile of the window into one of
// VB_FINE_CLASSES cost classes, and each class into two lists: list 2k holds the tiles whose commands from their occlusion
// start are only FILL / SOLID / COLOR / JUMP, list 2k + 1 the others (flagged). A frame is painted either by one k_fine over
// every list, or by k_fine_solid over the simple lists followed by k_fine over the flagged ones.
#define FI_LISTS_ALL 0u
#define FI_LISTS_SIMPLE 1u
#define FI_LISTS_FLAGGED 2u

// ---- the tile queue: queue position -> {tile of the window, occlusion start}. Walking the launch's lists in class order
// makes the heavy tiles the FIRST ones every warp takes (longest-processing-time-first), which is what bounds a persistent
// kernel's tail when a stripe has only a few tiles per warp. Lane l < VB_FINE_LISTS holds the first queue position of list l
// when the launch walks it (~0 otherwise), so the list of a position is the last lane whose start is at or below it.
struct FineQueue {
    uint32_t n_tiles; // queue positions of the launch (warp-uniform)
    uint32_t cpre;    // this lane's list's first queue position
    bool ordered;     // false: the window's tiles in their natural order, with their occlusion starts from tile_start
};
template <bool DMG>
__device__ __forceinline__ FineQueue fine_queue(const VbConfig &cfg, const FineArgs &A, uint32_t lane) {
    FineQueue q;
    q.n_tiles = cfg.width_in_tiles * (cfg.win_ty1 - cfg.win_ty0);
    q.cpre = ~0u;
    q.ordered = A.cls_count != nullptr;
    if (q.ordered) {
        const uint32_t c = lane < VB_FINE_LISTS ? min(__ldg(A.cls_count + lane), A.cls_stride) : 0u;
        const bool walked = lane < VB_FINE_LISTS && (A.lists == FI_LISTS_ALL || (lane & 1u) == (A.lists == FI_LISTS_FLAGGED ? 1u : 0u));
        const uint32_t incl = vb_warp_incl_scan(walked ? c : 0u);
        if (walked) q.cpre = incl - c;
        q.ordered = DMG || vb_warp_sum(c) == q.n_tiles; // a launch over part of the window (read-back bands) keeps the natural order
        if (q.ordered) q.n_tiles = __shfl_sync(VB_FULL, incl, 31);
    }
    if (!q.ordered && A.lists == FI_LISTS_SIMPLE) q.n_tiles = 0u; // the k_fine after it paints every tile then
    return q;
}
__device__ __forceinline__ uint2 fine_entry(const VbConfig &cfg, const FineArgs &A, const FineQueue &q, uint32_t pos) {
    if (q.ordered) {
        const uint32_t l = 31u - (uint32_t)__clz((int)__ballot_sync(VB_FULL, pos >= q.cpre));
        return __ldg(A.cls_list + (size_t)l * A.cls_stride + (pos - __shfl_sync(VB_FULL, q.cpre, l)));
    }
    return make_uint2(pos, A.cull != 0u ? __ldg(A.tile_start + cfg.win_ty0 * cfg.width_in_tiles + pos) : 0u);
}

// ---- the command windows
__device__ __forceinline__ void fine_wait(WarpIo &io, uint32_t buf, uint32_t &phase) {
    mbar_wait(&io.mbar[buf], (phase >> buf) & 1u);
    phase ^= 1u << buf;
}
// The command word at cmd_ix and its (up to 3) operands, from the staged window; when the pointer leaves the window (a list
// longer than the window, CMD_JUMP into another chunk) the window is staged again there.
__device__ __forceinline__ const uint32_t *fine_cmd_words(WarpIo &io, const uint32_t *ptcl, uint32_t cmd_ix, uint32_t &win_base, uint32_t buf,
                                                          uint32_t &phase, uint32_t lane) {
    uint32_t off = cmd_ix - win_base;
    if (off > WIN_WORDS - 4u) {
        win_base = cmd_ix & ~3u;
        __syncwarp();
        if (lane == 0u) {
            mbar_expect_tx(&io.mbar[buf], WIN_WORDS * 4u);
            bulk_g2s(io.ptcl[buf], ptcl + win_base, WIN_WORDS * 4u, &io.mbar[buf]);
        }
        fine_wait(io, buf, phase);
        off = cmd_ix - win_base;
    }
    return io.ptcl[buf] + off;
}

// ---- the persistent tile loop of both kernels. For every tile of the launch's queue it calls
// paint(io, S, lut, tile_ix, cell, gx, gy, start, buf, phase): the warp's command windows and MSAA state, the mask LUT, the
// tile's index in the frame's tile grid, the cell of a batch, the lane's pixels (cell row gy, columns gx..gx+7), the PTCL
// offset the tile starts at, and the window its commands are staged in (wait for it with fine_wait).
template <int AA, bool DMG, class Paint>
__device__ __forceinline__ void fine_tiles(const VbConfig &cfg, const FineArgs &A, Paint &&paint) {
    extern __shared__ __align__(16) unsigned char smem[];
    typedef WarpMs<AA == 0 ? 1 : AA> Ms;
    if (A.bump->failed != 0u) return; // upstream failure (the reference flags it through ptcl[0], path_tiling_setup.wgsl:25; see vb_frame.cu)
    const uint32_t lane = vb_lane(), warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    const FineQueue q = fine_queue<DMG>(cfg, A, lane);
    // a CTA none of whose warps has a tile leaves before its set-up (k_fine after k_fine_solid when few or no tiles are flagged)
    if (blockIdx.x * n_warps >= q.n_tiles) return;
    uint32_t *lut = reinterpret_cast<uint32_t *>(smem);
    uint64_t *lut_bar = reinterpret_cast<uint64_t *>(smem + FineSmem<AA>::LUT_WORDS * 4u);
    WarpIo &io = *reinterpret_cast<WarpIo *>(smem + FineSmem<AA>::LUT_WORDS * 4u + 16u + warp * (uint32_t)sizeof(WarpIo));
    Ms &S = *reinterpret_cast<Ms *>(smem + FineSmem<AA>::LUT_WORDS * 4u + 16u + n_warps * (uint32_t)sizeof(WarpIo) + warp * FineSmem<AA>::MS_BYTES);

    // ---- one-time set-up: barriers, the mask LUT (one bulk copy per CTA), the clean MSAA state of this warp
    if (lane == 0u) {
        mbar_init(&io.mbar[0], 1u);
        mbar_init(&io.mbar[1], 1u);
        if (AA != 0 && warp == 0u) mbar_init(lut_bar, 1u);
        mbar_fence_init();
    }
    if (AA != 0) ms_init(S, lane);
    __syncthreads();
    if (AA != 0) {
        if (threadIdx.x == 0u) {
            mbar_expect_tx(lut_bar, FineSmem<AA>::LUT_WORDS * 4u);
            bulk_g2s(lut, A.mask_lut, FineSmem<AA>::LUT_WORDS * 4u, lut_bar);
        }
    }

    // ---- tile queue. Warp g of G takes queue positions g and g + G, then whatever the queue hands out (2G + atomicAdd). The
    // pipeline is three tiles deep: while tile k is painted, the command window of tile k+1 is in flight (bulk copy), the
    // occlusion start of tile k+2 is being loaded and the queue ticket of tile k+3 is being taken, so none of those latencies
    // is exposed.
    const uint32_t wt = cfg.width_in_tiles;
    const uint32_t n_tiles = q.n_tiles;
    const uint32_t G = gridDim.x * n_warps, g = blockIdx.x * n_warps + warp;
    const uint32_t first_tile = cfg.win_ty0 * wt;
#define START_OF(t, s0) ((s0) != 0u && A.cull != 0u ? (s0) : (first_tile + (t)) * VB_PTCL_INITIAL_ALLOC + 1u)
    uint32_t p_cur = g, p_nxt = g + G; // queue positions
    uint32_t buf = 0u, phase = 0u; // phase: bit b = parity to wait for on mbar[b]
    uint32_t t_cur = 0u, start_cur = 0u, ticket = 0u;
    uint2 e_nxt = make_uint2(0u, 0u);
    if (p_cur < n_tiles) {
        const uint2 e = fine_entry(cfg, A, q, p_cur);
        t_cur = e.x;
        start_cur = START_OF(e.x, e.y);
        if (lane == 0u) {
            mbar_expect_tx(&io.mbar[0], WIN_WORDS * 4u);
            bulk_g2s(io.ptcl[0], A.ptcl + (start_cur & ~3u), WIN_WORDS * 4u, &io.mbar[0]);
            ticket = atomicAdd(A.queue, 1u);
        }
        if (p_nxt < n_tiles) e_nxt = fine_entry(cfg, A, q, p_nxt);
    }
    if (AA != 0) mbar_wait(lut_bar, 0u); // every thread of the CTA observes the LUT copy before its first use

    const uint32_t ly = lane >> 1, h = lane & 1u;
    while (p_cur < n_tiles) {
        // ---- pipeline bookkeeping for the tiles after this one
        const uint32_t t_nxt = e_nxt.x;
        const uint32_t start_nxt = START_OF(e_nxt.x, e_nxt.y);
        if (p_nxt < n_tiles && lane == 0u) {
            mbar_expect_tx(&io.mbar[buf ^ 1u], WIN_WORDS * 4u);
            bulk_g2s(io.ptcl[buf ^ 1u], A.ptcl + (start_nxt & ~3u), WIN_WORDS * 4u, &io.mbar[buf ^ 1u]);
        }
        const uint32_t p_nn = 2u * G + __shfl_sync(VB_FULL, ticket, 0);
        uint2 e_nn = make_uint2(0u, 0u);
        if (p_nn < n_tiles) {
            e_nn = fine_entry(cfg, A, q, p_nn);
            if (lane == 0u) ticket = atomicAdd(A.queue, 1u);
        }

        // ---- this tile
        const uint32_t tile_x = t_cur % wt, tile_y = cfg.win_ty0 + t_cur / wt;
        const uint32_t tile_ix = tile_y * wt + tile_x;
        // batch: the tile row of the tall frame names the cell; pixels (brushes, output row) are the cell's own
        uint32_t cell = 0u;
        if (cfg.n_cells > 1u) cell = tile_y / cfg.height_in_tiles;
        const uint32_t gx = tile_x * 16u + h * 8u, gy = (tile_y - cell * cfg.height_in_tiles) * 16u + ly;
        paint(io, S, lut, tile_ix, cell, gx, gy, start_cur, buf, phase);
        __syncwarp();
        p_cur = p_nxt; t_cur = t_nxt; start_cur = start_nxt;
        p_nxt = p_nn; e_nxt = e_nn;
        buf ^= 1u;
    }
#undef START_OF
}

// ---- store: rgba8unorm with separated alpha (fine.wgsl:1386-1397). When every pixel of the warp is opaque (the common case)
// a_inv is exactly 1 and the three multiplications are identities, so they are skipped. FI_DST also stores premultiplied alpha
// (unorm8 of each channel) and float texels (store_float).
template <bool DST, class Args>
__device__ __forceinline__ void fine_store(const VbConfig &cfg, const Args &A, rgba_t (&rgba)[PX], uint32_t tile_ix, uint32_t gx, uint32_t gy) {
    bool opaque = true;
#pragma unroll
    for (int i = 0; i < PX; i++) opaque = opaque && rgba[i].a == 1.0f;
    const bool all_opaque = __all_sync(VB_FULL, opaque);
    bool float_texels = false, premul = false; // FI_DST: a float destination, premultiplied alpha
    if constexpr (DST) {
        float_texels = A.texel != 4u;
        premul = A.premul != 0u;
    }
    if (float_texels && gy < cfg.target_height && gy >= cfg.out_row0) {
        if constexpr (DST) store_float(A, cfg, rgba, gx, gy, all_opaque);
    } else if (gy < cfg.target_height && gy >= cfg.out_row0) {
        uint32_t px[PX];
        if (all_opaque) {
#pragma unroll
            for (int i = 0; i < PX; i++) px[i] = unorm8(rgba[i].r) | (unorm8(rgba[i].g) << 8) | (unorm8(rgba[i].b) << 16) | 0xff000000u;
        } else if (premul) {
#pragma unroll
            for (int i = 0; i < PX; i++) px[i] = pack4x8unorm(rgba[i]);
        } else {
#pragma unroll
            for (int i = 0; i < PX; i++) {
                const rgba_t fg = rgba[i];
                const float a_inv = 1.0f / fmaxf(fg.a, 1e-6f);
                px[i] = unorm8(fg.r * a_inv) | (unorm8(fg.g * a_inv) << 8) | (unorm8(fg.b * a_inv) << 16) | (unorm8(fg.a) << 24);
            }
        }
        bool stored = false;
        if constexpr (DST) {
#pragma unroll
            for (int i = 0; i < PX; i++) px[i] = __byte_perm(px[i], 0u, A.swz);
            if (A.array) {
                // gy is the frame's own row, also in a window. Texels out of the array's range are dropped
                // (cudaBoundaryModeZero), though the host refuses a frame that does not fit before it is enqueued.
                const uint32_t x = A.x0 + gx, y = A.y0 + gy;
                if (gx + 7u < cfg.target_width && (x & 3u) == 0u) {
                    // two 128-bit stores: 32 contiguous bytes of one texel row per lane
                    surf2Dwrite(make_uint4(px[0], px[1], px[2], px[3]), A.surf, (int)(x * 4u), (int)y, cudaBoundaryModeZero);
                    surf2Dwrite(make_uint4(px[4], px[5], px[6], px[7]), A.surf, (int)(x * 4u + 16u), (int)y, cudaBoundaryModeZero);
                } else {
#pragma unroll
                    for (int i = 0; i < PX; i++)
                        if (gx + i < cfg.target_width) surf2Dwrite(px[i], A.surf, (int)((x + i) * 4u), (int)y, cudaBoundaryModeZero);
                }
                stored = true;
            }
        }
        if (!stored) {
            // the cell again, from the tile index (keeping it live across the interpreter would cost a register)
            const uint32_t out_cell = cfg.n_cells > 1u ? tile_ix / cfg.width_in_tiles / cfg.height_in_tiles : 0u;
            uint32_t *row = A.out + ((size_t)out_cell * cfg.target_height + (gy - cfg.out_row0)) * cfg.out_pitch_px;
            if (gx + 7u < cfg.target_width && (cfg.out_pitch_px & 3u) == 0u && ((uintptr_t)A.out & 15u) == 0u) {
                // two 128-bit stores: 32 contiguous bytes of one pixel row per lane
                uint4 *dst = reinterpret_cast<uint4 *>(row + gx);
                dst[0] = make_uint4(px[0], px[1], px[2], px[3]);
                dst[1] = make_uint4(px[4], px[5], px[6], px[7]);
            } else {
#pragma unroll
                for (int i = 0; i < PX; i++)
                    if (gx + i < cfg.target_width) row[gx + i] = px[i];
            }
        }
    }
}

// ---- k_fine: the whole interpreter. It paints every tile of a frame, or only the flagged ones after k_fine_solid.
template <int MODE>
__global__ void __launch_bounds__(FI_MAX_THREADS, FI_MINB)
k_fine(VbConfig cfg, FineArgsOf<MODE> A) {
    constexpr int AA = MODE & 15;
    constexpr bool DMG = (MODE & FI_DMG) != 0;
    constexpr bool DST = (MODE & FI_DST) != 0;
    constexpr bool BG = (MODE & FI_BG) != 0;
    static_assert(!BG || (DST && !DMG), "FI_BG goes with FI_DST and without FI_DMG");
    typedef WarpMs<AA == 0 ? 1 : AA> Ms;
    const uint32_t *__restrict__ ptcl = A.ptcl;
    const uint32_t *__restrict__ info = A.info;
    const uint32_t lane = vb_lane();
    const uint32_t ly = lane >> 1, h = lane & 1u;
    fine_tiles<AA, DMG>(cfg, A, [&](WarpIo &io, Ms &S, const uint32_t *lut, uint32_t tile_ix, uint32_t cell, uint32_t gx, uint32_t gy,
                                    uint32_t start_cur, uint32_t buf, uint32_t &phase) {
        // pixel coordinates are small integers: (float)(gx + i) is exactly the WGSL's xy.x + f32(i) of either 4-pixel group
#define xyy ((float)gy)
#define xyx0 ((float)gx)
#define xyx1 ((float)(gx + 4u))
        rgba_t rgba[PX];
        float area[PX];
        {
            const rgba_t base = unpack4x8unorm_uniform(cfg.base_color);
#pragma unroll
            for (int i = 0; i < PX; i++) { rgba[i] = base; area[i] = 0.0f; }
        }
        // FI_BG: the tile starts from the background's pixels, loaded before the wait for the command window. A tile that
        // starts at its occlusion start skips them: its first commands paint every pixel opaque, and over(bg, fg) =
        // fmaf(bg, 0, fg) = fg for any finite bg.
        if constexpr (BG) {
            if (gy < cfg.target_height && start_cur == tile_ix * VB_PTCL_INITIAL_ALLOC + 1u) load_bg(A.bg, cfg, cell, gx, gy, rgba);
        }
        // first BLEND_STACK_SPLIT levels of the blend stack: thread-private (local memory, L1 resident); deeper
        // levels spill to blend_spill exactly as in the reference
        // Dynamically indexed -> lives in local memory; every level is stored by BEGIN_CLIP before END_CLIP loads it.
        // (Do not turn this into a register array updated through `d == clip_depth ? new : old` selects without
        // initialising it: the optimiser folds selects on undefined values and clobbers live levels.)
        uint32_t blend_stack[VB_BLEND_STACK_SPLIT][PX];
        rgba_t t_rgba[PX]; // see PIX_TO_LOCAL
        float t_area[PX];
        uint32_t clip_depth = 0u;
        uint32_t cmd_ix = start_cur;
        uint32_t win_base = start_cur & ~3u;
        fine_wait(io, buf, phase);
#define PXX(i) ((((i) < 4) ? xyx0 : xyx1) + (float)((i) & 3))
        // The rarely used brushes loop over the lane's pixels WITHOUT unrolling (code size); they work on a copy in local
        // memory so that rgba[] / area[] themselves are only ever indexed by constants and live in registers.
#define PIX_TO_LOCAL() _Pragma("unroll") for (int q_ = 0; q_ < PX; q_++) { t_rgba[q_] = rgba[q_]; t_area[q_] = area[q_]; }
#define PIX_FROM_LOCAL() _Pragma("unroll") for (int q_ = 0; q_ < PX; q_++) rgba[q_] = t_rgba[q_]
        for (;;) {
            const uint32_t *cw = fine_cmd_words(io, ptcl, cmd_ix, win_base, buf, phase, lane);
            const uint32_t tag = cw[0];
            const uint32_t w1 = cw[1], w2 = cw[2], w3 = cw[3];
            if (tag == VB_CMD_END) break;
            switch (tag) {
            case VB_CMD_FILL: {
                fine_cmd_fill<AA>(A, S, lut, w1, w2, (int32_t)w3, lane, area);
                cmd_ix += 4u;
                break;
            }
            case VB_CMD_SOLID:
                fine_cmd_solid(area);
                cmd_ix += 1u;
                break;
            case VB_CMD_COLOR: {
                fine_cmd_color(w1, rgba, area);
                cmd_ix += 2u;
                break;
            }
            case VB_CMD_BEGIN_CLIP: {
                if (clip_depth < VB_BLEND_STACK_SPLIT) {
#pragma unroll
                    for (int i = 0; i < PX; i++) {
                        blend_stack[clip_depth][i] = pack4x8unorm(rgba[i]);
                        rgba[i] = RG(0, 0, 0, 0);
                    }
                } else {
                    const uint32_t blend_offset = __ldg(ptcl + tile_ix * VB_PTCL_INITIAL_ALLOC);
                    const uint32_t base_ix = blend_offset + (clip_depth - VB_BLEND_STACK_SPLIT) * 256u + h * 8u + ly * 16u;
#pragma unroll
                    for (int i = 0; i < PX; i++) {
                        if (base_ix + i < cfg.blend_size) A.blend_spill[base_ix + i] = pack4x8unorm(rgba[i]);
                        rgba[i] = RG(0, 0, 0, 0);
                    }
                }
                clip_depth += 1u;
                cmd_ix += 1u;
                break;
            }
            case VB_CMD_END_CLIP: {
                const uint32_t blend = w1;
                const float alpha = __uint_as_float(w2);
                clip_depth -= 1u;
                uint32_t blend_offset = 0u;
                if (clip_depth >= VB_BLEND_STACK_SPLIT) blend_offset = __ldg(ptcl + tile_ix * VB_PTCL_INITIAL_ALLOC);
#pragma unroll
                for (int i = 0; i < PX; i++) {
                    uint32_t bg_rgba;
                    if (clip_depth < VB_BLEND_STACK_SPLIT) {
                        bg_rgba = blend_stack[clip_depth][i];
                    } else {
                        const uint32_t ix = blend_offset + (clip_depth - VB_BLEND_STACK_SPLIT) * 256u + h * 8u + ly * 16u + i;
                        bg_rgba = ix < cfg.blend_size ? A.blend_spill[ix] : 0u;
                    }
                    const rgba_t bg = unpack4x8unorm(bg_rgba);
                    const rgba_t fg = rg_scale(rg_scale(rgba[i], area[i]), alpha);
                    if (blend == 0x10000u) {
                        if (area[i] == 0.0f) { rgba[i] = bg; continue; }
                        const float luminance = vb_clampf(svg_lum(unpremultiply(fg)) * fg.a, 0.0f, 1.0f);
                        rgba[i] = rg_scale(bg, luminance);
                    } else {
                        rgba[i] = blend_mix_compose(bg, fg, blend);
                    }
                }
                cmd_ix += 3u;
                break;
            }
            case VB_CMD_JUMP:
                cmd_ix = w1;
                break;
            case VB_CMD_BLUR_RECT: {
                const uint32_t io = w1;
                const rgba_t blur_rgba = unpack4x8unorm_uniform(w2);
                const float m0 = __uint_as_float(info[io]), m1 = __uint_as_float(info[io + 1]), m2 = __uint_as_float(info[io + 2]),
                            m3 = __uint_as_float(info[io + 3]);
                const float tx = __uint_as_float(info[io + 4]), ty = __uint_as_float(info[io + 5]);
                const float bw = __uint_as_float(info[io + 6]), bh = __uint_as_float(info[io + 7]), bradius = __uint_as_float(info[io + 8]);
                const float std_dev = fmaxf(__uint_as_float(info[io + 9]), 1e-5f);
                const float inv_std_dev = 1.0f / std_dev;
                const float min_edge = fminf(bw, bh);
                const float radius_max = 0.5f * min_edge;
                const float r0 = fminf(hypot_w(bradius, std_dev * 1.15f), radius_max);
                const float r1 = fminf(hypot_w(bradius, std_dev * 2.0f), radius_max);
                const float exponent = 2.0f * r1 / r0;
                const float inv_exponent = 1.0f / exponent;
                const float ew = 0.5f * inv_std_dev * bw, eh = 0.5f * inv_std_dev * bh;
                const float delta = 1.25f * std_dev * (vb_expf(-(ew * ew)) - vb_expf(-(eh * eh)));
                const float width = bw + fminf(delta, 0.0f);
                const float height = bh - fmaxf(delta, 0.0f);
                const float scale = 0.5f * erf7(inv_std_dev * 0.5f * (fmaxf(width, height) - 0.5f * bradius));
                PIX_TO_LOCAL();
#pragma unroll 1
                for (int i = 0; i < PX; i++) {
                    const float px = PXX(i), py = xyy;
                    const float x = (m0 * px + m2 * py) + tx;
                    const float y = (m1 * px + m3 * py) + ty;
                    const float y0 = fabsf(y) - (height * 0.5f - r1);
                    const float y1 = fmaxf(y0, 0.0f);
                    const float x0 = fabsf(x) - (width * 0.5f - r1);
                    const float x1 = fmaxf(x0, 0.0f);
                    const float d_pos = vb_powf_pos(vb_powf_pos(x1, exponent) + vb_powf_pos(y1, exponent), inv_exponent);
                    const float d_neg = fminf(fmaxf(x0, y0), 0.0f);
                    const float d = d_pos + d_neg - r1;
                    const float alpha = scale * (erf7(inv_std_dev * (min_edge + d)) - erf7(inv_std_dev * d));
                    t_rgba[i] = over(t_rgba[i], rg_scale(rg_scale(blur_rgba, alpha), t_area[i]));
                }
                PIX_FROM_LOCAL();
                cmd_ix += 3u;
                break;
            }
            case VB_CMD_LIN_GRAD: {
                const uint32_t index_mode = w1, io = w2;
                const uint32_t index = index_mode >> 2, ext = index_mode & 3u;
                const float line_x = __uint_as_float(info[io]), line_y = __uint_as_float(info[io + 1]), line_c = __uint_as_float(info[io + 2]);
                const float d0 = (line_x * xyx0 + line_y * xyy) + line_c;
                const float d1 = (line_x * xyx1 + line_y * xyy) + line_c;
    #pragma unroll
                for (int i = 0; i < PX; i++) {
                    const float my_d = (i < 4 ? d0 : d1) + line_x * (float)(i & 3);
                    const int32_t x = vb_f2i_sat(rintf(extend_mode_normalized(my_d, ext) * (float)(GRADIENT_WIDTH - 1)));
                    rgba[i] = over(rgba[i], rg_scale(ramp_load(A, cfg, x, index), area[i]));
                }
                cmd_ix += 3u;
                break;
            }
            case VB_CMD_RAD_GRAD: {
                const uint32_t index_mode = w1, io = w2;
                const uint32_t index = index_mode >> 2, ext = index_mode & 3u;
                const float m0 = __uint_as_float(info[io]), m1 = __uint_as_float(info[io + 1]), m2 = __uint_as_float(info[io + 2]),
                            m3 = __uint_as_float(info[io + 3]);
                const float tx = __uint_as_float(info[io + 4]), ty = __uint_as_float(info[io + 5]);
                const float focal_x = __uint_as_float(info[io + 6]), radius = __uint_as_float(info[io + 7]);
                const uint32_t flags_kind = info[io + 8];
                const uint32_t flags = flags_kind >> 3, kind = flags_kind & 7u;
                const bool is_strip = kind == 2u, is_circular = kind == 1u, is_focal_on_circle = kind == 3u;
                const bool is_swapped = (flags & 1u) != 0u;
                const float r1_recip = is_circular ? 0.0f : 1.0f / radius;
                const float less_scale = (is_swapped || (1.0f - focal_x) < 0.0f) ? -1.0f : 1.0f;
                const float t_sign = vb_signf(1.0f - focal_x);
                PIX_TO_LOCAL();
#pragma unroll 1
                for (int i = 0; i < PX; i++) {
                    const float px = PXX(i), py = xyy;
                    const float x = (m0 * px + m2 * py) + tx;
                    const float y = (m1 * px + m3 * py) + ty;
                    const float xx = x * x, yy = y * y;
                    float tt = 0.0f;
                    bool is_valid = true;
                    if (is_strip) {
                        const float a = radius - yy;
                        tt = sqrtf(a) + x;
                        is_valid = a >= 0.0f;
                    } else if (is_focal_on_circle) {
                        tt = (xx + yy) / x;
                        is_valid = tt >= 0.0f && x != 0.0f;
                    } else if (radius > 1.0f) {
                        tt = sqrtf(xx + yy) - x * r1_recip;
                    } else {
                        const float a = xx - yy;
                        tt = less_scale * sqrtf(a) - x * r1_recip;
                        is_valid = a >= 0.0f && tt >= 0.0f;
                    }
                    if (is_valid) {
                        tt = extend_mode_normalized(focal_x + t_sign * tt, ext);
                        if (is_swapped) tt = 1.0f - tt;
                        const int32_t rx = vb_f2i_sat(rintf(tt * (float)(GRADIENT_WIDTH - 1)));
                        t_rgba[i] = over(t_rgba[i], rg_scale(ramp_load(A, cfg, rx, index), t_area[i]));
                    }
                }
                PIX_FROM_LOCAL();
                cmd_ix += 3u;
                break;
            }
            case VB_CMD_SWEEP_GRAD: {
                const uint32_t index_mode = w1, io = w2;
                const uint32_t index = index_mode >> 2, ext = index_mode & 3u;
                const float m0 = __uint_as_float(info[io]), m1 = __uint_as_float(info[io + 1]), m2 = __uint_as_float(info[io + 2]),
                            m3 = __uint_as_float(info[io + 3]);
                const float tx = __uint_as_float(info[io + 4]), ty = __uint_as_float(info[io + 5]);
                const float t0 = __uint_as_float(info[io + 6]), t1 = __uint_as_float(info[io + 7]);
                const float scale = 1.0f / (t1 - t0);
                PIX_TO_LOCAL();
#pragma unroll 1
                for (int i = 0; i < PX; i++) {
                    const float px = PXX(i), py = xyy;
                    const float x = (m0 * px + m2 * py) + tx;
                    const float y = (m1 * px + m3 * py) + ty;
                    const float xabs = fabsf(x), yabs = fabsf(y);
                    const float slope = fminf(xabs, yabs) / fmaxf(xabs, yabs);
                    const float s = slope * slope;
                    float phi = slope * (0.15912117063999176025390625f +
                                         s * (-5.185396969318389892578125e-2f +
                                              s * (2.476101927459239959716796875e-2f + s * (-7.0547382347285747528076171875e-3f))));
                    if (xabs < yabs) phi = 1.0f / 4.0f - phi;
                    if (x < 0.0f) phi = 1.0f / 2.0f - phi;
                    if (y < 0.0f) phi = 1.0f - phi;
                    if (phi != phi) phi = 0.0f;
                    phi = (phi - t0) * scale;
                    const float tt = extend_mode_normalized(phi, ext);
                    const int32_t rx = vb_f2i_sat(rintf(tt * (float)(GRADIENT_WIDTH - 1)));
                    t_rgba[i] = over(t_rgba[i], rg_scale(ramp_load(A, cfg, rx, index), t_area[i]));
                }
                PIX_FROM_LOCAL();
                cmd_ix += 3u;
                break;
            }
            case VB_CMD_IMAGE: {
                const uint32_t io = w1;
                const float m0 = __uint_as_float(info[io]), m1 = __uint_as_float(info[io + 1]), m2 = __uint_as_float(info[io + 2]),
                            m3 = __uint_as_float(info[io + 3]);
                const float tx = __uint_as_float(info[io + 4]), ty = __uint_as_float(info[io + 5]);
                const uint32_t xy = info[io + 6], wh = info[io + 7], sa = info[io + 8];
                const float alpha = (float)(sa & 0xFFu) / 255.0f;
                const uint32_t format = sa >> 15, alpha_type = (sa >> 14) & 1u, quality = (sa >> 12) & 3u;
                const uint32_t x_ext = (sa >> 10) & 3u, y_ext = (sa >> 8) & 3u;
                const float ox = (float)(xy >> 16), oy = (float)(xy & 0xffffu);
                const float ew = (float)(wh >> 16), eh = (float)(wh & 0xffffu);
                const float mx = ox + ew - 1.0f, my = oy + eh - 1.0f;
                PIX_TO_LOCAL();
#pragma unroll 1
                for (int i = 0; i < PX; i++) {
                    if (t_area[i] == 0.0f) continue;
                    const float px = PXX(i) + 0.5f, py = xyy + 0.5f;
                    float u = (m0 * px + m2 * py) + tx;
                    float v = (m1 * px + m3 * py) + ty;
                    u = extend_mode(u, x_ext, ew);
                    v = extend_mode(v, y_ext, eh);
                    rgba_t fg;
                    if (quality == 0u) {
                        u = u + ox; v = v + oy;
                        fg = maybe_premul(atlas_load(A, cfg, vb_clampf(u, ox, mx), vb_clampf(v, oy, my)), alpha_type);
                    } else if (quality == 2u) {
                        u = u + ox; v = v + oy;
                        fg = bicubic_sample(A, cfg, u, v, ox, oy, mx, my, alpha_type);
                    } else {
                        u = (u + ox) - 0.5f; v = (v + oy) - 0.5f;
                        const float uc = vb_clampf(u, ox, mx), vc = vb_clampf(v, oy, my);
                        const float qx0 = floorf(uc), qy0 = floorf(vc), qx1 = ceilf(uc), qy1 = ceilf(vc);
                        const float fu = u - floorf(u), fv = v - floorf(v);
                        const rgba_t a = maybe_premul(atlas_load(A, cfg, qx0, qy0), alpha_type);
                        const rgba_t b = maybe_premul(atlas_load(A, cfg, qx0, qy1), alpha_type);
                        const rgba_t c = maybe_premul(atlas_load(A, cfg, qx1, qy0), alpha_type);
                        const rgba_t d = maybe_premul(atlas_load(A, cfg, qx1, qy1), alpha_type);
                        const rgba_t ab = RG(mixf(a.r, b.r, fv), mixf(a.g, b.g, fv), mixf(a.b, b.b, fv), mixf(a.a, b.a, fv));
                        const rgba_t cd = RG(mixf(c.r, d.r, fv), mixf(c.g, d.g, fv), mixf(c.b, d.b, fv), mixf(c.a, d.a, fv));
                        fg = RG(mixf(ab.r, cd.r, fu), mixf(ab.g, cd.g, fu), mixf(ab.b, cd.b, fu), mixf(ab.a, cd.a, fu));
                    }
                    const rgba_t fg_i = pixel_format(rg_scale(rg_scale(fg, t_area[i]), alpha), format);
                    t_rgba[i] = over(t_rgba[i], fg_i);
                }
                PIX_FROM_LOCAL();
                cmd_ix += 2u;
                break;
            }
            default:
                cmd_ix += 1u;
                break;
            }
        }
#undef PXX
#undef PIX_TO_LOCAL
#undef PIX_FROM_LOCAL
#undef xyy
#undef xyx0
#undef xyx1
        fine_store<DST>(cfg, A, rgba, tile_ix, gx, gy);
    });
}

// ---- k_fine_solid: the lean interpreter of the tiles that run only FILL / SOLID / COLOR / JUMP from their occlusion start
// (coarse's simple lists), with the same tile loop, commands and store as k_fine, so a tile's pixels are the same bits
// whichever kernel paints it. Without the blend stack, the brushes' pixel copies and their code it needs no stack and fits
// FI_SOLID_WARPS x FI_SOLID_MINB resident warps per SM (DESIGN §3 "fine").
template <int AA>
__global__ void __launch_bounds__(32 * FI_SOLID_WARPS, FI_SOLID_MINB)
k_fine_solid(VbConfig cfg, FineArgs A) {
    typedef WarpMs<AA == 0 ? 1 : AA> Ms;
    const uint32_t lane = vb_lane();
    fine_tiles<AA, false>(cfg, A, [&](WarpIo &io, Ms &S, const uint32_t *lut, uint32_t tile_ix, uint32_t, uint32_t gx, uint32_t gy,
                                      uint32_t start_cur, uint32_t buf, uint32_t &phase) {
        rgba_t rgba[PX];
        float area[PX];
        {
            const rgba_t base = unpack4x8unorm_uniform(cfg.base_color);
#pragma unroll
            for (int i = 0; i < PX; i++) { rgba[i] = base; area[i] = 0.0f; }
        }
        uint32_t cmd_ix = start_cur;
        uint32_t win_base = start_cur & ~3u;
        fine_wait(io, buf, phase);
        for (;;) {
            const uint32_t *cw = fine_cmd_words(io, A.ptcl, cmd_ix, win_base, buf, phase, lane);
            const uint32_t tag = cw[0];
            if (tag == VB_CMD_END) break;
            if (tag == VB_CMD_FILL) {
                fine_cmd_fill<AA>(A, S, lut, cw[1], cw[2], (int32_t)cw[3], lane, area);
                cmd_ix += 4u;
            } else if (tag == VB_CMD_SOLID) {
                fine_cmd_solid(area);
                cmd_ix += 1u;
            } else if (tag == VB_CMD_COLOR) {
                fine_cmd_color(cw[1], rgba, area);
                cmd_ix += 2u;
            } else if (tag == VB_CMD_JUMP) {
                cmd_ix = cw[1];
            } else {
                cmd_ix += 1u; // not in a simple list (k_fine's default)
            }
        }
        fine_store<false>(cfg, A, rgba, tile_ix, gx, gy);
    });
}

typedef cudaError_t (*FineInit)();
template <int MODE> static cudaError_t fine_smem_limit() {
    return cudaFuncSetAttribute(k_fine<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FineSmem<MODE & 15>::bytes(FI_MAX_WARPS));
}
template <int AA> static cudaError_t fine_solid_smem_limit() {
    return cudaFuncSetAttribute(k_fine_solid<AA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FineSmem<AA>::bytes(FI_SOLID_WARPS));
}
// c_unorm of this object (k_fine.o and k_fine_bg.o each have their own), and the shared-memory limits of the kernels in `set`
static cudaError_t fine_init(const FineInit *set, int n) {
    float h[256];
    for (int i = 0; i < 256; i++) h[i] = (float)i / 255.0f;
    cudaError_t e = cudaMemcpyToSymbol(c_unorm, h, sizeof h);
    // the kernels use more than the default 48 KB of dynamic shared memory per CTA
    for (int k = 0; k < n; k++)
        if (e == cudaSuccess) e = set[k]();
    return e;
}

// k_fine<aa + FLAGS>, with FineArgs alone unless FLAGS has FI_DST, and FineDstArgs unless it has FI_BG
template <int FLAGS> static void launch_fine(int aa, uint32_t grid, uint32_t warps, cudaStream_t st, const VbConfig &cfg, const FineBgArgs &A) {
    const FineArgsOf<FLAGS> &a = A;
    if (aa == 0) k_fine<0 + FLAGS><<<grid, 32u * warps, FineSmem<0>::bytes(warps), st>>>(cfg, a);
    else if (aa == 1) k_fine<1 + FLAGS><<<grid, 32u * warps, FineSmem<1>::bytes(warps), st>>>(cfg, a);
    else k_fine<2 + FLAGS><<<grid, 32u * warps, FineSmem<2>::bytes(warps), st>>>(cfg, a);
}

#ifdef VB_FINE_BG
// k_fine_bg.o: the FI_BG instantiations, launched by vb_launch_fine
extern "C" int vb_fine_bg_init(void) {
    const FineInit set[] = {fine_smem_limit<0 + FI_DST + FI_BG>, fine_smem_limit<1 + FI_DST + FI_BG>,
                                                 fine_smem_limit<2 + FI_DST + FI_BG>};
    return (int)fine_init(set, 3);
}
extern "C" void vb_launch_fine_bg(int aa, uint32_t grid, uint32_t warps, cudaStream_t st, const VbConfig &cfg, const FineBgArgs &A) {
    launch_fine<FI_DST + FI_BG>(aa, grid, warps, st, cfg, A);
}
#else
extern "C" int vb_fine_bg_init(void);
extern "C" void vb_launch_fine_bg(int aa, uint32_t grid, uint32_t warps, cudaStream_t st, const VbConfig &cfg, const FineBgArgs &A);

extern "C" int vb_fine_init_constants(void) {
    const FineInit set[] = {
        fine_smem_limit<0>, fine_smem_limit<0 + FI_DMG>, fine_smem_limit<0 + FI_DST>, fine_smem_limit<0 + FI_DST + FI_DMG>,
        fine_smem_limit<1>, fine_smem_limit<1 + FI_DMG>, fine_smem_limit<1 + FI_DST>, fine_smem_limit<1 + FI_DST + FI_DMG>,
        fine_smem_limit<2>, fine_smem_limit<2 + FI_DMG>, fine_smem_limit<2 + FI_DST>, fine_smem_limit<2 + FI_DST + FI_DMG>,
        fine_solid_smem_limit<0>, fine_solid_smem_limit<1>, fine_solid_smem_limit<2>};
    const cudaError_t e = fine_init(set, 15);
    return e != cudaSuccess ? (int)e : vb_fine_bg_init();
}

// Persistent grid of `max_warps`-warp CTAs, `minb` per SM, for n tiles: small frames get smaller CTAs so that their tiles still
// spread over the SMs.
static void fine_grid(uint32_t n, int sm_count, uint32_t max_warps, uint32_t minb, uint32_t *grid, uint32_t *warps) {
    uint32_t w = max_warps;
    while (w > 2u && (n + w - 1u) / w < (uint32_t)sm_count * minb) w >>= 1;
    *warps = w;
    *grid = std::min((n + w - 1u) / w, (uint32_t)sm_count * minb * (max_warps / w));
}

// The launch's tile queue is control-block word VB_CTL_FINE_QUEUE + band, zeroed with the control block (8 of them, one per
// read-back band); the k_fine after k_fine_solid takes VB_CTL_FINE_QUEUE_FLAGGED.
extern "C" uint32_t vb_launch_fine(const VbConfig &cfg, const VbFrameBufs &b, const VbFineOut &o, const VbFineBg &bg, int aa, uint32_t cull,
                                   uint32_t band, bool cls_order, cudaStream_t st) {
    uint32_t rows = cfg.win_ty1 - cfg.win_ty0;
    uint32_t n = cfg.width_in_tiles * rows;
    if (n == 0) return 0;
    uint32_t grid, warps;
    fine_grid(n, b.sm_count, FI_MAX_WARPS, FI_MINB, &grid, &warps);
    FineBgArgs A;
    A.segments = b.segments; A.ptcl = b.ptcl; A.info = b.info_bin_data; A.blend_spill = b.blend_spill; A.out = o.out; A.ramps = b.ramps; A.atlas = b.atlas;
    A.mask_lut = aa == 2 ? b.mask16 : b.mask8;
    A.cull = cull;
    A.tile_start = b.tile_start;
    A.bump = b.bump();
    A.queue = b.ctl + VB_CTL_FINE_QUEUE + band;
    A.cls_list = b.cls_list;
    A.cls_count = cls_order ? b.ctl + VB_CTL_FINE_CLASS : nullptr;
    A.cls_stride = cfg.width_in_tiles * cfg.tile_rows;
    A.lists = FI_LISTS_ALL;
    A.surf = o.surf;
    A.swz = o.swz;
    A.array = o.array;
    A.x0 = o.x0;
    A.y0 = o.y0;
    A.texel = o.texel;
    A.premul = o.premul;
    A.bg = bg;
    const bool dmg = b.dmg.mode == VB_DMG_INCREMENTAL && cls_order; // the damaged tiles of coarse's lists only
    if (bg.on) {
        // always the FI_DST store (a plain pointer as linear RGBA8, straight alpha, bytes in place), never FI_DMG: a frame with a
        // background is full (damage_prepare)
        if (!o.dst) {
            A.swz = 0x3210u;
            A.texel = 4u;
        }
        vb_launch_fine_bg(aa, grid, warps, st, cfg, A);
    } else if (o.dst) {
        if (dmg) launch_fine<FI_DST + FI_DMG>(aa, grid, warps, st, cfg, A);
        else launch_fine<FI_DST>(aa, grid, warps, st, cfg, A);
    } else if (dmg) {
        launch_fine<FI_DMG>(aa, grid, warps, st, cfg, A);
    } else if (cls_order && cull != 0u) {
        // the simple tiles' lists in k_fine_solid, then the flagged ones in k_fine, whose tile count is read on the device (its
        // CTAs leave at once when there are none). Both grids are the machine's: only the lists say which tiles each paints.
        uint32_t grid_s, warps_s;
        fine_grid(n, b.sm_count, FI_SOLID_WARPS, FI_SOLID_MINB, &grid_s, &warps_s);
        FineArgs As = A;
        As.lists = FI_LISTS_SIMPLE;
        if (aa == 0) k_fine_solid<0><<<grid_s, 32u * warps_s, FineSmem<0>::bytes(warps_s), st>>>(cfg, As);
        else if (aa == 1) k_fine_solid<1><<<grid_s, 32u * warps_s, FineSmem<1>::bytes(warps_s), st>>>(cfg, As);
        else k_fine_solid<2><<<grid_s, 32u * warps_s, FineSmem<2>::bytes(warps_s), st>>>(cfg, As);
        A.lists = FI_LISTS_FLAGGED;
        A.queue = b.ctl + VB_CTL_FINE_QUEUE_FLAGGED;
        launch_fine<0>(aa, grid, warps, st, cfg, A);
        return 2;
    } else {
        launch_fine<0>(aa, grid, warps, st, cfg, A);
    }
    return 1;
}
#endif
