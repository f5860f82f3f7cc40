// k_compose.cu -- composition of resident fragments (vb_compose): the six streams of the scene
//   Scene::new(); for k: append(&fragment[k], transform_k)            (vello/src/scene.rs:464-469, encoding.rs:94-174)
// written in one launch from the fragments' device copies, without the host touching a stream byte.
//
// The launch is driven by the destination. Per stream the host stages the exclusive prefix of the instances' lengths (tag
// bytes, words, or transforms for the transform stream), so the destination of instance k's part of stream s starts at
// prefix[s][k]. The destination units of the six streams (tag WORDS, words, whole transforms) are cut into chunks of
// CP_UNITS_PER_CTA; every CTA takes one chunk and each of its threads the units threadIdx.x + j * CP_THREADS of it, so the
// grid covers one 14 MB fragment and ten thousand tiny ones alike. A thread finds the instance of its unit by binary search
// over the prefix, narrowed to the instances the CTA's chunk spans (no search at all inside a large fragment).
//
// Path tags are bytes and an instance starts at any byte offset, so a destination tag word can hold the tags of several
// instances: every destination word is assembled in registers and stored whole by the one thread that owns it. Bytes past
// the last tag are stored as zero; k_resolve_finish, which runs next, writes the padding and the PATH tags of open clips.
// Transforms are written whole, multiplied by the instance's transform (vb_affine_mul: Encoding::append's f32 product) when
// it has one. Patch words of the draw data are copied as the encoder left them; k_resolve_finish patches them too.
//
// k_instance_transforms, at the end, is the per-frame half of bound instance transforms: the transform stream again, with each
// instance's transform read from device memory when the frame runs.
#include "vb_device.cuh"
#include "vb_stages.h"

#define CP_THREADS 256u
#define CP_ITEMS 4u
#define CP_UNITS_PER_CTA (CP_THREADS * CP_ITEMS)

// stream s of instance k in its fragment's allocation: the fragment starts with the word offsets of its six streams
__device__ __forceinline__ const uint32_t *cp_stream(const CmpArgs &a, uint32_t k, uint32_t s) {
    const uint32_t *base = reinterpret_cast<const uint32_t *>(__ldg(a.src + k));
    return base + __ldg(base + s);
}

__global__ void __launch_bounds__(CP_THREADS) k_compose_streams(const CmpArgs a) {
    // the stream of this CTA, and its parameters (selected with constant indices: the parameter arrays stay in registers)
    const uint32_t b = blockIdx.x;
    uint32_t s = 0u;
#pragma unroll
    for (int i = 1; i < 6; i++) s += b >= a.cta0[i] ? 1u : 0u;
    uint32_t cta0 = 0u, units = 0u, dst = 0u;
#pragma unroll
    for (int i = 0; i < 6; i++)
        if ((uint32_t)i == s) {
            cta0 = a.cta0[i];
            units = a.units[i];
            dst = a.dst[i];
        }
    const uint32_t *__restrict__ P = a.prefix + (size_t)s * (a.n + 1u);
    const uint32_t u0 = (b - cta0) * CP_UNITS_PER_CTA, u1 = min(u0 + CP_UNITS_PER_CTA, units);
    // the instances the chunk spans (elements: tag bytes for the tag stream, else units)
    __shared__ uint32_t span[2];
    if (threadIdx.x < 2u) {
        uint32_t x = threadIdx.x == 0u ? u0 : u1 - 1u;
        if (s == 0u) x = threadIdx.x == 0u ? 4u * u0 : min(4u * u1, __ldg(P + a.n)) - 1u;
        span[threadIdx.x] = cp_find(P, 0u, a.n - 1u, x);
    }
    __syncthreads();
    const uint32_t kf = span[0], kl = span[1];
    uint32_t *__restrict__ out = a.scene + dst;

    if (s == 0u) { // path tags: word u holds tag bytes 4u .. 4u + 3
        const uint32_t total = __ldg(P + a.n);
        for (uint32_t u = u0 + threadIdx.x; u < u1; u += CP_THREADS) {
            const uint32_t b0 = 4u * u;
            uint32_t k = cp_find(P, kf, kl, b0);
            uint32_t p0 = __ldg(P + k), p1 = __ldg(P + k + 1u);
            const uint32_t *tags = cp_stream(a, k, 0u);
            uint32_t word = 0u;
            if (b0 + 3u < p1) { // all four bytes in instance k: two aligned source words, one funnel shift
                const uint32_t o = b0 - p0, sh = 8u * (o & 3u);
                const uint32_t w0 = __ldg(tags + (o >> 2));
                const uint32_t w1 = sh ? __ldg(tags + (o >> 2) + 1u) : 0u;
                word = __funnelshift_r(w0, w1, sh);
            } else { // the word crosses instances (or the end of the stream): byte by byte
                for (uint32_t i = 0u; i < 4u && b0 + i < total; i++) {
                    const uint32_t bi = b0 + i;
                    while (bi >= p1) { // the next instance with tags
                        k++;
                        p0 = p1;
                        p1 = __ldg(P + k + 1u);
                        tags = cp_stream(a, k, 0u);
                    }
                    word |= (uint32_t)__ldg(reinterpret_cast<const uint8_t *>(tags) + (bi - p0)) << (8u * i);
                }
            }
            out[u] = word;
        }
    } else if (s == 4u) { // transforms: unit u is transform u, written whole
        for (uint32_t u = u0 + threadIdx.x; u < u1; u += CP_THREADS) {
            const uint32_t k = cp_find(P, kf, kl, u);
            const uint32_t *src = cp_stream(a, k, 4u) + 6u * (u - __ldg(P + k));
            float t[6], r[6];
#pragma unroll
            for (int i = 0; i < 6; i++) t[i] = __uint_as_float(__ldg(src + i));
            const CmpXform x = a.xf[k];
            if (x.on) {
                vb_affine_mul(x.m, t, r);
            } else {
#pragma unroll
                for (int i = 0; i < 6; i++) r[i] = t[i];
            }
#pragma unroll
            for (int i = 0; i < 6; i++) out[6u * u + i] = __float_as_uint(r[i]);
        }
    } else { // path data, draw tags, draw data, styles: word for word; the loads of a thread's units are issued together
        uint32_t v[CP_ITEMS];
#pragma unroll
        for (uint32_t j = 0u; j < CP_ITEMS; j++) {
            const uint32_t u = u0 + j * CP_THREADS + threadIdx.x;
            v[j] = 0u;
            if (u < u1) {
                const uint32_t k = cp_find(P, kf, kl, u);
                v[j] = __ldg(cp_stream(a, k, s) + (u - __ldg(P + k)));
            }
        }
#pragma unroll
        for (uint32_t j = 0u; j < CP_ITEMS; j++) {
            const uint32_t u = u0 + j * CP_THREADS + threadIdx.x;
            if (u < u1) out[u] = v[j];
        }
    }
}

// Bound instance transforms (vb_bind_instance_transforms): transform u of the composed scene belongs to instance
// k = cp_find(prefix, u) and is rendered as row_k * T, the product vb_compose makes for transform = row k, T being the
// fragment's untransformed transform. A row with a coefficient that is not finite leaves its instance as composed (the
// compose-time transform, or T itself for an instance appended without one), so that no NaN reaches flatten.
__global__ void __launch_bounds__(256) k_instance_transforms(const uint8_t *__restrict__ rows, uint32_t pitch, const uint32_t *__restrict__ prefix,
                                                             const CmpXform *__restrict__ xf, const uint32_t *__restrict__ src, uint32_t *dst,
                                                             uint32_t n, uint32_t n_transforms) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_transforms) return;
    const uint32_t k = cp_find(prefix, 0u, n - 1u, u);
    const float *row = reinterpret_cast<const float *>(rows + (size_t)k * pitch);
    float m[6], t[6], r[6];
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 6; i++) {
        m[i] = __ldg(row + i);
        finite = finite && isfinite(m[i]);
        t[i] = __uint_as_float(__ldg(src + 6u * u + i));
    }
    bool on = true;
    if (!finite) {
        const CmpXform x = xf[k];
        on = x.on != 0u;
#pragma unroll
        for (int i = 0; i < 6; i++) m[i] = x.m[i];
    }
    if (on) {
        vb_affine_mul(m, t, r);
    } else {
#pragma unroll
        for (int i = 0; i < 6; i++) r[i] = t[i];
    }
#pragma unroll
    for (int i = 0; i < 6; i++) dst[6u * u + i] = __float_as_uint(r[i]);
}

extern "C" uint32_t vb_launch_instance_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbRows &rows = b.bound.rows[VB_BIND_INSTANCES];
    if (!rows.rows) return 0u;
    // the bound region prepare reserved: at transform_base, or with a view on top of it at the view's source (view_src)
    const uint32_t n = b.xf_len;
    if (n == 0u) return 0u;
    uint32_t *dst = const_cast<uint32_t *>(b.scene) + (b.view ? cfg.view_src : cfg.layout.transform_base);
    k_instance_transforms<<<(n + 255u) / 256u, 256, 0, st>>>(rows.rows, rows.pitch, b.bound.inst_prefix, b.bound.inst_xf, b.bound.inst_src, dst,
                                                             rows.n, n);
    return 1u;
}

extern "C" uint32_t vb_launch_compose(CmpArgs a, cudaStream_t st) {
    uint64_t ctas = 0u;
    for (int s = 0; s < 6; s++) {
        a.cta0[s] = (uint32_t)ctas;
        ctas += (a.units[s] + CP_UNITS_PER_CTA - 1u) / CP_UNITS_PER_CTA;
    }
    if (ctas == 0u || a.n == 0u) return 0u;
    k_compose_streams<<<(uint32_t)ctas, CP_THREADS, 0, st>>>(a);
    return 1u;
}
