// k_exchange.cu -- flatten sharded by tag range across the GPUs of one box, with the line soup exchanged through peer memory.
//
// SURVEY.md 8(e) option B. In the stripe split every GPU needs the lines that touch ITS tile rows and the bounding box of
// every path; computing them is the stage that does not shrink with the stripe (the replicated floor of round 1,
// largest on the cubic-heavy workload). Here GPU r flattens only partitions
// [P*r/G, P*(r+1)/G) of the tag stream and the results are exchanged over NVLink / NVSwitch WITHOUT a host round trip or a
// library collective -- peers read each other's memory directly and synchronise through flags in that memory:
//
//   k_route_count / k_route_scatter   sort my lines by destination stripe (a line goes to every stripe whose pixel rows it
//                                     touches, +-1 px) into my OUTBOX, a region of my exchange arena
//   k_xsignal                         publish {offset, count} per destination, fence, then store the frame's epoch into
//                                     flags[me] of EVERY peer's arena (st.release.sys through the peer mapping)
//   k_xwait                           spin (ld.acquire.sys) until flags[s] >= epoch for every source s  [bounded: times out]
//   k_bbox_combine                    PathBbox[p] = min/max over the peers' partial boxes (read through the peer mappings)
//   k_lines_pull                      copy {source 0's lines for me, source 1's, ...} into my `lines` arena, set bump.lines
//
// Lines keep the order (source rank, then the source's own order), i.e. a subsequence of the single-GPU order up to the
// routing kernel's block order; everything downstream is order-insensitive exactly as on one GPU (per-tile segment slots
// come from atomics there too) and MSAA pixels are integer sample counts, so the assembled frame is bit-identical.
// The arena has two halves used by even / odd epochs: a GPU can only be one frame ahead of its slowest peer (it cannot
// pass k_xwait of frame e+1 before every peer has signalled e+1, i.e. finished reading frame e), so half (e & 1) is never
// overwritten while somebody still reads it. Works across processes (arenas exported with CUDA IPC) and inside one
// (vb_group), and -- for the tests -- between several renderers on ONE GPU.
#include "vb_device.cuh"
#include "vb_stages.h"

// layout of one arena half (bytes): [XHdr 256][VbPathBbox x n_paths][pad to 256][VbLineSoup x lines_cap]
struct XHdr {
    uint32_t off[XG_MAX + 1]; // outbox offset of destination d's lines (in lines), off[G] = total
    uint32_t pad[64 - (XG_MAX + 1)];
};
// An arena: [flags: XG_MAX words][epoch counter: word 16][pad to 256 B][half 0][half 1]. The epoch counter is advanced by the
// frame's first kernel (k_frame_init, vb_frame.cu) and READ by the kernels below, so a captured CUDA graph replays correctly.
// The peer table (XPeers) is in vb_stages.h.
#define X_EPOCH_WORD 16u
__device__ __forceinline__ uint32_t x_epoch(const XPeers &X) { return *(reinterpret_cast<const volatile uint32_t *>(X.base[X.rank]) + X_EPOCH_WORD); }
__device__ __forceinline__ unsigned char *x_half(const XPeers &X, uint32_t s, uint32_t epoch) {
    return X.base[s] + 256 + ((epoch & 1u) ? X.half_bytes : 0ull);
}
__device__ __forceinline__ uint32_t *x_flags(const XPeers &X, uint32_t s) { return reinterpret_cast<uint32_t *>(X.base[s]); }
__host__ __device__ inline size_t x_bbox_off() { return 256; }
__host__ __device__ inline size_t x_lines_off(uint32_t n_paths) { return (256 + (size_t)n_paths * sizeof(VbPathBbox) + 255) & ~(size_t)255; }
extern "C" size_t vb_exchange_half_bytes(uint32_t n_paths, uint32_t lines_cap) { return x_lines_off(n_paths) + (size_t)lines_cap * sizeof(VbLineSoup) + 256; }
extern "C" uint32_t vb_exchange_epoch_word(void) { return X_EPOCH_WORD; }

__device__ __forceinline__ uint32_t x_dest_mask(const XPeers &X, float y0, float y1) {
    const float lo = fminf(y0, y1), hi = fmaxf(y0, y1);
    uint32_t m = 0u;
    for (uint32_t d = 0; d < X.world; d++) {
        const float top = (float)(X.rows[d] * VB_TILE_HEIGHT) - 1.0f, bot = (float)(X.rows[d + 1] * VB_TILE_HEIGHT) + 1.0f;
        // written so that a NaN coordinate (degenerate strokes produce them) is sent everywhere, as the replicated path keeps it
        if (!(hi < top) && !(lo > bot) && X.rows[d + 1] > X.rows[d]) m |= 1u << d;
    }
    return m;
}

// counts[d] += lines of mine that destination d needs (ballots per destination: one shared-memory atomic per warp and stripe)
__global__ void __launch_bounds__(256)
k_route_count(XPeers X, const VbBump *__restrict__ bump, uint32_t lines_size, const VbLineSoup *__restrict__ lines, uint32_t *counts) {
    __shared__ uint32_t sh[XG_MAX];
    if (threadIdx.x < XG_MAX) sh[threadIdx.x] = 0u;
    __syncthreads();
    const uint32_t n = min(bump->lines, lines_size);
    const uint32_t lane = vb_lane();
    uint32_t acc = 0u; // lane d accumulates destination d's count of this warp
    for (uint32_t base = blockIdx.x * 256u; base < n; base += gridDim.x * 256u) {
        const uint32_t i = base + threadIdx.x;
        uint32_t m = 0u;
        if (i < n) {
            const uint2 *lp = reinterpret_cast<const uint2 *>(lines + i);
            const uint2 a = __ldg(lp + 1), b = __ldg(lp + 2);
            m = x_dest_mask(X, __uint_as_float(a.y), __uint_as_float(b.y));
        }
        for (uint32_t d = 0; d < X.world; d++) {
            const uint32_t c = (uint32_t)__popc(__ballot_sync(VB_FULL, (m >> d) & 1u));
            if (lane == d) acc += c;
        }
    }
    if (lane < X.world && acc != 0u) atomicAdd(&sh[lane], acc);
    __syncthreads();
    if (threadIdx.x < X.world && sh[threadIdx.x] != 0u) atomicAdd(&counts[threadIdx.x], sh[threadIdx.x]);
}

// outbox[off[d] + ...] = my lines for destination d (off = exclusive prefix of counts). Slots: rank inside the warp from a
// ballot, warp base from one shared-memory atomic per (warp, stripe), block base from one global atomic per (block, stripe).
__global__ void __launch_bounds__(256)
k_route_scatter(XPeers X, VbBump *bump, uint32_t lines_size, const VbLineSoup *__restrict__ lines, const uint32_t *__restrict__ counts,
                uint32_t *cursors) {
    __shared__ uint32_t sh_cnt[XG_MAX], sh_base[XG_MAX], sh_off[XG_MAX + 1];
    VbLineSoup *outbox = reinterpret_cast<VbLineSoup *>(x_half(X, X.rank, x_epoch(X)) + x_lines_off(X.n_paths));
    if (threadIdx.x == 0u) {
        uint32_t acc = 0u;
        for (uint32_t d = 0; d < X.world; d++) { sh_off[d] = acc; acc += counts[d]; }
        sh_off[X.world] = acc;
        if (acc > X.lines_cap && blockIdx.x == 0u) atomicOr(&bump->failed, VB_STAGE_EXCHANGE);
    }
    const uint32_t n = min(bump->lines, lines_size);
    const uint32_t lane = vb_lane();
    for (uint32_t base = blockIdx.x * 256u; base < n; base += gridDim.x * 256u) {
        if (threadIdx.x < XG_MAX) sh_cnt[threadIdx.x] = 0u;
        __syncthreads();
        const uint32_t i = base + threadIdx.x;
        uint32_t m = 0u;
        uint2 w0 = make_uint2(0u, 0u), w1 = w0, w2 = w0;
        if (i < n) {
            const uint2 *lp = reinterpret_cast<const uint2 *>(lines + i);
            w0 = __ldg(lp); w1 = __ldg(lp + 1); w2 = __ldg(lp + 2);
            m = x_dest_mask(X, __uint_as_float(w1.y), __uint_as_float(w2.y));
        }
        // pass 1: slot of each (line, destination) inside the block
        uint32_t slot_lo = 0u, slot_hi = 0u; // 8 destinations x 8 bits: my slot inside the block for each of them (< 256)
        for (uint32_t d = 0; d < X.world; d++) {
            const uint32_t b = __ballot_sync(VB_FULL, (m >> d) & 1u);
            uint32_t wbase = 0u;
            if (b != 0u && lane == (uint32_t)(__ffs((int)b) - 1)) wbase = atomicAdd(&sh_cnt[d], (uint32_t)__popc(b));
            wbase = __shfl_sync(VB_FULL, wbase, b != 0u ? __ffs((int)b) - 1 : 0);
            const uint32_t sl = (wbase + (uint32_t)__popc(b & ((1u << lane) - 1u))) & 0xffu;
            if (d < 4u) slot_lo |= sl << (8u * d); else slot_hi |= sl << (8u * (d - 4u));
        }
        __syncthreads();
        if (threadIdx.x < X.world) sh_base[threadIdx.x] = sh_cnt[threadIdx.x] ? atomicAdd(&cursors[threadIdx.x], sh_cnt[threadIdx.x]) : 0u;
        __syncthreads();
        for (uint32_t mm = m; mm;) {
            const uint32_t d = (uint32_t)__ffs((int)mm) - 1u;
            mm &= mm - 1u;
            const uint32_t sl = d < 4u ? (slot_lo >> (8u * d)) & 0xffu : (slot_hi >> (8u * (d - 4u))) & 0xffu;
            const uint32_t o = sh_off[d] + sh_base[d] + sl;
            if (o < X.lines_cap) {
                uint2 *dst = reinterpret_cast<uint2 *>(outbox + o);
                dst[0] = w0; dst[1] = w1; dst[2] = w2;
            }
        }
        __syncthreads();
    }
}

// my partial path boxes (flatten wrote them into the renderer's own array) -> my arena half, where the peers read them
__global__ void __launch_bounds__(256) k_bbox_publish(XPeers X, const VbPathBbox *__restrict__ local) {
    const uint32_t p = blockIdx.x * 256u + threadIdx.x;
    if (p >= X.n_paths) return;
    const uint2 *src = reinterpret_cast<const uint2 *>(local + p);
    uint2 *dst = reinterpret_cast<uint2 *>(x_half(X, X.rank, x_epoch(X)) + x_bbox_off() + (size_t)p * sizeof(VbPathBbox));
    dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
}

// publish the header of my arena half, then raise my flag in every peer's arena
__global__ void k_xsignal(XPeers X, const uint32_t *__restrict__ counts) {
    const uint32_t epoch = x_epoch(X);
    XHdr *hdr = reinterpret_cast<XHdr *>(x_half(X, X.rank, epoch));
    if (threadIdx.x == 0u) {
        uint32_t acc = 0u;
        for (uint32_t d = 0; d < X.world; d++) { hdr->off[d] = acc; acc += counts[d]; }
        hdr->off[X.world] = acc;
    }
    __syncthreads();
    __threadfence_system(); // outbox, boxes and header are visible system-wide before any flag is
    if (threadIdx.x < X.world) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(x_flags(X, threadIdx.x) + X.rank), "r"(epoch) : "memory");
}

// wait until every source has raised its flag for this epoch (flags live in MY arena). Bounded: a peer that never
// arrives (a rank that died) turns into a failed frame, not a hung GPU.
__global__ void k_xwait(XPeers X, VbBump *bump, unsigned long long timeout_cycles) {
    if (threadIdx.x >= X.world) return;
    const uint32_t epoch = x_epoch(X);
    const uint32_t *f = x_flags(X, X.rank) + threadIdx.x;
    const unsigned long long t0 = clock64();
    for (;;) {
        uint32_t v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
        if ((int32_t)(v - epoch) >= 0) break;
        if ((unsigned long long)(clock64() - t0) > timeout_cycles) {
            atomicOr(&bump->failed, VB_STAGE_EXCHANGE);
            break;
        }
        __nanosleep(200);
    }
}

// PathBbox of every path = union of the partial boxes the peers computed from their tag ranges
__global__ void __launch_bounds__(256) k_bbox_combine(XPeers X, VbPathBbox *out) {
    const uint32_t p = blockIdx.x * 256u + threadIdx.x;
    if (p >= X.n_paths) return;
    VbPathBbox r;
    r.x0 = 0x7fffffff; r.y0 = 0x7fffffff; r.x1 = (int32_t)0x80000000; r.y1 = (int32_t)0x80000000; r.draw_flags = 0u; r.trans_ix = 0u;
    const uint32_t epoch = x_epoch(X);
    for (uint32_t s = 0; s < X.world; s++) {
        const uint2 *src = reinterpret_cast<const uint2 *>(x_half(X, s, epoch) + x_bbox_off() + (size_t)p * sizeof(VbPathBbox));
        const uint2 a = src[0], b = src[1], c = src[2]; // plain loads: the data may live in another GPU
        r.x0 = min(r.x0, (int32_t)a.x); r.y0 = min(r.y0, (int32_t)a.y);
        r.x1 = max(r.x1, (int32_t)b.x); r.y1 = max(r.y1, (int32_t)b.y);
        r.draw_flags = max(r.draw_flags, c.x); // written once, by the GPU that holds the path's PATH tag; 0 elsewhere
        r.trans_ix = max(r.trans_ix, c.y);
    }
    out[p] = r;
}

// lines = concat over sources s of outbox_s[off_s[me] .. off_s[me + 1])
__global__ void __launch_bounds__(256) k_lines_pull(XPeers X, VbBump *bump, uint32_t lines_size, VbLineSoup *lines) {
    __shared__ uint32_t sh_pre[XG_MAX + 1], sh_src0[XG_MAX];
    const uint32_t epoch = x_epoch(X);
    if (threadIdx.x == 0u) {
        uint32_t acc = 0u;
        for (uint32_t s = 0; s < X.world; s++) {
            const XHdr *h = reinterpret_cast<const XHdr *>(x_half(X, s, epoch));
            const uint32_t o0 = h->off[X.rank], o1 = h->off[X.rank + 1u];
            sh_pre[s] = acc;
            sh_src0[s] = o0;
            acc += o1 - o0;
        }
        sh_pre[X.world] = acc;
        if (blockIdx.x == 0u) {
            bump->lines = acc;
            if (acc > lines_size) atomicOr(&bump->failed, VB_STAGE_FLATTEN);
        }
    }
    __syncthreads();
    const uint32_t total = min(sh_pre[X.world], lines_size);
    // a line is three 8-byte words: consecutive threads move consecutive words, so every warp reads and writes 256
    // contiguous bytes whether the source is local or behind NVLink
    uint2 *dflat = reinterpret_cast<uint2 *>(lines);
    for (uint64_t j = (uint64_t)blockIdx.x * 256u + threadIdx.x; j < (uint64_t)total * 3u; j += (uint64_t)gridDim.x * 256u) {
        const uint32_t i = (uint32_t)(j / 3u), part = (uint32_t)(j - (uint64_t)i * 3u);
        uint32_t s = 0u;
        for (uint32_t q = 1; q < X.world; q++)
            if (i >= sh_pre[q]) s = q;
        const uint2 *src = reinterpret_cast<const uint2 *>(reinterpret_cast<const VbLineSoup *>(x_half(X, s, epoch) + x_lines_off(X.n_paths)) + sh_src0[s] +
                                                           (i - sh_pre[s]));
        dflat[j] = src[part];
    }
}

// counts / cursors: 2 * XG_MAX words of scratch in the control block (zeroed with it at frame start).
// send = everything up to raising my flags; recv = wait for the peers, combine the boxes, pull my lines. They are separate
// entry points so that a host driving several renderers on ONE device can issue every send before any recv (a wait kernel
// never sits in front of the signal it waits for in a shared hardware queue).
extern "C" uint32_t vb_launch_exchange_send(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &X, cudaStream_t st) {
    const uint32_t grid = (uint32_t)b.sm_count * 8u;
    uint32_t *scratch = b.ctl + VB_CTL_XCHG_SCRATCH;
    k_route_count<<<grid, 256, 0, st>>>(X, b.bump(), cfg.lines_size, b.lines, scratch);
    k_route_scatter<<<grid, 256, 0, st>>>(X, b.bump(), cfg.lines_size, b.lines, scratch, scratch + XG_MAX);
    if (X.n_paths) k_bbox_publish<<<(X.n_paths + 255u) / 256u, 256, 0, st>>>(X, b.path_bboxes);
    k_xsignal<<<1, 32, 0, st>>>(X, scratch);
    return X.n_paths ? 4 : 3;
}
extern "C" uint32_t vb_launch_exchange_recv(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &X, cudaStream_t st) {
    const uint32_t grid = (uint32_t)b.sm_count * 8u;
    k_xwait<<<1, 32, 0, st>>>(X, b.bump(), 4000000000ull); // ~2 s at 2 GHz
    if (X.n_paths) k_bbox_combine<<<(X.n_paths + 255u) / 256u, 256, 0, st>>>(X, b.path_bboxes);
    k_lines_pull<<<grid, 256, 0, st>>>(X, b.bump(), cfg.lines_size, b.lines);
    return X.n_paths ? 3 : 2;
}
