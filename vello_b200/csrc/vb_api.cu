// vb_api.cu -- host orchestration + the extern "C" ABI declared in include/vello_b200.h.
//
// Replaces vello/src/render.rs (graph: stage order, bindings, buffer lifetimes) and
// vello/src/wgpu_engine.rs (engine) with a CUDA-stream pipeline. Unlike the reference
// (config.rs:398-408 fixed `1 << 21` arenas; lib.rs:762 "TODO: re-run on overflow") every
// bump-allocated arena is sized from the scene and grown + re-run when a frame overflows.
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/vello_b200.h"
#include "vb_device.cuh"
#include "vb_stages.h"
#include "vb_textures.h"
#include "vb_types.h"

// path_tiling_setup.wgsl:21-26 flags a failed frame to fine through ptcl[0] = ~0. That word is also tile 0's blend offset
// and is only rewritten when coarse visits tile 0 -- which a stripe window with bin_row0 > 0 never does, so the flag of a
// failed attempt would outlive the successful re-run and every later frame of that renderer. fine therefore reads
// bump.failed (zeroed with the control block at the start of every attempt) directly; ptcl[0] is not used as a flag.

// Statistics for the roofline of `fine`: PTCL words each tile's interpreter reads and segments it
// references (one thread per tile walks its command stream, as fine does).
__global__ void k_ptcl_stats(VbConfig cfg, const uint32_t *__restrict__ ptcl, const uint32_t *__restrict__ tile_start,
                             unsigned long long *out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t wt = cfg.width_in_tiles, rows = cfg.win_ty1 - cfg.win_ty0;
    if (t >= wt * rows) return;
    uint32_t tile_ix = (cfg.win_ty0 + t / wt) * wt + t % wt;
    uint32_t ix = tile_ix * VB_PTCL_INITIAL_ALLOC + 1u;
    unsigned long long words = 1, segs = 0, fills = 0;
    if (tile_start && tile_start[tile_ix]) { // occlusion start: the interpreter begins at the tile's last opaque cover
        ix = tile_start[tile_ix];
        words += 1;
    }
    for (uint32_t guard = 0; guard < (1u << 24); guard++) {
        uint32_t tag = ptcl[ix];
        uint32_t size = 1;
        if (tag == VB_CMD_END) { words += 1; break; }
        if (tag == VB_CMD_JUMP) { words += 2; ix = ptcl[ix + 1]; continue; }
        if (tag == VB_CMD_FILL) { size = 4; segs += ptcl[ix + 1] >> 1; fills++; }
        else if (tag == VB_CMD_COLOR || tag == VB_CMD_IMAGE) size = 2;
        else if (tag == VB_CMD_LIN_GRAD || tag == VB_CMD_RAD_GRAD || tag == VB_CMD_SWEEP_GRAD || tag == VB_CMD_END_CLIP || tag == VB_CMD_BLUR_RECT) size = 3;
        words += size;
        ix += size;
    }
    atomicAdd(out, words);
    atomicAdd(out + 1, segs);
    atomicAdd(out + 2, fills);
}

// Frame start: zero the control block (bump counters, look-back descriptors, fine's tile queues) and reset the path bounding
// boxes (bbox_clear.wgsl: (+INT_MAX, -INT_MAX)) -- one launch; blocks past the control block clear 256 boxes each.
__global__ void k_frame_init(uint32_t *ctl, uint32_t words, uint32_t ctl_blocks, VbPathBbox *path_bboxes, uint32_t n_paths, uint32_t *xepoch) {
    if (xepoch != nullptr && blockIdx.x == 0u && threadIdx.x == 0u) *xepoch += 1u; // multi-GPU exchange: this attempt's epoch
    if (blockIdx.x < ctl_blocks) {
        for (uint32_t i = blockIdx.x * 1024u + threadIdx.x; i < min(words, (blockIdx.x + 1u) * 1024u); i += 256u) ctl[i] = 0u;
    } else {
        const uint32_t i = (blockIdx.x - ctl_blocks) * 256u + threadIdx.x;
        if (i < n_paths) {
            VbPathBbox b;
            b.x0 = 0x7fffffff; b.y0 = 0x7fffffff; b.x1 = (int32_t)0x80000000; b.y1 = (int32_t)0x80000000;
            b.draw_flags = 0; b.trans_ix = 0;
            path_bboxes[i] = b;
        }
    }
}
__global__ void k_publish_bump(const VbBump *bump, VbBump *host) {
    if (threadIdx.x < sizeof(VbBump) / 4u) {
        reinterpret_cast<volatile uint32_t *>(host)[threadIdx.x] = reinterpret_cast<const uint32_t *>(bump)[threadIdx.x];
        __threadfence_system();
    }
}

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0; // bytes
};

// the seven bump-allocated arenas, in the order of VbConfig::lines_size .. ptcl_size (ARENAS below)
enum { ARENA_LINES, ARENA_BINNING, ARENA_TILES, ARENA_SEG_COUNTS, ARENA_SEGMENTS, ARENA_BLEND, ARENA_PTCL, N_ARENAS };
static_assert(offsetof(VbConfig, ptcl_size) - offsetof(VbConfig, lines_size) == (N_ARENAS - 1) * sizeof(uint32_t),
              "VbConfig's arena sizes are consecutive words in ARENA_* order");

// Where a frame's pixels go: a device pointer, or the renderer's own target (target_alt when `alt`), and optionally a copy of
// the frame in host memory, read back in `bands` row bands while fine runs.
struct Dest {
    void *dev = nullptr, *host = nullptr;
    bool alt = false;
    uint32_t bands = 1;
};

// key of a captured frame: the inputs of its launches (see enqueue)
struct GraphKey {
    VbConfig cfg;
    VbFrameBufs bufs;
    const void *out;
    const VbBump *h_bump_dev;
    uint32_t aa, cull, last;
    const void *xarena; // exchange: the arena holding the epoch counter, and the peer table; zero while it is off
    XPeers xpeers;
};
static_assert(sizeof(VbFrameBufs) == offsetof(VbFrameBufs, sm_count) + sizeof(int), "VbFrameBufs has no padding (GraphKey is compared bytewise)");
struct GraphSlot {
    GraphKey key;
    cudaGraphExec_t exec = nullptr;
    uint32_t launches = 0;
};

struct vb_renderer {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool timing = false;
    uint32_t max_retries = 6;
    std::string err;
    int sm_count = 132;

    // Streaming (vb_render_begin) keeps TWO frames in flight: while frame k is rasterised, frame k+1's scene is uploaded
    // into the other slot on its own stream and frame k-1's pixels drain to the host. `cur` is the slot frames render from.
    struct SceneSlot {
        bool have_scene = false;
        VbLayout layout{};
        size_t scene_words = 0;
        uint32_t n_ramps = 0, atlas_w = 0, atlas_h = 0;
        DevBuf scene, ramps, atlas;
        VbBump *h_bump = nullptr;     // pinned + mapped: the device writes the counters straight into host memory
        VbBump *h_bump_dev = nullptr; // device-side address of h_bump
        // the images of the last device resolve that were copied from an override, with their atlas places: a dirty one is
        // copied again before the next frame (refresh_overrides), without a new resolve
        struct OverridePlace {
            const void *key;
            const uint8_t *src;
            size_t pitch;
            uint32_t w, h, x, y;
            bool dirty;
        };
        std::vector<OverridePlace> overridden;
    } slot[2];
    SceneSlot *cur = slot;
    DevBuf mask8, mask16;

    // fixed-size intermediates
    DevBuf tag_monoids, path_bboxes, draw_monoids, info_bin_data, clip_inp, clip_bboxes, clip_scratch, draw_bboxes, bin_headers, paths,
        ctl, target, target_alt, tile_start, cls_list;
    // Renderer::override_image: images (by key) whose pixels come from device memory at the device resolve
    struct Override {
        const uint8_t *src;
        size_t pitch;
        uint32_t w, h;
    };
    std::unordered_map<const void *, Override> overrides;
    DevBuf blit_rects;                  // k_atlas_blit's rectangles, staged through blit_host (pinned)
    VbBlitRect *blit_host = nullptr;
    size_t blit_host_cap = 0;           // rectangles
    cudaEvent_t blit_staged = nullptr;  // the last copy out of blit_host
    // bump arenas (ARENAS), capacities in elements
    DevBuf resolve_tmp; // patches, ramp descriptors and stops of vb_scene_upload_streams
    DevBuf lines, line_scratch, flatten_jobs, flatten_parts, tiles, seg_counts, segments, ptcl, blend_spill;
    uint32_t cap[N_ARENAS] = {};
    // test-only capacity limits (vb_debug_limit_arena); UINT32_MAX = none
    uint32_t limit[N_ARENAS] = {UINT32_MAX, UINT32_MAX, UINT32_MAX, UINT32_MAX, UINT32_MAX, UINT32_MAX, UINT32_MAX};

    // batch (vb_set_cells): the draw-object offsets of the cells of the current scene (n_cells + 1 entries, a copy of cell_draw);
    // empty = one cell, no batch. Every scene upload empties it.
    std::vector<uint32_t> cells;
    DevBuf cell_draw;
    bool grouped = false; // a renderer of a vb_group: no batches

    // per-frame
    VbConfig cfg{};
    vb_params params{};
    Dest dest; // of the frame frame_prepare set up
    uint32_t retries = 0, launches = 0;
    VbFrameBufs bufs{};           // the buffers of the frame prepare set up, as the launchers take them
    bool use_graph = true;        // replay whole frames as CUDA graphs (see enqueue)
    GraphSlot graphs[4];
    uint32_t graph_next = 0;
    uint32_t readback_bands = 8; // fine launches per frame when the pixels go to the host (vb_render); 1 while streaming
    uint32_t occlusion_cull = 1; // fine starts each tile at its last opaque full-tile cover
    // path_tiling runs on its own stream beside coarse: forked after backdrop, joined before fine (enqueue_direct)
    cudaStream_t tiling_stream = nullptr;
    cudaEvent_t tiling_fork = nullptr, tiling_join = nullptr;
    cudaEvent_t ev[VB_N_STAGE_IDS + 1]{};
    cudaEvent_t frame_ev[2]{}; // around every whole frame (vb_last_frame_ms: the signal stripe balancing uses)
    bool frame_timed = false;
    bool ev_ok = false;
    // read-back pipeline of vb_render (host output): fine runs in row bands, each band's D2H copy overlaps the next band
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t band_ev[8]{};
    // streaming read-back (vb_render_begin): frames alternate between two targets so that the copy of frame n can
    // still be draining while frame n+1 is rasterised
    bool stream_pending = false;
    cudaEvent_t copy_done[3]{};
    bool frame_pending = false;

    cudaStream_t upload_stream = nullptr;
    cudaEvent_t upload_done[2]{}, raster_done[2]{};
    struct RingFrame { // a streamed frame between vb_render_begin and its completion on the host
        bool pending = false, raster_checked = false;
        vb_params params{};
        void *out_host = nullptr;
        uint32_t slot = 0;
        vb_frame_stats stats{};
    } ring[3];
    uint64_t stream_seq = 0;

    // multi-GPU exchange (flatten sharded by tag range; k_exchange.cu)
    struct Exchange {
        bool configured = false, enabled = false;
        uint32_t rank = 0, world = 1, lines_cap = 0, n_paths = 0;
        size_t half_bytes = 0;
        DevBuf arena;
        void *peer[8] = {};
        uint32_t rows[9] = {};
    } xc;
};

// Every device buffer the renderer owns, each once: what vb_renderer_free frees and vb_frame_stats::arena_bytes counts.
template <class F> static void for_each_buf(vb_renderer *r, F f) {
    DevBuf *const all[] = {&r->slot[0].scene, &r->slot[0].ramps, &r->slot[0].atlas, &r->slot[1].scene, &r->slot[1].ramps, &r->slot[1].atlas,
                           &r->mask8, &r->mask16, &r->tag_monoids, &r->path_bboxes, &r->draw_monoids, &r->info_bin_data, &r->clip_inp,
                           &r->clip_bboxes, &r->clip_scratch, &r->draw_bboxes, &r->bin_headers, &r->paths, &r->ctl, &r->tile_start,
                           &r->cls_list, &r->lines, &r->line_scratch, &r->flatten_jobs, &r->flatten_parts, &r->tiles, &r->seg_counts,
                           &r->segments, &r->ptcl, &r->blend_spill, &r->cell_draw, &r->target, &r->target_alt, &r->resolve_tmp,
                           &r->blit_rects, &r->xc.arena};
    for (DevBuf *b : all) f(*b);
}

#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) {                                                                  \
            r->err = std::string(#call) + ": " + cudaGetErrorString(e_);                          \
            return VB_E_CUDA;                                                                     \
        }                                                                                         \
    } while (0)

static int ensure(vb_renderer *r, DevBuf &b, size_t bytes) {
    if (bytes < 256) bytes = 256;
    if (b.cap >= bytes) return VB_OK;
    if (b.p) CK(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = (bytes + 255) & ~(size_t)255;
    CK(cudaMalloc(&b.p, want));
    b.cap = want;
    return VB_OK;
}
// One entry per bump arena: the name vb_debug_limit_arena takes, the buffer, its element size and its VbBump counter.
// The special cases are in arena_offset, arena_need, ensure_arena and the first guesses of prepare.
using RendererBuf = DevBuf vb_renderer::*;
using BumpCounter = uint32_t VbBump::*;
struct ArenaDesc {
    const char *name;
    const char *download; // vb_debug_download's name of the buffer when it differs from the arena's
    RendererBuf buf;
    size_t elem_bytes;
    BumpCounter counter;
};
static const ArenaDesc ARENAS[N_ARENAS] = {
    {"lines", nullptr, &vb_renderer::lines, sizeof(VbLineSoup), &VbBump::lines},
    {"binning", "info_bin_data", &vb_renderer::info_bin_data, 4, &VbBump::binning},
    {"tiles", nullptr, &vb_renderer::tiles, sizeof(VbTile), &VbBump::tile},
    {"seg_counts", nullptr, &vb_renderer::seg_counts, sizeof(VbSegmentCount), &VbBump::seg_counts},
    {"segments", nullptr, &vb_renderer::segments, sizeof(VbSegment), &VbBump::segments},
    {"blend", "blend_spill", &vb_renderer::blend_spill, 4, &VbBump::blend},
    {"ptcl", nullptr, &vb_renderer::ptcl, 4, &VbBump::ptcl},
};
static int arena_index(const char *name) {
    for (int a = 0; a < N_ARENAS; a++)
        if (!strcmp(name, ARENAS[a].name)) return a;
    return -1;
}
// ptcl starts with a static command area of VB_PTCL_INITIAL_ALLOC words per tile; its capacity includes it, bump.ptcl does not
static uint64_t ptcl_static(const VbConfig &c) { return (uint64_t)c.width_in_tiles * c.tile_rows * VB_PTCL_INITIAL_ALLOC; }
// elements of the arena's buffer in front of the arena: binning lives after the draw info in info_bin_data
static size_t arena_offset(const vb_renderer *r, int a) { return a == ARENA_BINNING ? r->cur->layout.bin_data_start : 0; }
// what the last attempt asked of an arena, in the units of its capacity
static uint64_t arena_need(const vb_renderer *r, int a) {
    const uint64_t n = r->cur->h_bump->*ARENAS[a].counter;
    return a == ARENA_PTCL ? ptcl_static(r->cfg) + n : n;
}
// Allocate arena a for its capacity. ptcl gets 512 bytes of slack for fine's 256-byte command windows; the lines capacity
// also sizes flatten's scratch arenas.
static int ensure_arena(vb_renderer *r, int a) {
    const ArenaDesc &d = ARENAS[a];
    int rc = ensure(r, r->*d.buf, (arena_offset(r, a) + r->cap[a]) * d.elem_bytes + (a == ARENA_PTCL ? 512 : 0));
    if (rc || a != ARENA_LINES) return rc;
    size_t lit_bytes, job_bytes;
    vb_flatten_arena_bytes(r->cap[a], &lit_bytes, &job_bytes);
    if ((rc = ensure(r, r->line_scratch, lit_bytes))) return rc;
    return ensure(r, r->flatten_jobs, job_bytes);
}

// Keys of registered textures (vb_register_texture). Each is a fresh address inside one reserved, inaccessible (PROT_NONE)
// range of the process's address space, so no host buffer can have it, even after the texture is unregistered: the host
// resolve recognises such a key by its address alone and never reads through it (vb_texture_key). The range is never
// unmapped and a key is never handed out twice. `owner` is the renderer that registered the key.
static std::mutex g_tex_mutex;
static std::unordered_map<const void *, vb_renderer *> g_tex_owner;
static uint8_t *g_tex_base = nullptr;
static size_t g_tex_next = 0;
static const size_t TEX_KEY_STRIDE = 16, TEX_RANGE_BYTES = (size_t)1 << 30;

extern "C" int vb_texture_key(const void *key) { // for vb_scene.cpp's host resolve
    const uint8_t *p = (const uint8_t *)key, *base = __atomic_load_n(&g_tex_base, __ATOMIC_ACQUIRE);
    return base != nullptr && p >= base && p < base + TEX_RANGE_BYTES;
}
static const void *new_texture_key(vb_renderer *owner) {
    std::lock_guard<std::mutex> lock(g_tex_mutex);
    if (!g_tex_base) {
        void *m = mmap(nullptr, TEX_RANGE_BYTES, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (m == MAP_FAILED) return nullptr;
        __atomic_store_n(&g_tex_base, (uint8_t *)m, __ATOMIC_RELEASE);
    }
    if (g_tex_next + TEX_KEY_STRIDE > TEX_RANGE_BYTES) return nullptr;
    const void *key = g_tex_base + g_tex_next;
    g_tex_next += TEX_KEY_STRIDE;
    g_tex_owner[key] = owner;
    return key;
}
static void drop_registrations(vb_renderer *r) {
    std::lock_guard<std::mutex> lock(g_tex_mutex);
    for (auto it = g_tex_owner.begin(); it != g_tex_owner.end();) it = it->second == r ? g_tex_owner.erase(it) : std::next(it);
}

// mask LUTs: vello_encoding/src/mask.rs:10-98 (f64 maths like the reference)
static uint32_t one_mask(double slope, double translation, bool is_pos, const uint8_t *pattern, int n) {
    if (is_pos) translation = 1. - translation;
    uint32_t result = 0;
    for (int i = 0; i < n; i++) {
        double y = (i + 0.5) * (1.0 / n);
        double x = (pattern[i] + 0.5) * (1.0 / n);
        if (!is_pos) y = 1. - y;
        if ((x - (1.0 - translation)) * (1. - slope) - (y - translation) * slope >= 0.) result |= 1u << i;
    }
    return result;
}
static void make_mask_luts(std::vector<uint32_t> &l8, std::vector<uint32_t> &l16) {
    static const uint8_t P8[8] = {0, 5, 3, 7, 1, 4, 6, 2};
    static const uint8_t P16[16] = {1, 8, 4, 11, 15, 7, 3, 12, 0, 9, 5, 13, 2, 10, 6, 14};
    l8.assign(256, 0);
    l16.assign(2048, 0);
    for (int i = 0; i < 32 * 32; i++) {
        int u = i % 32, v = i / 32;
        l8[i / 4] |= one_mask(((v % 16) + 0.5) * (1.0 / 16), (u + 0.5) * (1.0 / 32), v >= 16, P8, 8) << ((i % 4) * 8);
    }
    for (int i = 0; i < 64 * 64; i++) {
        int u = i % 64, v = i / 64;
        l16[i / 2] |= one_mask(((v % 32) + 0.5) * (1.0 / 32), (u + 0.5) * (1.0 / 64), v >= 32, P16, 16) << ((i % 2) * 16);
    }
}

extern "C" int vb_renderer_new(const vb_options *opt, vb_renderer **out) {
    if (!out) return VB_E_INVALID;
    vb_renderer *r = new vb_renderer();
    r->device = opt ? opt->device : 0;
    r->timing = opt && opt->timing;
    if (opt && opt->max_retries) r->max_retries = opt->max_retries;
    cudaError_t e = cudaSetDevice(r->device);
    if (e != cudaSuccess) {
        fprintf(stderr, "vello_b200: cudaSetDevice(%d): %s\n", r->device, cudaGetErrorString(e));
        delete r;
        return VB_E_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, r->device) == cudaSuccess) r->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&r->upload_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&r->tiling_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&r->tiling_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&r->tiling_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&r->blit_staged, cudaEventDisableTiming) != cudaSuccess) {
        delete r;
        return VB_E_CUDA;
    }
    for (auto &s : r->slot) {
        if (cudaHostAlloc((void **)&s.h_bump, sizeof(VbBump), cudaHostAllocMapped) != cudaSuccess ||
            cudaHostGetDevicePointer((void **)&s.h_bump_dev, s.h_bump, 0) != cudaSuccess) {
            delete r;
            return VB_E_CUDA;
        }
        memset(s.h_bump, 0, sizeof(VbBump));
    }
    for (auto &ev : r->upload_done) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto &ev : r->raster_done) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto &ev : r->ev) cudaEventCreate(&ev);
    for (auto &ev : r->frame_ev) cudaEventCreate(&ev);
    for (auto &ev : r->band_ev) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto &ev : r->copy_done) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (getenv("VELLO_B200_NO_GRAPH")) r->use_graph = false;
    if (cudaStreamCreateWithFlags(&r->copy_stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete r;
        return VB_E_CUDA;
    }
    r->ev_ok = true;
    if (vb_fine_init_constants() != 0) {
        delete r;
        return VB_E_CUDA;
    }
    std::vector<uint32_t> l8, l16;
    make_mask_luts(l8, l16);
    if (ensure(r, r->mask8, l8.size() * 4) || ensure(r, r->mask16, l16.size() * 4)) {
        delete r;
        return VB_E_CUDA;
    }
    cudaMemcpy(r->mask8.p, l8.data(), l8.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(r->mask16.p, l16.data(), l16.size() * 4, cudaMemcpyHostToDevice);
    *out = r;
    return VB_OK;
}

extern "C" void vb_renderer_free(vb_renderer *r) {
    if (!r) return;
    cudaSetDevice(r->device);
    if (r->stream) cudaStreamSynchronize(r->stream);
    for_each_buf(r, [](DevBuf &b) {
        if (b.p) cudaFree(b.p);
    });
    for (auto &s : r->slot)
        if (s.h_bump) cudaFreeHost(s.h_bump);
    if (r->blit_host) cudaFreeHost(r->blit_host);
    if (r->blit_staged) cudaEventDestroy(r->blit_staged);
    drop_registrations(r);
    if (r->ev_ok) {
        for (auto &ev : r->ev) cudaEventDestroy(ev);
        for (auto &ev : r->frame_ev) cudaEventDestroy(ev);
        for (auto &ev : r->band_ev) cudaEventDestroy(ev);
        for (auto &ev : r->copy_done) cudaEventDestroy(ev);
        for (auto &ev : r->upload_done) cudaEventDestroy(ev);
        for (auto &ev : r->raster_done) cudaEventDestroy(ev);
        for (auto &gs : r->graphs)
            if (gs.exec) cudaGraphExecDestroy(gs.exec);
    }
    if (r->tiling_stream) cudaStreamSynchronize(r->tiling_stream);
    if (r->tiling_fork) cudaEventDestroy(r->tiling_fork);
    if (r->tiling_join) cudaEventDestroy(r->tiling_join);
    if (r->tiling_stream) cudaStreamDestroy(r->tiling_stream);
    if (r->copy_stream) cudaStreamDestroy(r->copy_stream);
    if (r->upload_stream) cudaStreamDestroy(r->upload_stream);
    if (r->stream) cudaStreamDestroy(r->stream);
    delete r;
}

extern "C" const char *vb_strerror(int code) {
    switch (code) {
    case VB_OK: return "ok";
    case VB_E_INVALID: return "invalid argument";
    case VB_E_CUDA: return "CUDA error (see vb_last_error)";
    case VB_E_BUMP_OVERFLOW: return "bump arena overflow persisted after grow-and-retry";
    case VB_E_NO_SCENE: return "no scene uploaded";
    case VB_E_UNKNOWN_BUFFER: return "unknown buffer name";
    default: return "unknown error";
    }
}
extern "C" const char *vb_last_error(vb_renderer *r) { return r ? r->err.c_str() : ""; }
extern "C" void *vb_stream(vb_renderer *r) { return r ? (void *)r->stream : nullptr; }
extern "C" void *vb_target(vb_renderer *r, size_t *bytes) {
    if (!r) return nullptr;
    if (bytes) *bytes = r->target.cap;
    return r->target.p;
}
extern "C" int vb_copy_to_host(vb_renderer *r, const void *src_device, void *dst_host, size_t bytes) {
    if (!r || !src_device || !dst_host) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaMemcpyAsync(dst_host, src_device, bytes, cudaMemcpyDeviceToHost, r->stream));
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

static int upload_on(vb_renderer *r, cudaStream_t st, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                     uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h) {
    if (!r || !layout || (scene_len && !scene) || (scene_len & 3)) return VB_E_INVALID;
    if (ramp_h && ramp_w != 512) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    memcpy(&r->cur->layout, layout, sizeof(VbLayout));
    r->cur->scene_words = scene_len / 4;
    int rc;
    if ((rc = ensure(r, r->cur->scene, scene_len + 64))) return rc;
    if (scene_len) CK(cudaMemcpyAsync(r->cur->scene.p, scene, scene_len, cudaMemcpyHostToDevice, st));
    r->cur->n_ramps = ramp_h;
    if ((rc = ensure(r, r->cur->ramps, (size_t)ramp_h * 512 * 4))) return rc;
    if (ramp_h) CK(cudaMemcpyAsync(r->cur->ramps.p, ramps, (size_t)ramp_h * 512 * 4, cudaMemcpyHostToDevice, st));
    r->cur->atlas_w = atlas ? atlas_w : 0;
    r->cur->atlas_h = atlas ? atlas_h : 0;
    if ((rc = ensure(r, r->cur->atlas, (size_t)r->cur->atlas_w * r->cur->atlas_h * 4))) return rc;
    if (r->cur->atlas_w && r->cur->atlas_h)
        CK(cudaMemcpyAsync(r->cur->atlas.p, atlas, (size_t)r->cur->atlas_w * r->cur->atlas_h * 4, cudaMemcpyHostToDevice, st));
    r->cur->overridden.clear(); // a caller-packed atlas: overrides do not apply
    r->cur->have_scene = true;
    r->cells.clear(); // a new scene is one cell until vb_set_cells says otherwise
    return VB_OK;
}

extern "C" int vb_readback_wait(vb_renderer *r);
// A non-streaming entry point used while streamed frames are still in flight completes them first.
static int drain_stream(vb_renderer *r) {
    if (r->stream_pending) return vb_readback_wait(r);
    return VB_OK;
}

extern "C" int vb_scene_upload(vb_renderer *r, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                               uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h) {
    if (!r) return VB_E_INVALID;
    int rc = drain_stream(r);
    if (rc) return rc;
    return upload_on(r, r->stream, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h);
}

static uint32_t grow(uint32_t need) {
    uint64_t g = (uint64_t)need + need / 4 + 1024;
    return g > 0xfffffff0ull ? 0xfffffff0u : (uint32_t)g;
}

// Compute the config for these params, size the fixed buffers, and (first time / after growth) the arenas.
static int prepare(vb_renderer *r, const vb_params *p) {
    // RenderParams sanity (the reference panics / produces nothing on these; here they are argument errors)
    if (p->width == 0u || p->height == 0u || p->aa > 2u || p->width > 65536u || p->height > 65536u) {
        r->err = "vb_params: width/height must be 1..65536 and aa 0..2";
        return VB_E_INVALID;
    }
    const uint32_t n_cells = r->cells.empty() ? 1u : (uint32_t)r->cells.size() - 1u;
    if (n_cells > 1u) {
        if (p->bin_row1 > p->bin_row0 || p->tile_row1 > p->tile_row0 || r->xc.enabled || r->grouped) {
            r->err = "batch: cells cannot be combined with bin_row / tile_row windows, vb_group or the exchange";
            return VB_E_INVALID;
        }
        const uint64_t hb = ((p->height + 15u) / 16u + 15u) / 16u, wb = ((p->width + 15u) / 16u + 15u) / 16u;
        const uint64_t parts = (r->cur->layout.n_draw_objects + 255u) / 256u, bins = ((wb * hb * n_cells + 255u) & ~255ull);
        if (hb * n_cells * 2u > 65535u || parts * bins >= 0xffffffffull) {
            r->err = "batch: too many cells of this size (bin rows or bin headers exceed what the kernels index)";
            return VB_E_INVALID;
        }
    }
    {
        const uint64_t nt = (uint64_t)((p->width + 15u) / 16u) * ((p->height + 15u) / 16u) * n_cells;
        if (nt * VB_PTCL_INITIAL_ALLOC + nt * (VB_PTCL_INCREMENT / 8u) + 65536u > 0xf0000000ull) {
            r->err = n_cells > 1u ? "batch: tile count * PTCL allocation exceeds 32-bit word offsets"
                                  : "vb_params: tile count * PTCL allocation exceeds 32-bit word offsets";
            return VB_E_INVALID;
        }
    }
    VbConfig &c = r->cfg;
    memset(&c, 0, sizeof c);
    c.width_in_tiles = (p->width + 15u) / 16u;
    c.height_in_tiles = (p->height + 15u) / 16u;
    c.target_width = p->width;
    c.target_height = p->height;
    c.base_color = p->base_color;
    c.layout = r->cur->layout;
    const uint32_t hb = (c.height_in_tiles + 15u) / 16u, wb = (c.width_in_tiles + 15u) / 16u;
    c.win_by0 = 0;
    c.win_by1 = hb;
    if (p->bin_row1 > p->bin_row0) {
        c.win_by0 = p->bin_row0 < hb ? p->bin_row0 : hb;
        c.win_by1 = p->bin_row1 < hb ? p->bin_row1 : hb;
    }
    c.win_ty0 = c.win_by0 * 16u;
    c.win_ty1 = c.win_by1 * 16u < c.height_in_tiles ? c.win_by1 * 16u : c.height_in_tiles;
    if (p->tile_row1 > p->tile_row0) {
        // stripe in tile rows: binning / coarse cover the bins that contain it, tile_alloc clamps every path to its rows
        // (so the extra tiles of a partly covered bin row hold empty command lists), fine paints exactly the stripe
        c.win_ty0 = p->tile_row0 < c.height_in_tiles ? p->tile_row0 : c.height_in_tiles;
        c.win_ty1 = p->tile_row1 < c.height_in_tiles ? p->tile_row1 : c.height_in_tiles;
        c.win_by0 = c.win_ty0 / 16u;
        c.win_by1 = (c.win_ty1 + 15u) / 16u;
    }
    c.win_cull = (c.win_ty0 > 0u || c.win_ty1 < c.height_in_tiles) ? 1u : 0u;
    c.n_tag_words = r->cur->layout.path_data_base - r->cur->layout.path_tag_base;
    c.scene_words = (uint32_t)r->cur->scene_words;
    c.n_ramps = r->cur->n_ramps;
    c.atlas_w = r->cur->atlas_w;
    c.atlas_h = r->cur->atlas_h;
    c.out_pitch_px = p->width;
    c.out_row0 = c.win_ty0 * 16u;
    c.n_cells = n_cells;
    c.tile_rows = c.height_in_tiles * n_cells;
    c.cell_draw = n_cells > 1u ? (const uint32_t *)r->cell_draw.p : nullptr;
    r->params = *p;

    const VbLayout &L = r->cur->layout;
    const uint32_t n_draw = L.n_draw_objects, n_paths = L.n_paths, n_clips = L.n_clips;
    const uint32_t n_tiles = c.width_in_tiles * c.tile_rows;
    const uint32_t n_bins = wb * hb * n_cells, aligned_n_bins = (n_bins + 255u) & ~255u;
    int rc;
    if ((rc = ensure(r, r->tag_monoids, (size_t)c.n_tag_words * sizeof(VbTagMonoid)))) return rc;
    if ((rc = ensure(r, r->path_bboxes, (size_t)n_paths * sizeof(VbPathBbox)))) return rc;
    if ((rc = ensure(r, r->draw_monoids, (size_t)n_draw * sizeof(VbDrawMonoid)))) return rc;
    if ((rc = ensure(r, r->clip_inp, (size_t)n_clips * sizeof(VbClipInp)))) return rc;
    if ((rc = ensure(r, r->clip_bboxes, (size_t)n_clips * sizeof(VbBbox4)))) return rc;
    if ((rc = ensure(r, r->clip_scratch, vb_clip_scratch_words(n_clips) * 4))) return rc;
    if ((rc = ensure(r, r->draw_bboxes, (size_t)n_draw * sizeof(VbBbox4)))) return rc;
    if ((rc = ensure(r, r->bin_headers, (size_t)((n_draw + 255u) / 256u) * aligned_n_bins * sizeof(VbBinHeader)))) return rc;
    if ((rc = ensure(r, r->paths, (size_t)((n_draw + 255u) & ~255u) * sizeof(VbPath)))) return rc;
    if ((rc = ensure(r, r->tile_start, ((size_t)n_tiles + 256) * 4))) return rc;
    if ((rc = ensure(r, r->cls_list, (size_t)VB_FINE_CLASSES * n_tiles * 8))) return rc; // fine's cost-ordered tile lists

    // arena capacities (elements) start at a first guess and only ever grow; seg_counts and segments follow the capacities
    // before them. A test-only limit lowers the capacity the kernels see, never the allocation (vb_debug_limit_arena).
    const uint64_t guess[N_ARENAS] = {(uint64_t)(c.n_tag_words * 4u) * 2 + 4096, (uint64_t)n_draw * 4 + 4096, (uint64_t)n_draw * 16 + 4096,
                                      0, 0, 256, ptcl_static(c) + (uint64_t)VB_PTCL_INCREMENT * (64 + n_tiles / 8)};
    uint32_t *size = &c.lines_size;
    for (int a = 0; a < N_ARENAS; a++) {
        const uint64_t g = a == ARENA_SEG_COUNTS ? (uint64_t)r->cap[ARENA_LINES] * 2 : a == ARENA_SEGMENTS ? r->cap[ARENA_SEG_COUNTS] : guess[a];
        r->cap[a] = (uint32_t)std::max<uint64_t>(r->cap[a], std::min<uint64_t>(g, 0xfffffff0ull));
        if ((rc = ensure_arena(r, a))) return rc;
        size[a] = std::min(r->cap[a], r->limit[a]);
    }

    // control block: [bump (8 words, padded to 16), header words] [look-back states]
    VbFrameBufs &b = r->bufs;
    memset(&b, 0, sizeof b);
    b.parts_pathtag = vb_pathtag_parts(c.n_tag_words);
    b.parts_flatten = vb_flatten_parts(c.n_tag_words);
    b.parts_draw = vb_draw_parts(n_draw);
    b.parts_tile = vb_tile_alloc_parts(n_draw);
    b.parts_backdrop = vb_backdrop_parts(c.tiles_size); // follows the tile arena: set above, regrown on retry
    size_t off = VB_CTL_HEADER_WORDS;
    const size_t o_pathtag = off; off += vb_lookback_words(b.parts_pathtag, 5);
    const size_t o_flatten = off; // flatten: [0] literal-record counter, [1] job counter, [2] work-list length, [4..] look-back state of its partition scan
    off += 4 + vb_lookback_words((b.parts_flatten + 8191u) / 8192u, 1);
    const size_t o_draw = off; off += vb_lookback_words(b.parts_draw, 4);
    const size_t o_tile = off; off += vb_lookback_words(b.parts_tile, 1);
    const size_t o_clip = off; off += vb_lookback_words(vb_clip_parts(n_clips), 1);
    const size_t o_backdrop = off; off += vb_lookback_words(b.parts_backdrop, 3);
    b.ctl_words = off;
    if ((rc = ensure(r, r->ctl, off * 4))) return rc;
    if ((rc = ensure(r, r->flatten_parts, vb_flatten_part_words(b.parts_flatten) * 4))) return rc;

    // every buffer has its size: the launchers' view of them
    b.scene = (const uint32_t *)r->cur->scene.p;
    b.ramps = (const uint32_t *)r->cur->ramps.p;
    b.atlas = (const uint8_t *)r->cur->atlas.p;
    b.mask8 = (const uint32_t *)r->mask8.p;
    b.mask16 = (const uint32_t *)r->mask16.p;
    b.tag_monoids = (VbTagMonoid *)r->tag_monoids.p;
    b.path_bboxes = (VbPathBbox *)r->path_bboxes.p;
    b.draw_monoids = (VbDrawMonoid *)r->draw_monoids.p;
    b.info_bin_data = (uint32_t *)r->info_bin_data.p;
    b.clip_inp = (VbClipInp *)r->clip_inp.p;
    b.clip_bboxes = (VbBbox4 *)r->clip_bboxes.p;
    b.clip_scratch = (int32_t *)r->clip_scratch.p;
    b.draw_bboxes = (VbBbox4 *)r->draw_bboxes.p;
    b.bin_headers = (VbBinHeader *)r->bin_headers.p;
    b.paths = (VbPath *)r->paths.p;
    b.tile_start = (uint32_t *)r->tile_start.p;
    b.cls_list = (uint2 *)r->cls_list.p;
    b.lines = (VbLineSoup *)r->lines.p;
    b.line_scratch = (FlLit *)r->line_scratch.p;
    b.flatten_jobs = (FlJob *)r->flatten_jobs.p;
    b.flatten_parts = (uint32_t *)r->flatten_parts.p;
    b.tiles = (VbTile *)r->tiles.p;
    b.seg_counts = (VbSegmentCount *)r->seg_counts.p;
    b.segments = (VbSegment *)r->segments.p;
    b.ptcl = (uint32_t *)r->ptcl.p;
    b.blend_spill = (uint32_t *)r->blend_spill.p;
    b.ctl = (uint32_t *)r->ctl.p;
    b.lb_pathtag = b.ctl + o_pathtag;
    b.lb_flatten = b.ctl + o_flatten;
    b.lb_draw = b.ctl + o_draw;
    b.lb_tile = b.ctl + o_tile;
    b.lb_clip = b.ctl + o_clip;
    b.lb_backdrop = b.ctl + o_backdrop;
    b.sm_count = r->sm_count;
    return VB_OK;
}

static void xpeers_of(const vb_renderer *r, XPeers *X) {
    memset(X, 0, sizeof *X);
    for (uint32_t i = 0; i < r->xc.world; i++) X->base[i] = (unsigned char *)r->xc.peer[i];
    for (uint32_t i = 0; i <= r->xc.world; i++) X->rows[i] = r->xc.rows[i];
    X->world = r->xc.world; X->rank = r->xc.rank; X->n_paths = r->xc.n_paths; X->lines_cap = r->xc.lines_cap; X->half_bytes = r->xc.half_bytes;
}

static void rec(vb_renderer *r, int i) {
    if (r->timing) cudaEventRecord(r->ev[i], r->stream);
}

// The rows fine paints: the window's tile rows, launched in `bands` row bands when the pixels also go to the host (up to 8,
// for at least 64 rows), so that the read-back of band k overlaps the rasterisation of band k+1. A batch paints every tile
// row of its tall frame in one launch: its cells are not rows of one image, and its pixel rows are n_cells * height.
struct FineRows {
    uint32_t ty0, ty1, bands; // tile rows [ty0, ty1) in `bands` launches
    size_t y1;                // the last pixel row they cover (+1); rows from ty0 * 16
    size_t dest_rows;         // pixel rows the destination holds, from row out_row0
    // tile rows [*by0, *by1) of band b; false once the bands have run out of rows
    bool band(uint32_t b, uint32_t *by0, uint32_t *by1) const {
        const uint32_t n = (ty1 - ty0 + bands - 1u) / bands;
        *by0 = ty0 + b * n;
        *by1 = *by0 + n < ty1 ? *by0 + n : ty1;
        return *by0 < *by1;
    }
};
static FineRows fine_rows(const VbConfig &c, const Dest &d) {
    const bool batch = c.n_cells > 1u;
    FineRows f;
    f.ty0 = batch ? 0u : c.win_ty0;
    f.ty1 = batch ? c.tile_rows : c.win_ty1;
    const uint32_t rows = f.ty1 - f.ty0;
    f.bands = d.host && rows >= 64u && !batch ? d.bands : 1u;
    f.y1 = std::min((size_t)f.ty1 * 16u, (size_t)c.n_cells * c.target_height);
    f.dest_rows = batch ? (size_t)c.n_cells * c.target_height : (size_t)rows * 16u;
    return f;
}

// Queue the copy of band `band`'s pixel rows to d.host on the copy stream, behind everything on the renderer's stream.
static int queue_readback(vb_renderer *r, const VbConfig &c, const FineRows &f, uint32_t band, const Dest &d) {
    uint32_t ty0, ty1;
    f.band(band, &ty0, &ty1);
    const size_t y0 = (size_t)ty0 * 16u, y1 = std::min((size_t)ty1 * 16u, f.y1);
    if (y1 <= y0) return VB_OK;
    const size_t off = (y0 - c.out_row0) * c.out_pitch_px * 4u, bytes = (y1 - y0) * c.out_pitch_px * 4u;
    CK(cudaEventRecord(r->band_ev[band], r->stream));
    CK(cudaStreamWaitEvent(r->copy_stream, r->band_ev[band], 0));
    CK(cudaMemcpyAsync((char *)d.host + off, (const char *)d.dev + off, bytes, cudaMemcpyDeviceToHost, r->copy_stream));
    return VB_OK;
}

// Enqueue stages first..last into d.dev (and d.host). Does not synchronise. `clear_queues` (vb_run_stages): a range that
// starts after stage 0 does not zero the control block, but fine's tile queues must start at 0 and coarse must append to
// empty class lists.
static int enqueue_direct(vb_renderer *r, int first, int last, const Dest &d, bool clear_queues) {
    const VbConfig &c = r->cfg;
    const VbFrameBufs &b = r->bufs;
    cudaStream_t st = r->stream;
    uint32_t launches = 0;
    int rc;
    XPeers X; // multi-GPU exchange
    if (r->xc.enabled) xpeers_of(r, &X);
    if (first == 0) {
        // a kernel, not cudaMemsetAsync: small memsets / copies are served by a copy engine and would queue behind a
        // 64 MiB read-back still draining from the previous frame
        const unsigned ctl_blocks = (unsigned)((b.ctl_words + 1023) / 1024), bb_blocks = (c.layout.n_paths + 255u) / 256u;
        uint32_t *xepoch = r->xc.enabled ? (uint32_t *)r->xc.arena.p + vb_exchange_epoch_word() : nullptr;
        k_frame_init<<<ctl_blocks + bb_blocks, 256, 0, st>>>(b.ctl, (uint32_t)b.ctl_words, ctl_blocks, b.path_bboxes, c.layout.n_paths, xepoch);
        launches++;
    }
    else if (clear_queues) {
        if (last >= VB_STAGE_ID_FINE) CK(cudaMemsetAsync(b.ctl + VB_CTL_FINE_QUEUE, 0, 8 * sizeof(uint32_t), st));
        if (first <= VB_STAGE_ID_COARSE && last >= VB_STAGE_ID_COARSE)
            CK(cudaMemsetAsync(b.ctl + VB_CTL_FINE_CLASS, 0, VB_FINE_CLASSES * sizeof(uint32_t), st));
        if (first <= VB_STAGE_ID_BACKDROP && last >= VB_STAGE_ID_BACKDROP)
            CK(cudaMemsetAsync(b.lb_backdrop, 0, VB_LB_ZERO_WORDS(b.parts_backdrop) * sizeof(uint32_t), st));
    }
    // path_tiling and coarse both depend on backdrop only (it assigns the segment slices): path_tiling is forked onto the
    // tiling stream and joined again before the next stage, so the two kernels share the GPU. Launch counts are unchanged;
    // with per-stage timing on, the stages stay serial so that each one's events time it alone.
    const bool fork_tiling = !r->timing && first <= VB_STAGE_ID_COARSE && last >= VB_STAGE_ID_PATH_TILING;
    rec(r, 0);
    for (int s = first; s <= last; s++) {
        switch (s) {
        case VB_STAGE_ID_PATHTAG: launches += vb_launch_pathtag(c, b, st); break;
        case VB_STAGE_ID_FLATTEN: {
            // with the exchange on, this GPU flattens its share of the tag stream (no stripe culling: the lines are for
            // everybody), then the lines and path boxes are exchanged through peer memory (k_exchange.cu)
            VbConfig cf = c;
            uint32_t p0 = 0u, p1 = b.parts_flatten;
            if (r->xc.enabled) {
                cf.win_cull = 0u;
                const uint32_t P = b.parts_flatten, G = r->xc.world, k = r->xc.rank;
                p0 = (uint32_t)((uint64_t)P * k / G) & ~7u;
                p1 = k + 1u == G ? P : ((uint32_t)((uint64_t)P * (k + 1u) / G) & ~7u);
            }
            launches += vb_launch_flatten(cf, b, first != 0, p0, p1, st);
            if (r->xc.enabled) launches += vb_launch_exchange_send(c, b, X, st);
            break;
        }
        case VB_STAGE_ID_DRAW:
            if (r->xc.enabled) // second half of the exchange: my lines and the complete path boxes arrive before draw_leaf reads them
                launches += vb_launch_exchange_recv(c, b, X, st);
            launches += vb_launch_draw(c, b, st);
            break;
        case VB_STAGE_ID_CLIP: launches += vb_launch_clip(c, b, st); break;
        case VB_STAGE_ID_BINNING: launches += vb_launch_binning(c, b, st); break;
        case VB_STAGE_ID_TILE_ALLOC: launches += vb_launch_tile_alloc(c, b, st); break;
        case VB_STAGE_ID_PATH_COUNT: launches += vb_launch_path_count(c, b, st); break;
        case VB_STAGE_ID_BACKDROP: launches += vb_launch_backdrop(c, b, st); break;
        case VB_STAGE_ID_COARSE:
            // coarse is enqueued first, so that its CTAs (one per bin quadrant, all resident at once) are placed before
            // path_tiling's grid fills the rest of the GPU
            if (fork_tiling) CK(cudaEventRecord(r->tiling_fork, st));
            launches += vb_launch_coarse(c, b, st);
            if (fork_tiling) {
                CK(cudaStreamWaitEvent(r->tiling_stream, r->tiling_fork, 0));
                launches += vb_launch_path_tiling(c, b, r->tiling_stream);
                CK(cudaEventRecord(r->tiling_join, r->tiling_stream));
                CK(cudaStreamWaitEvent(st, r->tiling_join, 0));
            }
            break;
        case VB_STAGE_ID_PATH_TILING:
            if (!fork_tiling) launches += vb_launch_path_tiling(c, b, st); // else launched beside coarse
            break;
        case VB_STAGE_ID_FINE: {
            // with a host destination, each band's device->host copy is queued on the copy stream behind an event (only
            // the last band's copy is exposed)
            const FineRows f = fine_rows(c, d);
            for (uint32_t band = 0; band < f.bands; band++) {
                VbConfig cb = c;
                if (!f.band(band, &cb.win_ty0, &cb.win_ty1)) break;
                launches += vb_launch_fine(cb, b, (uint32_t *)d.dev, (int)r->params.aa, r->occlusion_cull, band, f.bands == 1u, st);
                if (d.host && (rc = queue_readback(r, c, f, band, d))) return rc;
            }
            break;
        }
        default: return VB_E_INVALID;
        }
        rec(r, s + 1);
    }
    k_publish_bump<<<1, 32, 0, st>>>(b.bump(), r->cur->h_bump_dev); // zero-copy store to mapped host memory (no copy engine)
    launches++;
    CK(cudaGetLastError());
    r->launches = launches;
    return VB_OK;
}

// ---- whole-frame CUDA graphs ---------------------------------------------------------------------------------------------
// A frame is ~20 kernel launches. Each launch makes the GPU fetch a command buffer from host memory over PCIe; while a
// 64 MiB read-back of the previous frame is streaming the other way that fetch queues behind it (tools/e2e_probe.py
// shows every stage of a streamed frame starting late). In steady state
// the launches of a frame are identical -- same kernels, grids, arena pointers, config -- so they are captured once into a
// graph and replayed with ONE submission. The key is the inputs of the launches; growing an arena or changing the scene
// layout / frame size / window simply misses the cache and re-captures.
static void graph_key(vb_renderer *r, int last, const void *out_dev, GraphKey *k) {
    memset(k, 0, sizeof *k);
    k->cfg = r->cfg;
    memcpy(&k->bufs, &r->bufs, sizeof k->bufs);
    k->out = out_dev;
    k->h_bump_dev = r->cur->h_bump_dev;
    k->aa = r->params.aa;
    k->cull = r->occlusion_cull;
    k->last = (uint32_t)last;
    if (r->xc.enabled) {
        k->xarena = r->xc.arena.p;
        xpeers_of(r, &k->xpeers);
    }
}

// Enqueue stages first..last: through a cached graph for whole frames, directly otherwise.
static int enqueue(vb_renderer *r, int first, int last, const Dest &d, bool clear_queues) {
    if (!r->use_graph || r->timing || first != 0 || last != VB_N_STAGE_IDS - 1) return enqueue_direct(r, first, last, d, clear_queues);
    // with a host destination split into bands, fine and its interleaved copies stay outside the graph
    const FineRows f = fine_rows(r->cfg, d);
    const bool banded = f.bands > 1u;
    const int g_last = banded ? VB_STAGE_ID_FINE - 1 : last;
    GraphKey key;
    graph_key(r, g_last, d.dev, &key);
    GraphSlot *slot = nullptr;
    for (GraphSlot &gs : r->graphs)
        if (gs.exec && memcmp(&gs.key, &key, sizeof key) == 0) slot = &gs;
    // Any refusal along the way (a tool or driver that does not allow capture here) turns graph replay off for this renderer
    // and the frame is launched kernel by kernel: graphs are an optimisation, never a requirement.
    auto direct = [&]() {
        cudaGetLastError();
        r->use_graph = false;
        return enqueue_direct(r, first, last, d, clear_queues);
    };
    if (!slot) {
        slot = &r->graphs[r->graph_next++ % (sizeof r->graphs / sizeof r->graphs[0])];
        if (slot->exec) {
            cudaGraphExecDestroy(slot->exec);
            slot->exec = nullptr;
        }
        if (cudaStreamBeginCapture(r->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) return direct();
        Dest captured = d;
        captured.host = nullptr; // the captured fine is one launch; its read-back is queued after the graph, below
        const int rc = enqueue_direct(r, 0, g_last, captured, false);
        cudaGraph_t g = nullptr;
        const cudaError_t e = cudaStreamEndCapture(r->stream, &g);
        if (rc != VB_OK || e != cudaSuccess || !g) {
            if (g) cudaGraphDestroy(g);
            return direct();
        }
        const cudaError_t ei = cudaGraphInstantiate(&slot->exec, g, 0);
        cudaGraphDestroy(g);
        if (ei != cudaSuccess) {
            slot->exec = nullptr;
            return direct();
        }
        memcpy(&slot->key, &key, sizeof key); // with its (zeroed) padding: keys are compared bytewise
        slot->launches = r->launches;
    }
    if (cudaGraphLaunch(slot->exec, r->stream) != cudaSuccess) {
        cudaGraphExecDestroy(slot->exec);
        slot->exec = nullptr;
        return direct();
    }
    r->launches = slot->launches;
    if (banded) {
        const int rc = enqueue_direct(r, VB_STAGE_ID_FINE, VB_STAGE_ID_FINE, d, false);
        r->launches += slot->launches;
        return rc;
    }
    if (d.host) return queue_readback(r, r->cfg, f, 0, d);
    return VB_OK;
}

// The frame's device destination: the given pointer, or the renderer's own target (allocated for this frame's window).
static int pick_out(vb_renderer *r, Dest *d) {
    if (d->dev) return VB_OK;
    const VbConfig &c = r->cfg;
    DevBuf &t = d->alt ? r->target_alt : r->target;
    int rc = ensure(r, t, (size_t)c.out_pitch_px * 4u * fine_rows(c, *d).dest_rows);
    d->dev = t.p;
    return rc;
}

// ---- images from device memory: Renderer::override_image / register_texture (vello/src/lib.rs:536-603) ----------------------
// An override names an image by its key (the `pixels` pointer of its vb_image / vb_image_patch). The device resolve
// (vb_scene_upload_streams) copies such an image into its atlas slot from the override's device memory with k_atlas_blit and
// records the slot; marking the image dirty later queues the same copy in front of the next frame (refresh_overrides).

// A device image must be memory of this renderer's device (or managed memory), with 4-byte aligned rows of at least 4 * w bytes.
static int check_device_pixels(vb_renderer *r, const void *px, uint32_t w, uint32_t h, size_t pitch) {
    auto bad = [&](const char *why) {
        r->err = std::string("device image: ") + why;
        return VB_E_INVALID;
    };
    if (!w || !h) return bad("a dimension is 0");
    if (((uintptr_t)px & 3u) || (pitch & 3u)) return bad("the pointer and the row pitch must be multiples of 4 bytes");
    if (pitch < (size_t)w * 4u) return bad("the row pitch is less than 4 * width");
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, px) != cudaSuccess) {
        cudaGetLastError();
        return bad("not a CUDA pointer");
    }
    if (a.type == cudaMemoryTypeManaged) return VB_OK;
    if (a.type != cudaMemoryTypeDevice || a.device != r->device) return bad("not device memory of the renderer's device");
    return VB_OK;
}

// Copy `rects` into an atlas of atlas_w texels per row with one k_atlas_blit on the renderer's stream. The rectangles reach
// the device through a pinned staging buffer, which is rewritten only once the previous copy out of it has run.
static int enqueue_blits(vb_renderer *r, std::vector<VbBlitRect> &rects, void *atlas, uint32_t atlas_w) {
    if (rects.empty()) return VB_OK;
    uint64_t units = 0;
    for (VbBlitRect &b : rects) {
        b.spr = vb_atlas_blit_units_per_row(b.w);
        b.unit0 = units;
        units += (uint64_t)b.h * b.spr;
    }
    const size_t bytes = rects.size() * sizeof(VbBlitRect);
    CK(cudaEventSynchronize(r->blit_staged));
    if (r->blit_host_cap < rects.size()) {
        if (r->blit_host) CK(cudaFreeHost(r->blit_host));
        r->blit_host = nullptr;
        r->blit_host_cap = 0;
        CK(cudaMallocHost((void **)&r->blit_host, bytes));
        r->blit_host_cap = rects.size();
    }
    memcpy(r->blit_host, rects.data(), bytes);
    int rc = ensure(r, r->blit_rects, bytes);
    if (rc) return rc;
    CK(cudaMemcpyAsync(r->blit_rects.p, r->blit_host, bytes, cudaMemcpyHostToDevice, r->stream));
    CK(cudaEventRecord(r->blit_staged, r->stream));
    vb_launch_atlas_blit((const VbBlitRect *)r->blit_rects.p, (uint32_t)rects.size(), units, (uint8_t *)atlas, atlas_w, r->stream);
    CK(cudaGetLastError());
    return VB_OK;
}

// Before a frame: copy the dirty overridden images of the current scene slot into their atlas places. The copy runs ahead of
// every kernel of the frame (and outside any captured graph), so a frame that draws its own destination reads the old pixels.
// The atlas does not move, so a captured frame stays valid. Nothing dirty: nothing is enqueued.
static int refresh_overrides(vb_renderer *r) {
    std::vector<VbBlitRect> rects;
    for (const auto &o : r->cur->overridden)
        if (o.dirty) rects.push_back(VbBlitRect{o.src, o.pitch, 0, o.w, o.h, o.x, o.y, 0, 0});
    if (rects.empty()) return VB_OK;
    const int rc = enqueue_blits(r, rects, r->cur->atlas.p, r->cur->atlas_w);
    if (rc) return rc;
    for (auto &o : r->cur->overridden) o.dirty = false;
    return VB_OK;
}

extern "C" int vb_override_image(vb_renderer *r, const void *key, uint32_t width, uint32_t height, const void *device_pixels,
                                 size_t row_pitch_bytes) {
    if (!r) return VB_E_INVALID;
    if (!key) {
        r->err = "vb_override_image: NULL key";
        return VB_E_INVALID;
    }
    if (device_pixels) {
        CK(cudaSetDevice(r->device));
        const int rc = check_device_pixels(r, device_pixels, width, height, row_pitch_bytes);
        if (rc) return rc;
        r->overrides[key] = vb_renderer::Override{(const uint8_t *)device_pixels, row_pitch_bytes, width, height};
    } else {
        r->overrides.erase(key);
    }
    // recorded atlas places: a new source of the same size is copied before the next frame; a removed override (or one of
    // another size) keeps the pixels copied last and takes effect at the next device resolve
    for (auto &s : r->slot) {
        auto &v = s.overridden;
        v.erase(std::remove_if(v.begin(), v.end(),
                               [&](const auto &o) { return o.key == key && (!device_pixels || o.w != width || o.h != height); }),
                v.end());
        for (auto &o : v)
            if (o.key == key) {
                o.src = (const uint8_t *)device_pixels;
                o.pitch = row_pitch_bytes;
                o.dirty = true;
            }
    }
    return VB_OK;
}

extern "C" int vb_mark_override_image_dirty(vb_renderer *r, const void *key) {
    if (!r) return VB_E_INVALID;
    if (!r->overrides.count(key)) {
        r->err = "vb_mark_override_image_dirty: no override for this key";
        return VB_E_INVALID;
    }
    for (auto &s : r->slot)
        for (auto &o : s.overridden)
            if (o.key == key) o.dirty = true;
    return VB_OK;
}

// Renderer::register_texture / unregister_texture; vb_register_texture / vb_unregister_texture (vb_scene.cpp, which owns vb_image)
// wrap these two.
extern "C" int vb_texture_register(vb_renderer *r, const void *device_pixels, uint32_t width, uint32_t height, size_t row_pitch_bytes,
                                   const void **key_out) {
    if (!r || !key_out) return VB_E_INVALID;
    if (!device_pixels) {
        r->err = "vb_register_texture: NULL pixels";
        return VB_E_INVALID;
    }
    CK(cudaSetDevice(r->device));
    int rc = check_device_pixels(r, device_pixels, width, height, row_pitch_bytes);
    if (rc) return rc;
    const void *key = new_texture_key(r);
    if (!key) {
        r->err = "vb_register_texture: no texture key left";
        return VB_E_INVALID;
    }
    if ((rc = vb_override_image(r, key, width, height, device_pixels, row_pitch_bytes))) return rc;
    *key_out = key;
    return VB_OK;
}

extern "C" int vb_texture_unregister(vb_renderer *r, const void *key) {
    if (!r) return VB_E_INVALID;
    {
        std::lock_guard<std::mutex> lock(g_tex_mutex);
        auto it = vb_texture_key(key) ? g_tex_owner.find(key) : g_tex_owner.end();
        if (it == g_tex_owner.end() || it->second != r) {
            r->err = "vb_unregister_texture: not a texture registered on this renderer";
            return VB_E_INVALID;
        }
        g_tex_owner.erase(it);
    }
    return vb_override_image(r, key, 0, 0, nullptr, 0);
}

// A frame is enqueued in two steps: everything that may allocate, free or otherwise synchronise with the device (config,
// arenas, the output target), then the launches. vb_group runs step 1 for ALL its renderers before step 2 of any: with the
// exchange on, a renderer's frame contains a kernel that waits for its peers, and a peer that shares the device (tests)
// must not be stuck in a cudaFree behind that kernel.
static int frame_prepare(vb_renderer *r, const vb_params *p, const Dest &d) {
    if (!r || !p) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    CK(cudaSetDevice(r->device));
    int rc = prepare(r, p);
    if (rc) return rc;
    r->dest = d;
    return pick_out(r, &r->dest);
}
static int frame_launch(vb_renderer *r) {
    CK(cudaSetDevice(r->device));
    int rc = refresh_overrides(r);
    if (rc) return rc;
    CK(cudaEventRecord(r->frame_ev[0], r->stream));
    rc = enqueue(r, 0, VB_N_STAGE_IDS - 1, r->dest, false);
    if (rc == VB_OK) CK(cudaEventRecord(r->frame_ev[1], r->stream));
    r->frame_timed = rc == VB_OK;
    r->frame_pending = rc == VB_OK;
    return rc;
}

// The same frame in two submissions (plain launches): up to and including flatten + the sending half of the exchange, then
// the rest. Used by vb_group when renderers share a device, see k_exchange.cu.
static int frame_launch_half(vb_renderer *r, int half) {
    CK(cudaSetDevice(r->device));
    if (half == 0) {
        CK(cudaEventRecord(r->frame_ev[0], r->stream));
        return enqueue_direct(r, 0, VB_STAGE_ID_FLATTEN, r->dest, false);
    }
    uint32_t first_half = r->launches;
    int rc = enqueue_direct(r, VB_STAGE_ID_DRAW, VB_N_STAGE_IDS - 1, r->dest, false);
    r->launches += first_half;
    // (with a host destination enqueue_direct queues the read-back behind fine itself)
    if (rc == VB_OK) CK(cudaEventRecord(r->frame_ev[1], r->stream));
    r->frame_timed = rc == VB_OK;
    r->frame_pending = rc == VB_OK;
    return rc;
}

static int render_enqueue(vb_renderer *r, const vb_params *p, const Dest &d) {
    int rc = frame_prepare(r, p, d);
    if (rc) return rc;
    return frame_launch(r);
}
extern "C" int vb_render_enqueue(vb_renderer *r, const vb_params *p, void *out_device) {
    return render_enqueue(r, p, Dest{out_device});
}

static void fill_stats(vb_renderer *r, vb_frame_stats *s) {
    if (!s) return;
    memset(s, 0, sizeof *s);
    memcpy(s, r->cur->h_bump, sizeof(VbBump));
    s->retries = r->retries;
    s->kernel_launches = r->launches;
    for_each_buf(r, [&](DevBuf &b) { s->arena_bytes += b.cap; });
    if (r->timing) {
        for (int i = 0; i < VB_N_STAGE_IDS; i++) cudaEventElapsedTime(&s->stage_ms[i], r->ev[i], r->ev[i + 1]);
        cudaEventElapsedTime(&s->total_ms, r->ev[0], r->ev[VB_N_STAGE_IDS]);
    }
}

// After a failed attempt: enlarge whatever overflowed, using the counters the kernels kept counting.
static void grow_arenas(vb_renderer *r) {
    for (int a = 0; a < N_ARENAS; a++) {
        const uint64_t need = arena_need(r, a);
        // a test-only limit lasts for one overflow of its arena: the re-run sees the real capacity
        if (need > r->limit[a]) r->limit[a] = UINT32_MAX;
        const uint64_t want = need + (a == ARENA_PTCL ? VB_PTCL_INCREMENT : 0u);
        if (want > r->cap[a]) r->cap[a] = grow((uint32_t)std::min<uint64_t>(want, 0xf0000000ull));
    }
    uint32_t *cap = r->cap;
    if (cap[ARENA_SEG_COUNTS] < cap[ARENA_LINES]) cap[ARENA_SEG_COUNTS] = cap[ARENA_LINES];
    if (cap[ARENA_SEGMENTS] < cap[ARENA_SEG_COUNTS] && (r->cur->h_bump->failed & VB_STAGE_PATH_COUNT)) cap[ARENA_SEGMENTS] = cap[ARENA_SEG_COUNTS];
}

extern "C" int vb_frame_finish(vb_renderer *r, vb_frame_stats *stats) {
    if (!r) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    r->frame_pending = false;
    fill_stats(r, stats);
    return r->cur->h_bump->failed ? VB_E_BUMP_OVERFLOW : VB_OK;
}

// One frame, re-run with grown arenas until it fits. Streamed frames still in flight are left alone: the streaming calls
// re-run their own frames through here.
static int render_sync(vb_renderer *r, const vb_params *p, const Dest &d, vb_frame_stats *stats) {
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    r->retries = 0;
    for (uint32_t attempt = 0;; attempt++) {
        int rc = render_enqueue(r, p, d);
        if (rc) return rc;
        CK(cudaStreamSynchronize(r->stream));
        r->frame_pending = false;
        if (r->cur->h_bump->failed == 0) break;
        if (r->xc.enabled) {
            // every attempt of an exchanged frame is a collective step (all GPUs advance their epoch together): grow what
            // overflowed here and let the caller re-issue the frame on every GPU
            grow_arenas(r);
            fill_stats(r, stats);
            r->err = "bump overflow in an exchanged frame: re-issue the frame on every GPU";
            return VB_E_BUMP_OVERFLOW;
        }
        if (attempt >= r->max_retries) {
            fill_stats(r, stats);
            r->err = "bump overflow persisted";
            return VB_E_BUMP_OVERFLOW;
        }
        grow_arenas(r);
        r->retries++;
    }
    fill_stats(r, stats);
    return VB_OK;
}

// render_sync with a host destination, then wait for its copies
static int render_sync_host(vb_renderer *r, const vb_params *p, const Dest &d, vb_frame_stats *stats) {
    int rc = render_sync(r, p, d, stats);
    // the band copies were queued behind the fine bands; a re-run after an arena overflow simply copies again
    cudaError_t e = cudaStreamSynchronize(r->copy_stream);
    if (rc == VB_OK && e != cudaSuccess) {
        r->err = std::string("copy stream: ") + cudaGetErrorString(e);
        return VB_E_CUDA;
    }
    return rc;
}

extern "C" int vb_render_resident(vb_renderer *r, const vb_params *p, void *out_device, vb_frame_stats *stats) {
    if (!r || !p) return VB_E_INVALID;
    int rc = drain_stream(r);
    if (rc) return rc;
    return render_sync(r, p, Dest{out_device}, stats);
}

extern "C" int vb_render_uploaded(vb_renderer *r, const vb_params *p, void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    if (!r || !p || !out) return VB_E_INVALID;
    if (out_is_device) return vb_render_resident(r, p, out, stats);
    int rc = drain_stream(r);
    if (rc) return rc;
    return render_sync_host(r, p, Dest{nullptr, out, false, r->readback_bands}, stats);
}

extern "C" int vb_render(vb_renderer *r, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                         uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, const vb_params *p,
                         void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    if (!r || !p || !out) return VB_E_INVALID;
    int rc = vb_scene_upload(r, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h);
    if (rc) return rc;
    return vb_render_uploaded(r, p, out, out_is_device, stats);
}

// ---- streaming: vb_render_begin / vb_readback_wait ------------------------------------------------------------------------
// Back-to-back frames with HOST buffers (a viewer / exporter reading every frame back, examples/headless/src/main.rs:188-210).
// Three frames are in flight: vb_render_begin(k) uploads frame k's scene into the free scene slot on the upload stream and
// enqueues its rasterisation and read-back; it then makes sure frame k-1 was RASTERISED without an arena overflow and that
// frame k-2's PIXELS are on the host. In steady state the GPU sees  upload(k+1) | raster(k) | read-back(k-1)  side by side and a
// frame costs max(raster, read-back) instead of their sum. On return every frame before the previous one is complete in its
// out_host and `stats` describes frame k-2 (zeros while there is none); vb_readback_wait completes the rest. THREE alternating
// out_host buffers are needed. An arena overflow is found at the rasterisation check; that frame (and the one enqueued behind
// it) is then re-run synchronously with grown arenas -- rare (first frames of a new scene size) and exact.
static int rerun_frame_sync(vb_renderer *r, uint32_t q, vb_frame_stats *stats) {
    const uint32_t slot = r->ring[q].slot;
    r->cur = &r->slot[slot];
    return render_sync_host(r, &r->ring[q].params, Dest{nullptr, r->ring[q].out_host, slot != 0u, 1u}, stats);
}

// Frame in ring entry q: wait for its kernels, look at its bump counters, re-run on overflow (together with the younger frame
// enqueued behind it, ring entry `younger`, or -1).
static int check_raster(vb_renderer *r, uint32_t q, int younger) {
    vb_renderer::RingFrame &f = r->ring[q];
    if (!f.pending || f.raster_checked) return VB_OK;
    vb_renderer::SceneSlot *const keep = r->cur;
    CK(cudaEventSynchronize(r->raster_done[f.slot]));
    r->cur = &r->slot[f.slot];
    int rc = VB_OK;
    if (r->cur->h_bump->failed != 0u) {
        CK(cudaStreamSynchronize(r->stream));
        CK(cudaStreamSynchronize(r->copy_stream));
        grow_arenas(r);
        rc = rerun_frame_sync(r, q, &f.stats);
        CK(cudaEventRecord(r->copy_done[q], r->copy_stream));
        if (rc == VB_OK && younger >= 0 && r->ring[younger].pending) {
            r->cur = &r->slot[r->ring[younger].slot];
            if (r->cur->h_bump->failed != 0u) {
                rc = rerun_frame_sync(r, (uint32_t)younger, &r->ring[younger].stats);
                CK(cudaEventRecord(r->raster_done[r->ring[younger].slot], r->stream));
                CK(cudaEventRecord(r->copy_done[younger], r->copy_stream));
            }
        }
    } else {
        r->retries = 0;
        fill_stats(r, &f.stats);
    }
    f.raster_checked = true;
    r->cur = keep;
    return rc;
}

static int complete_host(vb_renderer *r, uint32_t q, vb_frame_stats *stats) {
    vb_renderer::RingFrame &f = r->ring[q];
    if (!f.pending) return VB_OK;
    int rc = check_raster(r, q, -1);
    CK(cudaEventSynchronize(r->copy_done[q]));
    if (stats) *stats = f.stats;
    f.pending = false;
    return rc;
}

extern "C" int vb_render_begin(vb_renderer *r, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                               uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h,
                               const vb_params *p, void *out_host, vb_frame_stats *stats) {
    if (!r || !p || !out_host) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    if (stats) memset(stats, 0, sizeof *stats);
    const uint64_t k = r->stream_seq;
    const uint32_t slot = (uint32_t)(k & 1u), q = (uint32_t)(k % 3u), q1 = (uint32_t)((k + 2u) % 3u), q2 = (uint32_t)((k + 1u) % 3u);
    // frame k-2 (same scene slot, same device target) was checked by the previous call; frame k-3 (ring entry q) is complete
    r->cur = &r->slot[slot];
    int rc = upload_on(r, r->upload_stream, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h);
    if (rc) return rc;
    CK(cudaEventRecord(r->upload_done[slot], r->upload_stream));
    CK(cudaStreamWaitEvent(r->stream, r->upload_done[slot], 0));
    if (k >= 2u && r->ring[q2].pending) CK(cudaStreamWaitEvent(r->stream, r->copy_done[q2], 0)); // its read-back still reads this target
    // one band: the whole read-back overlaps the next frames, no reason to split fine
    rc = render_enqueue(r, p, Dest{nullptr, out_host, slot != 0u, 1u});
    if (rc) return rc;
    r->frame_pending = false;
    CK(cudaEventRecord(r->raster_done[slot], r->stream));
    CK(cudaEventRecord(r->copy_done[q], r->copy_stream));
    r->ring[q].pending = true;
    r->ring[q].raster_checked = false;
    r->ring[q].params = *p;
    r->ring[q].out_host = out_host;
    r->ring[q].slot = slot;
    memset(&r->ring[q].stats, 0, sizeof(vb_frame_stats));
    r->stream_seq = k + 1u;
    r->stream_pending = true;
    // frame k-1: rasterised without overflow?  frame k-2: pixels on the host?
    if (k >= 1u) rc = check_raster(r, q1, (int)q);
    if (k >= 2u) {
        const int rc2 = complete_host(r, q2, stats);
        if (rc == VB_OK) rc = rc2;
    }
    return rc;
}

extern "C" int vb_readback_wait(vb_renderer *r) {
    if (!r) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    int rc = VB_OK;
    const uint64_t k = r->stream_seq; // the next frame number: complete k-3 .. k-1 in order
    for (uint64_t j = k >= 3u ? k - 3u : 0u; j < k; j++) {
        const uint32_t q = (uint32_t)(j % 3u);
        const int younger = j + 1u < k ? (int)((j + 1u) % 3u) : -1;
        int rc1 = check_raster(r, q, younger);
        if (rc1 == VB_OK) rc1 = complete_host(r, q, nullptr);
        if (rc == VB_OK) rc = rc1;
    }
    CK(cudaStreamSynchronize(r->copy_stream));
    r->stream_pending = false;
    return rc;
}

extern "C" int vb_run_stages(vb_renderer *r, const vb_params *p, int first, int last, void *out_device) {
    if (!r || !p || first < 0 || last >= VB_N_STAGE_IDS || first > last) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    CK(cudaSetDevice(r->device));
    int rc = prepare(r, p);
    if (rc) return rc;
    Dest d{out_device};
    if (last == VB_STAGE_ID_FINE && (rc = pick_out(r, &d))) return rc;
    if ((rc = enqueue(r, first, last, d, true))) return rc;
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

struct NamedBuf {
    const char *name;
    DevBuf *buf;
    size_t bytes;
};
static std::vector<NamedBuf> named(vb_renderer *r) {
    const VbConfig &c = r->cfg;
    const VbLayout &L = r->cur->layout;
    const uint32_t wb = (c.width_in_tiles + 15u) / 16u, hb = (c.height_in_tiles + 15u) / 16u;
    const uint32_t aligned_n_bins = (wb * hb * std::max(c.n_cells, 1u) + 255u) & ~255u;
    std::vector<NamedBuf> v = {
        {"scene", &r->cur->scene, r->cur->scene_words * 4}, // the uploaded / device-resolved inputs
        {"ramps", &r->cur->ramps, (size_t)r->cur->n_ramps * 512 * 4},
        {"atlas", &r->cur->atlas, (size_t)r->cur->atlas_w * r->cur->atlas_h * 4},
        {"tag_monoids", &r->tag_monoids, (size_t)c.n_tag_words * sizeof(VbTagMonoid)},
        {"path_bboxes", &r->path_bboxes, (size_t)L.n_paths * sizeof(VbPathBbox)},
        {"draw_monoids", &r->draw_monoids, (size_t)L.n_draw_objects * sizeof(VbDrawMonoid)},
        {"clip_inp", &r->clip_inp, (size_t)L.n_clips * sizeof(VbClipInp)},
        {"clip_bboxes", &r->clip_bboxes, (size_t)L.n_clips * sizeof(VbBbox4)},
        {"draw_bboxes", &r->draw_bboxes, (size_t)L.n_draw_objects * sizeof(VbBbox4)},
        {"bin_headers", &r->bin_headers, (size_t)((L.n_draw_objects + 255u) / 256u) * aligned_n_bins * sizeof(VbBinHeader)},
        {"paths", &r->paths, (size_t)L.n_draw_objects * sizeof(VbPath)},
    };
    // an arena's buffer up to what the last attempt used of it, at most the capacity the kernels saw
    const uint32_t *size = &c.lines_size;
    for (int a = 0; a < N_ARENAS; a++) {
        const ArenaDesc &d = ARENAS[a];
        const size_t used = (size_t)std::min<uint64_t>(arena_need(r, a), size[a]);
        v.push_back({d.download ? d.download : d.name, &(r->*d.buf), (arena_offset(r, a) + used) * d.elem_bytes});
    }
    return v;
}

// The guard region of a limited arena (vb_debug_limit_arena): the bytes of its allocation past the limit. `name` is an arena
// name, or "line_scratch" / "flatten_jobs" (flatten's scratch arenas, sized from the lines capacity). Returns false for an
// unknown name; *buf is nullptr while the arena has no limit.
static bool guard_region(vb_renderer *r, const char *name, DevBuf **buf, size_t *off) {
    DevBuf *scratch = !strcmp(name, "line_scratch") ? &r->line_scratch : !strcmp(name, "flatten_jobs") ? &r->flatten_jobs : nullptr;
    const int a = scratch ? ARENA_LINES : arena_index(name);
    if (a < 0) return false;
    *buf = nullptr;
    *off = 0;
    const uint32_t lim = r->limit[a];
    if (lim == UINT32_MAX) return true;
    // ptcl: includes the 512 bytes of window slack that fine reads and never writes
    DevBuf *b = &(r->*ARENAS[a].buf);
    size_t o = (arena_offset(r, a) + lim) * ARENAS[a].elem_bytes;
    if (scratch) {
        size_t lit_bytes, job_bytes; // flatten sees lits_cap = lines_size, jobs_cap = lines_size / FL_DEFER_MIN + 1
        vb_flatten_arena_bytes(lim, &lit_bytes, &job_bytes);
        b = scratch;
        o = scratch == &r->line_scratch ? lit_bytes : job_bytes;
    }
    *buf = b;
    *off = o < b->cap ? o : b->cap;
    return true;
}

extern "C" int vb_debug_limit_arena(vb_renderer *r, const char *arena, uint32_t limit) {
    if (!r || !arena) return VB_E_INVALID;
    const int a = arena_index(arena);
    if (a < 0) {
        r->err = std::string("vb_debug_limit_arena: unknown arena ") + arena;
        return VB_E_INVALID;
    }
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    CK(cudaStreamSynchronize(r->upload_stream));
    if (limit == UINT32_MAX) {
        r->limit[a] = UINT32_MAX;
        return VB_OK;
    }
    // 0 is refused too: path_count and path_tiling size their grids from the capacity
    if (limit == 0u || limit > r->cap[a] || (a == ARENA_PTCL && limit < ptcl_static(r->cfg))) {
        r->err = "vb_debug_limit_arena: the limit must be at least 1 (the static area for ptcl) and at most the allocation";
        return VB_E_INVALID;
    }
    r->limit[a] = limit;
    const char *regions[3] = {ARENAS[a].name, "line_scratch", "flatten_jobs"};
    for (int k = 0; k < (a == ARENA_LINES ? 3 : 1); k++) {
        DevBuf *b;
        size_t off;
        guard_region(r, regions[k], &b, &off);
        if (b && b->cap > off) CK(cudaMemsetAsync((char *)b->p + off, VB_GUARD_BYTE, b->cap - off, r->stream));
    }
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

extern "C" int vb_debug_download(vb_renderer *r, const char *name, void *dst, size_t cap, size_t *bytes) {
    if (!r || !name) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    const size_t len = strlen(name);
    if (len > 6 && !strcmp(name + len - 6, ".guard")) {
        const std::string base(name, len - 6);
        DevBuf *b;
        size_t off;
        if (!guard_region(r, base.c_str(), &b, &off)) return VB_E_UNKNOWN_BUFFER;
        const size_t n = b ? b->cap - off : 0;
        if (bytes) *bytes = n;
        const size_t c = n < cap ? n : cap;
        if (dst && c) CK(cudaMemcpy(dst, (const char *)b->p + off, c, cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    if (!strcmp(name, "bump")) {
        if (bytes) *bytes = sizeof(VbBump);
        if (dst && cap >= sizeof(VbBump)) CK(cudaMemcpy(dst, r->ctl.p, sizeof(VbBump), cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    if (!strcmp(name, "seg_holes")) { // segment slots of the last frame that backdrop assigned and no CMD_FILL uses (k_tile.cu, k_coarse.cu)
        if (bytes) *bytes = 4;
        if (dst && cap >= 4) CK(cudaMemcpy(dst, (const uint32_t *)r->ctl.p + VB_CTL_SEG_HOLES, 4, cudaMemcpyDeviceToHost));
        return VB_OK;
    }
    if (!strcmp(name, "config")) {
        if (bytes) *bytes = sizeof(VbConfig);
        if (dst && cap >= sizeof(VbConfig)) memcpy(dst, &r->cfg, sizeof(VbConfig));
        return VB_OK;
    }
    for (auto &nb : named(r))
        if (!strcmp(name, nb.name)) {
            if (bytes) *bytes = nb.bytes;
            size_t n = nb.bytes < cap ? nb.bytes : cap;
            if (dst && n) CK(cudaMemcpy(dst, nb.buf->p, n, cudaMemcpyDeviceToHost));
            return VB_OK;
        }
    return VB_E_UNKNOWN_BUFFER;
}

extern "C" int vb_set_timing(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    r->timing = on != 0;
    return VB_OK;
}

extern "C" int vb_set_cuda_graph(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    r->use_graph = on != 0;
    return VB_OK;
}

extern "C" int vb_set_readback_bands(vb_renderer *r, uint32_t n) {
    if (!r || n < 1u || n > 8u) return VB_E_INVALID;
    r->readback_bands = n;
    return VB_OK;
}

extern "C" int vb_set_occlusion_cull(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    r->occlusion_cull = on ? 1u : 0u;
    return VB_OK;
}

// ---- batches: many scenes of one size in one pass (vb_scene_batch builds the scene) ---------------------------------------
// The offsets split the uploaded scene's draw objects into cells. Validated here against the uploaded draw tags (one download):
// a cell whose clips do not balance would pair a BEGIN_CLIP of one cell with an END_CLIP of the next. What depends on the
// frame size (arena indexing) and on the call (windows) is checked when a frame is prepared.
extern "C" int vb_set_cells(vb_renderer *r, const uint32_t *draw_offsets, uint32_t n_cells) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const std::string &why) {
        r->err = "vb_set_cells: " + why;
        return VB_E_INVALID;
    };
    if (!draw_offsets || n_cells == 0u) return bad("no offsets");
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    if (r->xc.enabled || r->grouped) return bad("a batch cannot be combined with vb_group or the exchange");
    int rc = drain_stream(r);
    if (rc) return rc;
    CK(cudaSetDevice(r->device));
    const VbLayout &L = r->cur->layout;
    const uint32_t n_draw = L.n_draw_objects;
    if (draw_offsets[0] != 0u || draw_offsets[n_cells] != n_draw) return bad("offsets must start at 0 and end at the scene's draw-object count");
    for (uint32_t c = 0; c < n_cells; c++)
        if (draw_offsets[c + 1] < draw_offsets[c]) return bad("offsets must not decrease");
    if (n_cells == 1u) { // the whole scene: no batch
        r->cells.clear();
        return VB_OK;
    }
    std::vector<uint32_t> tags(n_draw);
    if (n_draw) {
        CK(cudaMemcpyAsync(tags.data(), (const uint32_t *)r->cur->scene.p + L.draw_tag_base, (size_t)n_draw * 4, cudaMemcpyDeviceToHost, r->stream));
        CK(cudaStreamSynchronize(r->stream));
    }
    for (uint32_t c = 0; c < n_cells; c++) {
        int64_t depth = 0;
        for (uint32_t i = draw_offsets[c]; i < draw_offsets[c + 1] && depth >= 0; i++)
            depth += tags[i] == VB_DRAWTAG_BEGIN_CLIP ? 1 : tags[i] == VB_DRAWTAG_END_CLIP ? -1 : 0;
        if (depth != 0) return bad("the clips of cell " + std::to_string(c) + " do not balance");
    }
    if ((rc = ensure(r, r->cell_draw, ((size_t)n_cells + 1u) * 4u))) return rc;
    r->cells.assign(draw_offsets, draw_offsets + n_cells + 1u);
    // in stream order: a frame still running reads the previous offsets
    CK(cudaMemcpyAsync(r->cell_draw.p, r->cells.data(), r->cells.size() * 4u, cudaMemcpyHostToDevice, r->stream));
    return VB_OK;
}

extern "C" int vb_debug_fine_traffic(vb_renderer *r, uint64_t *ptcl_words, uint64_t *segment_refs, uint64_t *fill_cmds) {
    if (!r) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    unsigned long long *d = nullptr, h[3] = {0, 0, 0};
    CK(cudaMalloc(&d, sizeof h));
    CK(cudaMemset(d, 0, sizeof h));
    VbConfig c = r->cfg;
    const FineRows f = fine_rows(c, Dest{});
    c.win_ty0 = f.ty0, c.win_ty1 = f.ty1;
    uint32_t n = c.width_in_tiles * (c.win_ty1 - c.win_ty0);
    if (n) k_ptcl_stats<<<(n + 127) / 128, 128, 0, r->stream>>>(c, (const uint32_t *)r->ptcl.p,
                                                                r->occlusion_cull ? (const uint32_t *)r->tile_start.p : nullptr, d);
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaMemcpy(h, d, sizeof h, cudaMemcpyDeviceToHost));
    cudaFree(d);
    if (ptcl_words) *ptcl_words = h[0];
    if (segment_refs) *segment_refs = h[1];
    if (fill_cmds) *fill_cmds = h[2];
    return VB_OK;
}

extern "C" int vb_debug_upload(vb_renderer *r, const char *name, const void *src, size_t bytes) {
    if (!r || !name || !src) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    // "lines" and "tiles": the arena's contents and its bump counter. Growing the arena frees it without copying, and the
    // look-back state of backdrop is sized from the tile capacity when the next frame is prepared.
    for (int a : {ARENA_LINES, ARENA_TILES}) {
        if (strcmp(name, ARENAS[a].name)) continue;
        const uint32_t n = (uint32_t)(bytes / ARENAS[a].elem_bytes);
        if (n > r->cap[a]) {
            r->cap[a] = grow(n);
            int rc = ensure_arena(r, a);
            if (rc) return rc;
        }
        if (n) CK(cudaMemcpy((r->*ARENAS[a].buf).p, src, (size_t)n * ARENAS[a].elem_bytes, cudaMemcpyHostToDevice));
        VbBump *bump = (VbBump *)r->ctl.p;
        CK(cudaMemcpy(&(bump->*ARENAS[a].counter), &n, 4, cudaMemcpyHostToDevice));
        r->cur->h_bump->*ARENAS[a].counter = n;
        return VB_OK;
    }
    if (!strcmp(name, "path_bboxes")) {
        if (bytes > r->path_bboxes.cap) return VB_E_INVALID;
        CK(cudaMemcpy(r->path_bboxes.p, src, bytes, cudaMemcpyHostToDevice));
        return VB_OK;
    }
    if (!strcmp(name, "paths")) { // backdrop searches exactly n_draw_objects of them
        if (bytes != (size_t)r->cur->layout.n_draw_objects * sizeof(VbPath) || bytes > r->paths.cap) {
            r->err = "vb_debug_upload: \"paths\" takes exactly one record per draw object, after a frame of the scene";
            return VB_E_INVALID;
        }
        if (bytes) CK(cudaMemcpy(r->paths.p, src, bytes, cudaMemcpyHostToDevice));
        return VB_OK;
    }
    return VB_E_UNKNOWN_BUFFER;
}

extern "C" int vb_debug_lookback(vb_renderer *r, int op, uint32_t n_parts, const uint32_t *agg, const uint32_t *delay_ns, uint32_t *excl) {
    if (!r) return VB_E_INVALID;
    const uint32_t K = vb_debug_lookback_words(op);
    if (!agg || !excl || K == 0u || n_parts == 0u || n_parts > VB_LOOKBACK_MAX_PARTS) {
        r->err = "vb_debug_lookback: unknown op, no buffers, or n_parts outside 1..VB_LOOKBACK_MAX_PARTS";
        return VB_E_INVALID;
    }
    for (uint32_t p = 0; delay_ns && p < n_parts; p++)
        if (delay_ns[p] > VB_LOOKBACK_MAX_DELAY_NS) {
            r->err = "vb_debug_lookback: a delay exceeds VB_LOOKBACK_MAX_DELAY_NS";
            return VB_E_INVALID;
        }
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    // one allocation: [look-back state][agg: n_parts * K][delays: n_parts][excl: n_parts * K]
    const size_t lb_words = vb_lookback_words(n_parts, (int)K), vec = (size_t)n_parts * K;
    DevBuf d;
    int rc = ensure(r, d, (lb_words + 2 * vec + n_parts) * 4);
    if (rc) return rc;
    uint32_t *lb = (uint32_t *)d.p, *d_agg = lb + lb_words, *d_delay = d_agg + vec, *d_excl = d_delay + n_parts;
    auto run = [&]() -> int {
        CK(cudaMemsetAsync(lb, 0, lb_words * 4, r->stream));
        CK(cudaMemcpyAsync(d_agg, agg, vec * 4, cudaMemcpyHostToDevice, r->stream));
        if (delay_ns) CK(cudaMemcpyAsync(d_delay, delay_ns, (size_t)n_parts * 4, cudaMemcpyHostToDevice, r->stream));
        else CK(cudaMemsetAsync(d_delay, 0, (size_t)n_parts * 4, r->stream));
        vb_launch_debug_lookback(op, n_parts, lb, d_agg, d_delay, d_excl, r->stream);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(excl, d_excl, vec * 4, cudaMemcpyDeviceToHost, r->stream));
        CK(cudaStreamSynchronize(r->stream));
        return VB_OK;
    };
    rc = run();
    cudaFree(d.p);
    return rc;
}


extern "C" float vb_last_frame_ms(vb_renderer *r) {
    if (!r || !r->frame_timed) return 0.0f;
    cudaSetDevice(r->device);
    float ms = 0.0f;
    if (cudaEventSynchronize(r->frame_ev[1]) != cudaSuccess || cudaEventElapsedTime(&ms, r->frame_ev[0], r->frame_ev[1]) != cudaSuccess) {
        cudaGetLastError();
        return 0.0f;
    }
    return ms;
}

// ---- CUDA IPC helpers (one process per GPU: the frame buffer of rank 0 mapped into the other ranks) ----------------------
extern "C" int vb_frame_alloc(vb_renderer *r, size_t bytes, void **device_ptr) {
    if (!r || !device_ptr || !bytes) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaMalloc(device_ptr, bytes));
    return VB_OK;
}
extern "C" int vb_frame_free(vb_renderer *r, void *device_ptr) {
    if (!r) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    if (device_ptr) CK(cudaFree(device_ptr));
    return VB_OK;
}
extern "C" int vb_ipc_export(vb_renderer *r, void *device_ptr, uint8_t handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    if (!r || !device_ptr || !handle) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, device_ptr));
    memcpy(handle, &h, 64);
    return VB_OK;
}
extern "C" int vb_ipc_open(vb_renderer *r, const uint8_t handle[64], void **device_ptr) {
    if (!r || !handle || !device_ptr) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CK(cudaIpcOpenMemHandle(device_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return VB_OK;
}
extern "C" int vb_ipc_close(vb_renderer *r, void *device_ptr) {
    if (!r || !device_ptr) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaIpcCloseMemHandle(device_ptr));
    return VB_OK;
}

// ---- vb_group: one frame on several devices of one box, one host thread ---------------------------------------------------
struct vb_group {
    std::vector<vb_renderer *> subs;
    std::vector<int> devices;
    std::vector<uint32_t> bounds;   // tile-row boundaries, subs.size() + 1 entries
    std::vector<float> ms;          // device time of the last frame per renderer
    std::vector<char> peer_ok;      // renderer i can store into device 0's memory
    std::vector<cudaEvent_t> done;  // per renderer: its stripe is in the frame
    void *frame = nullptr;          // assembled frame on devices[0]
    size_t frame_cap = 0;
    uint32_t bounds_h = 0;          // height in tiles the boundaries were made for
    bool balancing = true;
    bool exchange = false;          // flatten sharded by tag range, lines exchanged through peer memory (k_exchange.cu)
    bool shared_device = false;     // two renderers on one GPU (tests)
    std::string err;
};

extern "C" int vb_group_new(const int32_t *devices, uint32_t n, const vb_options *opt, vb_group **out) {
    if (!devices || !n || n > 64 || !out) return VB_E_INVALID;
    vb_group *g = new vb_group();
    for (uint32_t i = 0; i < n; i++) {
        vb_options o{};
        if (opt) o = *opt;
        o.device = devices[i];
        vb_renderer *r = nullptr;
        int rc = vb_renderer_new(&o, &r);
        if (rc) {
            vb_group_free(g);
            return rc;
        }
        r->grouped = true;
        g->subs.push_back(r);
        g->devices.push_back(devices[i]);
        cudaEvent_t ev = nullptr;
        cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        g->done.push_back(ev);
        // stores of `fine` on device i land in device 0's frame buffer through peer mapping (NVLink / NVSwitch)
        char ok = 1;
        if (devices[i] != devices[0]) {
            int can = 0;
            cudaSetDevice(devices[i]);
            if (cudaDeviceCanAccessPeer(&can, devices[i], devices[0]) != cudaSuccess || !can) ok = 0;
            else {
                cudaError_t e = cudaDeviceEnablePeerAccess(devices[0], 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ok = 0;
                cudaGetLastError();
            }
        }
        g->peer_ok.push_back(ok);
    }
    g->ms.assign(n, 0.0f);
    *out = g;
    return VB_OK;
}

extern "C" void vb_group_free(vb_group *g) {
    if (!g) return;
    for (vb_renderer *r : g->subs) vb_renderer_free(r);
    if (!g->devices.empty()) cudaSetDevice(g->devices[0]);
    if (g->frame) cudaFree(g->frame);
    for (cudaEvent_t ev : g->done)
        if (ev) cudaEventDestroy(ev);
    delete g;
}
extern "C" uint32_t vb_group_size(const vb_group *g) { return g ? (uint32_t)g->subs.size() : 0u; }
extern "C" vb_renderer *vb_group_renderer(vb_group *g, uint32_t i) { return g && i < g->subs.size() ? g->subs[i] : nullptr; }
extern "C" const char *vb_group_last_error(vb_group *g) { return g ? g->err.c_str() : ""; }
extern "C" int vb_group_set_balancing(vb_group *g, int on) {
    if (!g) return VB_E_INVALID;
    g->balancing = on != 0;
    return VB_OK;
}
extern "C" void *vb_group_frame(vb_group *g, size_t *bytes) {
    if (!g) return nullptr;
    if (bytes) *bytes = g->frame_cap;
    return g->frame;
}
extern "C" int vb_group_stripes(vb_group *g, uint32_t *boundaries, float *device_ms) {
    if (!g) return VB_E_INVALID;
    if (boundaries)
        for (size_t i = 0; i < g->bounds.size(); i++) boundaries[i] = g->bounds[i];
    if (device_ms)
        for (size_t i = 0; i < g->ms.size(); i++) device_ms[i] = g->ms[i];
    return VB_OK;
}

// Move the stripe boundaries so that the device times of the last frame would have been equal, assuming the cost of a stripe is
// spread evenly over its tile rows (piecewise-linear cumulative cost); damped, every stripe keeps at least one tile row.
static void group_rebalance(vb_group *g, uint32_t ht) {
    const size_t n = g->subs.size();
    if (g->bounds.size() != n + 1 || g->bounds_h != ht) {
        g->bounds.assign(n + 1, 0u);
        for (size_t i = 0; i <= n; i++) g->bounds[i] = (uint32_t)((uint64_t)ht * i / n);
        g->bounds_h = ht;
        return;
    }
    if (!g->balancing || n < 2 || ht < n) return;
    double total = 0.0, lo = 1e30, hi = 0.0;
    for (size_t i = 0; i < n; i++) {
        if (!(g->ms[i] > 0.0f)) return; // no measurement yet
        total += g->ms[i];
        lo = std::min<double>(lo, g->ms[i]);
        hi = std::max<double>(hi, g->ms[i]);
    }
    if (hi - lo < 0.06 * (total / n)) return; // balanced within noise: keep the stripes (and the captured graphs)
    std::vector<uint32_t> nb(n + 1, 0u);
    nb[n] = ht;
    size_t seg = 0;
    double acc = 0.0; // cost of the stripes before `seg`
    for (size_t k = 1; k < n; k++) {
        const double want = total * k / n;
        while (seg + 1 < n && acc + g->ms[seg] < want) acc += g->ms[seg++];
        const double rows = (double)(g->bounds[seg + 1] - g->bounds[seg]);
        const double frac = g->ms[seg] > 0.0f ? (want - acc) / g->ms[seg] : 0.0;
        const double ideal = g->bounds[seg] + rows * frac;
        const double damped = 0.5 * g->bounds[k] + 0.5 * ideal;
        nb[k] = (uint32_t)(damped + 0.5);
    }
    for (size_t k = 1; k < n; k++) { // monotone, at least one row each
        if (nb[k] < nb[k - 1] + 1u) nb[k] = nb[k - 1] + 1u;
    }
    for (size_t k = n - 1; k >= 1; k--) {
        if (nb[k] > nb[k + 1] - 1u) nb[k] = nb[k + 1] - 1u;
    }
    g->bounds = nb;
}

#define GCK(call)                                                                                 \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) {                                                                  \
            g->err = std::string(#call) + ": " + cudaGetErrorString(e_);                          \
            return VB_E_CUDA;                                                                     \
        }                                                                                         \
    } while (0)

// (re)build the exchange arenas for the uploaded scene and introduce the renderers to each other
static int group_setup_exchange(vb_group *g) {
    const uint32_t n = (uint32_t)g->subs.size();
    if (n > 8u) return VB_E_INVALID;
    std::vector<void *> arenas(n, nullptr);
    for (uint32_t i = 0; i < n; i++) {
        int rc = vb_exchange_configure(g->subs[i], i, n, &arenas[i], nullptr);
        if (rc) {
            g->err = g->subs[i]->err;
            return rc;
        }
    }
    for (uint32_t i = 0; i < n; i++) {
        for (uint32_t j = 0; j < n; j++) {
            if (i == j) continue;
            if (g->devices[i] != g->devices[j]) { // every GPU reads every other GPU's arena
                int can = 0;
                cudaSetDevice(g->devices[i]);
                if (cudaDeviceCanAccessPeer(&can, g->devices[i], g->devices[j]) != cudaSuccess || !can) {
                    g->err = "exchange needs peer access between all devices of the group";
                    return VB_E_CUDA;
                }
                cudaError_t e = cudaDeviceEnablePeerAccess(g->devices[j], 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                    g->err = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e);
                    return VB_E_CUDA;
                }
                cudaGetLastError();
            }
            int rc = vb_exchange_attach(g->subs[i], j, arenas[j]);
            if (rc) return rc;
        }
    }
    bool shared_device = false;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t j = i + 1; j < n; j++) shared_device = shared_device || g->devices[i] == g->devices[j];
    g->shared_device = shared_device;
    for (uint32_t i = 0; i < n; i++) {
        int rc = vb_exchange_enable(g->subs[i], 1);
        if (rc) return rc;
        // renderers that share a GPU (tests): no graph (re-)instantiation while a peer's wait kernel is resident on that GPU
        if (shared_device) g->subs[i]->use_graph = false;
    }
    return VB_OK;
}

extern "C" int vb_group_set_exchange(vb_group *g, int on) {
    if (!g) return VB_E_INVALID;
    g->exchange = on != 0;
    if (!g->exchange) {
        for (vb_renderer *r : g->subs) vb_exchange_enable(r, 0);
        return VB_OK;
    }
    for (vb_renderer *r : g->subs)
        if (!r->cur->have_scene) return VB_OK; // arenas are built by the next vb_group_scene_upload
    return group_setup_exchange(g);
}

extern "C" int vb_group_scene_upload(vb_group *g, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                                     uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h) {
    if (!g) return VB_E_INVALID;
    // every device pulls the scene over its own PCIe link (asynchronous per renderer, so the copies run side by side)
    for (vb_renderer *r : g->subs) {
        int rc = vb_scene_upload(r, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h);
        if (rc) {
            g->err = r->err;
            return rc;
        }
    }
    return g->exchange ? group_setup_exchange(g) : VB_OK;
}

// out: nullptr (group frame), a device pointer on devices[0], or (host_out) a host pointer
static int group_render(vb_group *g, const vb_params *p, void *out_device, void *host_out, vb_frame_stats *stats) {
    if (!g || !p || p->bin_row1 > p->bin_row0 || p->tile_row1 > p->tile_row0) return VB_E_INVALID;
    const size_t n = g->subs.size();
    const uint32_t ht = (p->height + 15u) / 16u;
    if (g->exchange && ht < n) {
        g->err = "exchange needs at least one tile row per device";
        return VB_E_INVALID;
    }
    group_rebalance(g, ht);
    const size_t pitch = (size_t)p->width * 4u;
    void *frame = out_device;
    if (!host_out && !frame) {
        const size_t need = pitch * p->height;
        if (g->frame_cap < need) {
            GCK(cudaSetDevice(g->devices[0]));
            if (g->frame) GCK(cudaFree(g->frame));
            g->frame = nullptr;
            g->frame_cap = 0;
            GCK(cudaMalloc(&g->frame, need));
            g->frame_cap = need;
        }
        frame = g->frame;
    }
    // enqueue every device's stripe, then complete them (one host thread; the devices run side by side)
    std::vector<vb_params> ps(n, *p);
    // device destination: straight into the frame on devices[0] when peer-mapped; otherwise (and for a host destination) the
    // renderer's own target. Without the exchange a host destination's stripe is copied by the frame itself, on the
    // renderer's copy stream.
    auto dest_of = [&](size_t i) {
        const size_t row0 = (size_t)g->bounds[i] * 16u;
        Dest d;
        if (!host_out && g->peer_ok[i]) d.dev = (char *)frame + row0 * pitch;
        if (host_out && !g->exchange) d.host = (char *)host_out + row0 * pitch;
        return d;
    };
    int result = VB_OK;
    for (uint32_t attempt = 0;; attempt++) {
        if (g->exchange)
            for (vb_renderer *r : g->subs) vb_exchange_set_bounds(r, g->bounds.data());
        const bool halves = g->exchange && g->shared_device;
        // phases: 0 = configs and arenas of every renderer, 1 (and 2) = the launches, last = the read-backs of a host
        // destination. A copy into pageable host memory blocks the host until it is done, so it must not be issued before
        // every renderer's frame has been launched (with the exchange on, a frame waits for its peers).
        const int n_launch = halves ? 2 : 1;
        const bool late_copy = host_out != nullptr && g->exchange; // without the exchange every frame queues its own read-back
        for (int phase = 0; phase < 1 + n_launch + (late_copy ? 1 : 0); phase++) {
            for (size_t i = 0; i < n; i++) {
                vb_renderer *r = g->subs[i];
                ps[i].tile_row0 = g->bounds[i];
                ps[i].tile_row1 = g->bounds[i + 1];
                if (ps[i].tile_row1 <= ps[i].tile_row0) continue; // more devices than tile rows (never with the exchange on)
                const size_t row0 = (size_t)g->bounds[i] * 16u;
                int rc = VB_OK;
                if (phase == 0) rc = frame_prepare(r, &ps[i], dest_of(i));
                else if (phase <= n_launch) rc = halves ? frame_launch_half(r, phase - 1) : frame_launch(r);
                else {
                    const size_t h1 = std::min<size_t>((size_t)g->bounds[i + 1] * 16u, p->height);
                    cudaSetDevice(r->device);
                    if (h1 > row0 && cudaMemcpyAsync((char *)host_out + row0 * pitch, r->dest.dev, (h1 - row0) * pitch, cudaMemcpyDeviceToHost, r->stream) != cudaSuccess)
                        rc = VB_E_CUDA;
                }
                if (rc) {
                    g->err = r->err;
                    return rc;
                }
            }
        }
        result = VB_OK;
        bool redo = false;
        for (size_t i = 0; i < n; i++) {
            vb_renderer *r = g->subs[i];
            if (ps[i].tile_row1 <= ps[i].tile_row0) {
                if (stats) memset(&stats[i], 0, sizeof(vb_frame_stats));
                continue;
            }
            const size_t row0 = (size_t)g->bounds[i] * 16u;
            int rc = vb_frame_finish(r, stats ? &stats[i] : nullptr);
            if (rc == VB_E_BUMP_OVERFLOW) {
                if (g->exchange) { // an exchanged frame is re-issued on EVERY device (epochs advance together)
                    grow_arenas(r);
                    redo = true;
                    rc = VB_OK;
                } else {
                    // grow and re-run (first frames); with a host destination the re-run queues its read-back again.
                    // Growing first: the same attempt with the same arenas would only overflow again.
                    grow_arenas(r);
                    rc = render_sync(r, &ps[i], dest_of(i), stats ? &stats[i] : nullptr);
                    if (stats) stats[i].retries += 1;
                }
            }
            g->ms[i] = vb_last_frame_ms(r);
            if (rc == VB_OK && host_out && !late_copy) {
                cudaSetDevice(r->device);
                if (cudaStreamSynchronize(r->copy_stream) != cudaSuccess) rc = VB_E_CUDA;
            }
            if (rc == VB_OK && !host_out && !g->peer_ok[i]) {
                // no peer mapping between these two devices: stage through the renderer's own target
                const size_t h0 = row0, h1 = std::min<size_t>((size_t)g->bounds[i + 1] * 16u, p->height);
                cudaSetDevice(r->device);
                if (h1 > h0 && (cudaMemcpyPeerAsync((char *)frame + row0 * pitch, g->devices[0], r->dest.dev, r->device, (h1 - h0) * pitch, r->stream) != cudaSuccess ||
                                cudaStreamSynchronize(r->stream) != cudaSuccess))
                    rc = VB_E_CUDA;
            }
            if (rc && result == VB_OK) {
                result = rc;
                g->err = r->err;
            }
        }
        if (!redo || result != VB_OK) break;
        if (attempt >= 8u) {
            g->err = "bump overflow persisted in an exchanged frame; failed bits per renderer:";
            for (vb_renderer *q : g->subs) g->err += " 0x" + std::to_string(q->cur->h_bump->failed);
            return VB_E_BUMP_OVERFLOW;
        }
    }
    return result;
}

extern "C" int vb_group_render_resident(vb_group *g, const vb_params *p, void *out_device, vb_frame_stats *stats) {
    return group_render(g, p, out_device, nullptr, stats);
}

extern "C" int vb_group_render(vb_group *g, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                               uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, const vb_params *p,
                               void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    if (!g || !p) return VB_E_INVALID;
    int rc = vb_group_scene_upload(g, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h);
    if (rc) return rc;
    if (out && !out_is_device) return group_render(g, p, nullptr, out, stats);
    return group_render(g, p, out, nullptr, stats);
}


// ---- Resolver::resolve on the device (resolve.rs:183-399): see include/vello_b200.h and k_resolve.cu ---------------------------
extern "C" int vb_scene_upload_streams(vb_renderer *r, const vb_encoding_streams *e, vb_layout *layout_out) {
    if (!r || !e) return VB_E_INVALID;
    if ((e->n_path_tags && !e->path_tags) || (e->n_path_data && !e->path_data) || (e->n_draw_tags && !e->draw_tags) ||
        (e->n_draw_data && !e->draw_data) || (e->n_transforms && !e->transforms) || (e->n_styles && !e->styles) ||
        (e->n_ramp_patches && !e->ramp_patches) || (e->n_image_patches && !e->image_patches))
        return VB_E_INVALID;
    int rc = drain_stream(r);
    if (rc) return rc;
    CK(cudaSetDevice(r->device));
    cudaStream_t st = r->stream;
    std::vector<RsPatch> patches;
    std::vector<RsRamp> ramps;
    std::vector<vb_ramp_stop> stops;
    std::vector<const vb_ramp_patch *> ramp_of;
    // layout: sizes only (resolve.rs:107-154)
    VbLayout L;
    memset(&L, 0, sizeof L);
    L.n_paths = e->n_paths;
    L.n_clips = e->n_clips;
    L.n_draw_objects = e->n_paths;
    const uint32_t n_tags = e->n_path_tags + e->n_open_clips;
    const uint32_t padded = (n_tags + 1023u) & ~1023u; // 4 * PATH_REDUCE_WG bytes (resolve.rs:625, config.rs:237)
    uint32_t off = padded / 4u;
    L.path_tag_base = 0;
    L.path_data_base = off; off += e->n_path_data;
    L.draw_tag_base = off; off += e->n_draw_tags + e->n_open_clips;
    L.draw_data_base = off; off += e->n_draw_data;
    L.transform_base = off; off += e->n_transforms * 6u;
    L.style_base = off; off += e->n_styles * 2u;
    const size_t total_words = off;
    uint32_t info = 0;
    for (uint32_t i = 0; i < e->n_draw_tags; i++) info += (e->draw_tags[i] >> 6) & 0xFu;
    L.bin_data_start = info;
    // late-bound gradient ramps, de-duplicated by (stops, interpolation space) as the ramp cache does
    for (uint32_t i = 0; i < e->n_ramp_patches; i++) {
        const vb_ramp_patch &p = e->ramp_patches[i];
        if (!p.n_stops || !p.stops || p.draw_data_offset >= e->n_draw_data) return VB_E_INVALID;
        uint32_t rid = (uint32_t)ramp_of.size();
        for (uint32_t k = 0; k < ramp_of.size(); k++) {
            const vb_ramp_patch &q = *ramp_of[k];
            if ((q.premul_interp != 0u) == (p.premul_interp != 0u) && q.n_stops == p.n_stops &&
                memcmp(q.stops, p.stops, sizeof(vb_ramp_stop) * p.n_stops) == 0) { rid = k; break; }
        }
        if (rid == ramp_of.size()) {
            ramp_of.push_back(&p);
            ramps.push_back(RsRamp{(uint32_t)stops.size(), p.n_stops, p.premul_interp ? 1u : 0u, 0u});
            stops.insert(stops.end(), p.stops, p.stops + p.n_stops);
        }
        patches.push_back(RsPatch{L.draw_data_base + p.draw_data_offset, (rid << 2) | p.extend});
    }
    // late-bound images: shelf placement (ours; only the (x, y) written into the draw data matters to the pipeline)
    struct Placed { const uint8_t *key; uint32_t w, h, x, y; };
    std::vector<Placed> placed;
    uint32_t atlas_w = 1, x = 0, y = 0, shelf_h = 0;
    const uint32_t MAXW = 2048;
    for (uint32_t i = 0; i < e->n_image_patches; i++) {
        const vb_image_patch &im = e->image_patches[i];
        if (im.draw_data_offset >= e->n_draw_data) return VB_E_INVALID;
        const Placed *hit = nullptr;
        for (const Placed &q : placed)
            if (q.key == im.pixels && q.w == im.width && q.h == im.height) { hit = &q; break; }
        uint32_t px, py;
        if (!hit) {
            if (x + im.width > MAXW) { y += shelf_h; x = 0; shelf_h = 0; }
            placed.push_back(Placed{im.pixels, im.width, im.height, x, y});
            px = x; py = y;
            x += im.width;
            if (im.height > shelf_h) shelf_h = im.height;
            if (x > atlas_w) atlas_w = x;
        } else {
            px = hit->x; py = hit->y;
        }
        patches.push_back(RsPatch{L.draw_data_base + im.draw_data_offset, (px << 16) | py});
    }
    const uint32_t atlas_h = (y + shelf_h) > 1u ? (y + shelf_h) : 1u;
    // images with an override on this renderer come from device memory (one k_atlas_blit); a registered texture needs one
    std::vector<VbBlitRect> blits;
    std::vector<vb_renderer::SceneSlot::OverridePlace> over;
    std::vector<bool> from_device(placed.size(), false);
    for (size_t i = 0; i < placed.size(); i++) {
        const Placed &q = placed[i];
        const auto ov = q.key ? r->overrides.find(q.key) : r->overrides.end();
        if (ov != r->overrides.end()) {
            const vb_renderer::Override &o = ov->second;
            if (o.w != q.w || o.h != q.h) {
                r->err = "device resolve: an override's size differs from its image's (" + std::to_string(o.w) + "x" + std::to_string(o.h) +
                         " vs " + std::to_string(q.w) + "x" + std::to_string(q.h) + ")";
                return VB_E_INVALID;
            }
            blits.push_back(VbBlitRect{o.src, o.pitch, 0, q.w, q.h, q.x, q.y, 0, 0});
            over.push_back({q.key, o.src, o.pitch, q.w, q.h, q.x, q.y, false});
            from_device[i] = true;
        } else if (vb_texture_key(q.key)) {
            r->err = "device resolve: a registered texture has no override on this renderer";
            return VB_E_INVALID;
        }
    }

    // the six streams go straight to their places in the packed buffer
    if ((rc = ensure(r, r->cur->scene, total_words * 4 + 64))) return rc;
    char *base = (char *)r->cur->scene.p;
    if (e->n_path_tags) CK(cudaMemcpyAsync(base, e->path_tags, e->n_path_tags, cudaMemcpyHostToDevice, st));
    if (e->n_path_data) CK(cudaMemcpyAsync(base + (size_t)L.path_data_base * 4, e->path_data, (size_t)e->n_path_data * 4, cudaMemcpyHostToDevice, st));
    if (e->n_draw_tags) CK(cudaMemcpyAsync(base + (size_t)L.draw_tag_base * 4, e->draw_tags, (size_t)e->n_draw_tags * 4, cudaMemcpyHostToDevice, st));
    if (e->n_draw_data) CK(cudaMemcpyAsync(base + (size_t)L.draw_data_base * 4, e->draw_data, (size_t)e->n_draw_data * 4, cudaMemcpyHostToDevice, st));
    if (e->n_transforms) CK(cudaMemcpyAsync(base + (size_t)L.transform_base * 4, e->transforms, (size_t)e->n_transforms * 24, cudaMemcpyHostToDevice, st));
    if (e->n_styles) CK(cudaMemcpyAsync(base + (size_t)L.style_base * 4, e->styles, (size_t)e->n_styles * 8, cudaMemcpyHostToDevice, st));
    // patches, ramp descriptors and stops in one staging buffer
    static_assert(sizeof(RsStop) == sizeof(vb_ramp_stop), "the stops are staged as the caller gave them");
    const size_t pb = patches.size() * sizeof(RsPatch), rb = ramps.size() * sizeof(RsRamp), sb = stops.size() * sizeof(vb_ramp_stop);
    const size_t o_r = (pb + 15) & ~(size_t)15, o_s = (o_r + rb + 15) & ~(size_t)15;
    if ((rc = ensure(r, r->resolve_tmp, o_s + sb + 16))) return rc;
    char *tmp = (char *)r->resolve_tmp.p;
    if (pb) CK(cudaMemcpyAsync(tmp, patches.data(), pb, cudaMemcpyHostToDevice, st));
    if (rb) CK(cudaMemcpyAsync(tmp + o_r, ramps.data(), rb, cudaMemcpyHostToDevice, st));
    if (sb) CK(cudaMemcpyAsync(tmp + o_s, stops.data(), sb, cudaMemcpyHostToDevice, st));
    vb_launch_resolve_finish((uint32_t *)r->cur->scene.p, e->n_path_tags, e->n_open_clips, padded, L.draw_tag_base + e->n_draw_tags,
                             (const RsPatch *)tmp, (uint32_t)patches.size(), st);
    r->cur->n_ramps = (uint32_t)ramps.size();
    if ((rc = ensure(r, r->cur->ramps, (size_t)r->cur->n_ramps * 512 * 4))) return rc;
    vb_launch_make_ramps((const RsRamp *)(tmp + o_r), (const RsStop *)(tmp + o_s), r->cur->n_ramps, (uint32_t *)r->cur->ramps.p, st);
    r->cur->atlas_w = atlas_w;
    r->cur->atlas_h = atlas_h;
    if ((rc = ensure(r, r->cur->atlas, (size_t)atlas_w * atlas_h * 4))) return rc;
    CK(cudaMemsetAsync(r->cur->atlas.p, 0, (size_t)atlas_w * atlas_h * 4, st));
    for (size_t i = 0; i < placed.size(); i++) {
        const Placed &q = placed[i];
        if (q.key && q.w && q.h && !from_device[i])
            CK(cudaMemcpy2DAsync((char *)r->cur->atlas.p + ((size_t)q.y * atlas_w + q.x) * 4, (size_t)atlas_w * 4, q.key, (size_t)q.w * 4, (size_t)q.w * 4, q.h,
                                 cudaMemcpyHostToDevice, st));
    }
    if ((rc = enqueue_blits(r, blits, r->cur->atlas.p, atlas_w))) return rc;
    CK(cudaGetLastError());
    // the host vectors above are read by the asynchronous copies: they must outlive them
    CK(cudaStreamSynchronize(st));
    r->cur->overridden = std::move(over);
    r->cur->layout = L;
    r->cur->scene_words = total_words;
    r->cur->have_scene = true;
    r->cells.clear();
    if (layout_out) memcpy(layout_out, &L, sizeof(vb_layout));
    return VB_OK;
}


// ---- multi-GPU exchange set-up (k_exchange.cu) ----------------------------------------------------------------------------
// grow_arenas() is declared above; these entry points only manage the arena and the peer table.
extern "C" int vb_exchange_configure(vb_renderer *r, uint32_t rank, uint32_t world, void **arena, size_t *arena_bytes) {
    if (!r || world < 1u || world > 8u || rank >= world) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    vb_renderer::Exchange &x = r->xc;
    x.enabled = false;
    const uint32_t n_tags = (r->cur->layout.path_data_base - r->cur->layout.path_tag_base) * 4u;
    // my outbox holds my share of the lines (+ the ones needed by two stripes): generous and fixed, so that the arena -- which
    // the peers have mapped -- never moves
    const uint64_t cap = (uint64_t)n_tags * 4u / world * 2u + 262144u;
    x.lines_cap = cap > 0x7fffffffull ? 0x7fffffffu : (uint32_t)cap;
    x.n_paths = r->cur->layout.n_paths;
    x.half_bytes = vb_exchange_half_bytes(x.n_paths, x.lines_cap);
    const size_t bytes = 256 + 2 * x.half_bytes;
    int rc = ensure(r, x.arena, bytes);
    if (rc) return rc;
    CK(cudaMemset(x.arena.p, 0, 256)); // flags and epoch start at 0
    x.rank = rank;
    x.world = world;
    memset(x.peer, 0, sizeof x.peer);
    x.peer[rank] = x.arena.p;
    for (uint32_t i = 0; i <= world; i++) x.rows[i] = 0;
    x.configured = true;
    if (arena) *arena = x.arena.p;
    if (arena_bytes) *arena_bytes = bytes;
    return VB_OK;
}
extern "C" int vb_exchange_attach(vb_renderer *r, uint32_t peer_rank, void *peer_arena) {
    if (!r || !r->xc.configured || peer_rank >= r->xc.world || !peer_arena) return VB_E_INVALID;
    r->xc.peer[peer_rank] = peer_arena;
    return VB_OK;
}
extern "C" int vb_exchange_set_bounds(vb_renderer *r, const uint32_t *tile_rows) {
    if (!r || !r->xc.configured || !tile_rows) return VB_E_INVALID;
    for (uint32_t i = 0; i <= r->xc.world; i++) {
        if (i && tile_rows[i] < tile_rows[i - 1]) return VB_E_INVALID;
        r->xc.rows[i] = tile_rows[i];
    }
    return VB_OK;
}
extern "C" int vb_exchange_enable(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    if (on) {
        if (!r->xc.configured) return VB_E_INVALID;
        for (uint32_t i = 0; i < r->xc.world; i++)
            if (!r->xc.peer[i]) return VB_E_INVALID;
    }
    r->xc.enabled = on != 0;
    return VB_OK;
}
