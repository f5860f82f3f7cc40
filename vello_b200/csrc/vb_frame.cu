// vb_frame.cu -- the renderer and its frames: lifetime, arenas, the frame path (prepare, enqueue, whole-frame graphs,
// grow-and-re-run, streaming), views, hit testing and the renderer's settings, in the C ABI of include/vello_b200.h.
//
// Replaces vello/src/render.rs (graph: stage order, bindings, buffer lifetimes) and
// vello/src/wgpu_engine.rs (engine) with a CUDA-stream pipeline. Unlike the reference
// (config.rs:398-408 fixed `1 << 21` arenas; lib.rs:762 "TODO: re-run on overflow") every
// bump-allocated arena is sized from the scene and grown + re-run when a frame overflows.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "vb_device.cuh"
#include "vb_renderer.h"
#include "vb_textures.h"

// path_tiling_setup.wgsl:21-26 flags a failed frame to fine through ptcl[0] = ~0. That word is also tile 0's blend offset
// and is only rewritten when coarse visits tile 0 -- which a stripe window with bin_row0 > 0 never does, so the flag of a
// failed attempt would outlive the successful re-run and every later frame of that renderer. fine therefore reads
// bump.failed (zeroed with the control block at the start of every attempt) directly; ptcl[0] is not used as a flag.

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

int vb_host::ensure(vb_renderer *r, DevBuf &b, size_t bytes) {
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
// Wait for the last copy out of stage s, grow it to `bytes`, and return its host memory in *host.
int vb_host::stage_host(vb_renderer *r, PinnedStage &s, size_t bytes, uint8_t **host) {
    CK(cudaEventSynchronize(s.copied));
    if (s.cap < bytes) {
        if (s.host) CK(cudaFreeHost(s.host));
        s.host = nullptr;
        s.cap = 0;
        CK(cudaMallocHost((void **)&s.host, bytes));
        s.cap = bytes;
    }
    *host = s.host;
    return VB_OK;
}
// The copies out of stage s are enqueued on the renderer's stream: the next stage_host waits for them.
int vb_host::stage_copied(vb_renderer *r, PinnedStage &s) {
    CK(cudaEventRecord(s.copied, r->stream));
    return VB_OK;
}
// Hit testing's record of the frame it answers for (vb_renderer::hit).
void vb_host::hit_forget(vb_renderer *r) {
    r->hit.valid = false;
    r->hit_enq.valid = false;
}
static void hit_enqueued(vb_renderer *r) {
    r->hit.valid = false;
    r->hit_enq.valid = true;
    r->hit_enq.windowed = r->params.bin_row1 > r->params.bin_row0 || r->params.tile_row1 > r->params.tile_row0;
    r->hit_enq.cfg = r->cfg;
    r->hit_enq.bufs = r->bufs;
}
// the frame enqueued last has finished, successfully or not
static void hit_finished(vb_renderer *r, bool ok) {
    r->hit = r->hit_enq;
    r->hit.valid = ok && r->hit_enq.valid;
}

#define FIELD(f) offsetof(VbFrameBufs, f)
const FrameBufDesc vb_host::FRAME_BUFS[N_FRAME_BUFS] = {
    {"tag_monoids", FIELD(tag_monoids), true, [](const FrameCounts &n, bool) { return n.tag_words * sizeof(VbTagMonoid); }},
    {"path_bboxes", FIELD(path_bboxes), true, [](const FrameCounts &n, bool) { return n.paths * sizeof(VbPathBbox); }},
    {"path_draw", FIELD(path_draw), true, [](const FrameCounts &n, bool) { return n.paths * sizeof(uint2); }},
    {"draw_monoids", FIELD(draw_monoids), true, [](const FrameCounts &n, bool) { return n.draws * sizeof(VbDrawMonoid); }},
    {"clip_inp", FIELD(clip_inp), true, [](const FrameCounts &n, bool) { return n.clips * sizeof(VbClipInp); }},
    {"clip_bboxes", FIELD(clip_bboxes), true, [](const FrameCounts &n, bool) { return n.clips * sizeof(VbBbox4); }},
    {"clip_scratch", FIELD(clip_scratch), false, [](const FrameCounts &n, bool) { return vb_clip_scratch_words(n.clips) * 4; }},
    {"draw_bboxes", FIELD(draw_bboxes), true, [](const FrameCounts &n, bool) { return n.draws * sizeof(VbBbox4); }},
    {"bin_headers", FIELD(bin_headers), true,
     [](const FrameCounts &n, bool) { return (size_t)n.draw_parts * n.aligned_bins * sizeof(VbBinHeader); }},
    // allocated in whole partitions; the kernels write and read the first n_draw_objects records, and only those are downloaded
    {"paths", FIELD(paths), true,
     [](const FrameCounts &n, bool download) { return (download ? n.draws : (size_t)n.draw_parts * 256u) * sizeof(VbPath); }},
    {"tile_start", FIELD(tile_start), false, [](const FrameCounts &n, bool) { return ((size_t)n.tiles + 256) * 4; }},
    // fine's cost-ordered tile lists
    {"cls_list", FIELD(cls_list), true, [](const FrameCounts &n, bool) { return (size_t)VB_FINE_LISTS * n.tiles * 8; }},
    {"flatten_parts", FIELD(flatten_parts), false, [](const FrameCounts &n, bool) { return vb_flatten_part_words(n.flatten_parts) * 4; }},
    {"ctl", FIELD(ctl), false, [](const FrameCounts &n, bool) { return n.ctl_words * 4; }},
    // the arenas' buffers, from FB_LINES on
    {"lines", FIELD(lines)},
    {"info_bin_data", FIELD(info_bin_data)},
    {"tiles", FIELD(tiles)},
    {"seg_counts", FIELD(seg_counts)},
    {"segments", FIELD(segments)},
    {"blend_spill", FIELD(blend_spill)},
    {"ptcl", FIELD(ptcl)},
    {"line_scratch", FIELD(line_scratch)},
    {"flatten_jobs", FIELD(flatten_jobs)},
};
#undef FIELD
const ArenaDesc vb_host::ARENAS[N_ARENAS] = {
    {"lines", FB_LINES, sizeof(VbLineSoup), &VbBump::lines},
    {"binning", FB_INFO_BIN_DATA, 4, &VbBump::binning},
    {"tiles", FB_TILES, sizeof(VbTile), &VbBump::tile},
    {"seg_counts", FB_SEG_COUNTS, sizeof(VbSegmentCount), &VbBump::seg_counts},
    {"segments", FB_SEGMENTS, sizeof(VbSegment), &VbBump::segments},
    {"blend", FB_BLEND_SPILL, 4, &VbBump::blend},
    {"ptcl", FB_PTCL, 4, &VbBump::ptcl},
};
int vb_host::arena_index(const char *name) {
    for (int a = 0; a < N_ARENAS; a++)
        if (!strcmp(name, ARENAS[a].name)) return a;
    return -1;
}
// ptcl starts with a static command area of VB_PTCL_INITIAL_ALLOC words per tile; its capacity includes it, bump.ptcl does not
uint64_t vb_host::ptcl_static(const VbConfig &c) { return (uint64_t)c.width_in_tiles * c.tile_rows * VB_PTCL_INITIAL_ALLOC; }
// elements of the arena's buffer in front of the arena: binning lives after the draw info in info_bin_data
size_t vb_host::arena_offset(const vb_renderer *r, int a) { return a == ARENA_BINNING ? r->cur->layout.bin_data_start : 0; }
// what the last attempt asked of an arena, in the units of its capacity
uint64_t vb_host::arena_need(const vb_renderer *r, int a) {
    const uint64_t n = r->cur->h_bump->*ARENAS[a].counter;
    return a == ARENA_PTCL ? ptcl_static(r->cfg) + n : n;
}
// Allocate arena a for its capacity. ptcl gets 512 bytes of slack for fine's 256-byte command windows; the lines capacity
// also sizes flatten's scratch arenas.
int vb_host::ensure_arena(vb_renderer *r, int a) {
    const ArenaDesc &d = ARENAS[a];
    int rc = ensure(r, r->fb[d.buf], (arena_offset(r, a) + r->cap[a]) * d.elem_bytes + (a == ARENA_PTCL ? 512 : 0));
    if (rc || a != ARENA_LINES) return rc;
    size_t lit_bytes, job_bytes;
    vb_flatten_arena_bytes(r->cap[a], &lit_bytes, &job_bytes);
    if ((rc = ensure(r, r->fb[FB_LINE_SCRATCH], lit_bytes))) return rc;
    return ensure(r, r->fb[FB_FLATTEN_JOBS], job_bytes);
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

// The renderer's streams and events, each once, with the flags they are created with: what vb_renderer_new creates and
// vb_renderer_free destroys.
template <class S, class E> static void for_each_handle(vb_renderer *r, S stream, E event) {
    for (cudaStream_t *s : {&r->stream, &r->upload_stream, &r->tiling_stream, &r->copy_stream}) stream(*s);
    for (cudaEvent_t *e : {&r->tiling_fork, &r->tiling_join, &r->draw_fork, &r->draw_join}) event(*e, cudaEventDisableTiming);
    for (PinnedStage &s : r->pinned) event(s.copied, cudaEventDisableTiming);
    for (cudaEvent_t &e : r->upload_done) event(e, cudaEventDisableTiming);
    for (cudaEvent_t &e : r->raster_done) event(e, cudaEventDisableTiming);
    for (cudaEvent_t &e : r->band_ev) event(e, cudaEventDisableTiming);
    for (cudaEvent_t &e : r->copy_done) event(e, cudaEventDisableTiming);
    for (cudaEvent_t &e : r->ev) event(e, cudaEventDefault);
    for (cudaEvent_t &e : r->frame_ev) event(e, cudaEventDefault);
}

// Everything vb_renderer_new creates; on failure vb_renderer_free releases what was created.
static int renderer_init(vb_renderer *r) {
    const cudaError_t e = cudaSetDevice(r->device);
    if (e != cudaSuccess) {
        fprintf(stderr, "vello_b200: cudaSetDevice(%d): %s\n", r->device, cudaGetErrorString(e));
        return VB_E_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, r->device) == cudaSuccess) r->sm_count = prop.multiProcessorCount;
    cudaError_t created = cudaSuccess;
    for_each_handle(
        r, [&](cudaStream_t &s) { if (created == cudaSuccess) created = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); },
        [&](cudaEvent_t &ev, unsigned flags) { if (created == cudaSuccess) created = cudaEventCreateWithFlags(&ev, flags); });
    CK(created);
    for (auto &s : r->slot) {
        CK(cudaHostAlloc((void **)&s.h_bump, sizeof(VbBump), cudaHostAllocMapped));
        CK(cudaHostGetDevicePointer((void **)&s.h_bump_dev, s.h_bump, 0));
        memset(s.h_bump, 0, sizeof(VbBump));
    }
    if (vb_fine_init_constants() != 0) return VB_E_CUDA;
    std::vector<uint32_t> l8, l16;
    make_mask_luts(l8, l16);
    int rc;
    if ((rc = ensure(r, r->mask8, l8.size() * 4)) || (rc = ensure(r, r->mask16, l16.size() * 4))) return rc;
    CK(cudaMemcpy(r->mask8.p, l8.data(), l8.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(r->mask16.p, l16.data(), l16.size() * 4, cudaMemcpyHostToDevice));
    return VB_OK;
}

extern "C" int vb_renderer_new(const vb_options *opt, vb_renderer **out) {
    if (!out) return VB_E_INVALID;
    vb_renderer *r = new vb_renderer();
    r->device = opt ? opt->device : 0;
    r->timing = opt && opt->timing;
    if (opt && opt->max_retries) r->max_retries = opt->max_retries;
    if (getenv("VELLO_B200_NO_GRAPH")) r->use_graph = false;
    const int rc = renderer_init(r);
    if (rc) {
        vb_renderer_free(r);
        return rc;
    }
    *out = r;
    return VB_OK;
}

// Also frees a renderer that vb_renderer_new left partly built: every handle is checked.
extern "C" void vb_renderer_free(vb_renderer *r) {
    if (!r) return;
    cudaSetDevice(r->device);
    if (r->stream) cudaStreamSynchronize(r->stream);
    if (r->tiling_stream) cudaStreamSynchronize(r->tiling_stream);
    for_each_buf(r, [](DevBuf &b) {
        if (b.p) cudaFree(b.p);
    });
    for (auto &s : r->slot)
        if (s.h_bump) cudaFreeHost(s.h_bump);
    for (PinnedStage &s : r->pinned)
        if (s.host) cudaFreeHost(s.host);
    for (auto &f : r->fragments) cudaFree(f.second->mem);
    for (auto &f : r->freed) {
        cudaFree(f.mem);
        cudaEventDestroy(f.done);
    }
    drop_registrations(r);
    if (r->bg.d.surf) cudaDestroySurfaceObject(r->bg.d.surf);
    for (auto &gs : r->graphs)
        if (gs.exec) cudaGraphExecDestroy(gs.exec);
    for_each_handle(
        r, [](cudaStream_t &s) { if (s) cudaStreamDestroy(s); }, [](cudaEvent_t &ev, unsigned) { if (ev) cudaEventDestroy(ev); });
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
// A key given where a host pointer or a plain device pointer is needed: refused, since a key is an inaccessible address.
static int refuse_key(vb_renderer *r, const void *p, const char *who) {
    if (!vb_texture_key(p)) return VB_OK;
    r->err = std::string(who) + ": a texture or destination key is not a host or device pointer here";
    return VB_E_INVALID;
}
extern "C" int vb_copy_to_host(vb_renderer *r, const void *src_device, void *dst_host, size_t bytes) {
    if (!r || !src_device || !dst_host) return VB_E_INVALID;
    if (refuse_key(r, src_device, "vb_copy_to_host") || refuse_key(r, dst_host, "vb_copy_to_host")) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    CK(cudaMemcpyAsync(dst_host, src_device, bytes, cudaMemcpyDeviceToHost, r->stream));
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

// A view set, or transforms, colours or points bound, after the scene's upload: move the current slot's scene into an
// allocation with room for the transforms, draw data and path data frames write. The scene may still be arriving on the
// upload stream, and frames already enqueued read the old allocation.
static int reserve_transform_room(vb_renderer *r, size_t bytes) {
    DevBuf &sc = r->cur->scene;
    if (sc.cap >= bytes) return VB_OK;
    CK(cudaStreamSynchronize(r->upload_stream));
    CK(cudaStreamSynchronize(r->stream));
    DevBuf grown;
    grown.cap = (bytes + 255) & ~(size_t)255;
    CK(cudaMalloc(&grown.p, grown.cap));
    const cudaError_t e = cudaMemcpy(grown.p, sc.p, r->cur->scene_words * 4, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) {
        cudaFree(grown.p);
        r->err = std::string("moving the scene: ") + cudaGetErrorString(e);
        return VB_E_CUDA;
    }
    CK(cudaFree(sc.p));
    sc = grown;
    return VB_OK;
}

extern "C" int vb_readback_wait(vb_renderer *r);
// A non-streaming entry point used while streamed frames are still in flight completes them first.
int vb_host::drain_stream(vb_renderer *r) {
    if (r->stream_pending) return vb_readback_wait(r);
    return VB_OK;
}

uint32_t vb_host::grow(uint32_t need) {
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
    const uint32_t hb = ((p->height + 15u) / 16u + 15u) / 16u, wb = ((p->width + 15u) / 16u + 15u) / 16u;
    // bin_headers: one row of headers per partition of 256 draw objects, each row the bins of every cell rounded up to 256
    const uint64_t draw_parts = (r->cur->layout.n_draw_objects + 255ull) / 256u, aligned_bins = ((uint64_t)wb * hb * n_cells + 255u) & ~255ull;
    if (n_cells > 1u) {
        if (p->bin_row1 > p->bin_row0 || p->tile_row1 > p->tile_row0 || r->xc.enabled || r->grouped) {
            r->err = "batch: cells cannot be combined with bin_row / tile_row windows, vb_group or the exchange";
            return VB_E_INVALID;
        }
        if ((uint64_t)hb * n_cells * 2u > 65535u || draw_parts * aligned_bins >= 0xffffffffull) {
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
    // bound gradient stops: the frame reads the binding's ramps, the scene's and then one row per bound gradient
    const VbBound &B = r->bound;
    if (B.rows[VB_BIND_STOPS].rows) c.n_ramps = B.rs_ramp0 + B.rs_grads_n;
    c.atlas_w = r->cur->atlas_w;
    c.atlas_h = r->cur->atlas_h;
    c.out_pitch_px = p->width;
    c.out_row0 = c.win_ty0 * 16u;
    // The frame reads its transforms, draw data and path data from the regions past the scene's streams that it writes itself
    // (regions_of): the bound transforms from the caller's instance rows and transform rows, the viewed transforms from the
    // transforms before them (view_src; the region is empty for a layout whose transforms do not lie inside the uploaded words),
    // the draw data from the scene's, the colour rows, the bound gradients' ramp rows and the opacity rows, the path data from
    // the scene's and the point rows. Reserving them can move the scene.
    const bool bound_xf = B.rows[VB_BIND_INSTANCES].rows || B.rows[VB_BIND_TRANSFORMS].rows;
    const Regions g = regions_of(r->cur->layout, r->cur->scene_words, bound_xf, r->view.on, draw_data_bound(B),
                                 B.rows[VB_BIND_POINTS].rows != nullptr);
    if (bound_xf) c.layout.transform_base = (uint32_t)g.base[REGION_BOUND_XF];
    if (r->view.on) {
        c.view_src = c.layout.transform_base;
        c.layout.transform_base = (uint32_t)g.base[REGION_VIEW];
        c.frame_cull = 1u;
    }
    if (draw_data_bound(B)) c.layout.draw_data_base = (uint32_t)g.base[REGION_DRAW_DATA];
    if (B.rows[VB_BIND_POINTS].rows) c.layout.path_data_base = (uint32_t)g.base[REGION_PATH_DATA];
    c.scene_words = (uint32_t)g.words;
    if (int rc0 = reserve_transform_room(r, g.bytes)) return rc0; // nothing to do without regions: installations allocate as much
    c.n_cells = n_cells;
    c.tile_rows = c.height_in_tiles * n_cells;
    c.cell_draw = n_cells > 1u ? (const uint32_t *)r->cell_draw.p : nullptr;
    c.vis = B.rows[VB_BIND_VISIBILITY].rows ? (const uint32_t *)r->vis_mask.p : nullptr; // the mask k_draw_visibility writes
    c.widths = B.rows[VB_BIND_WIDTHS].rows ? (const float *)r->width_snap.p : nullptr; // the snapshot k_stroke_widths writes
    r->params = *p;

    const uint32_t n_draw = c.layout.n_draw_objects, n_tiles = c.width_in_tiles * c.tile_rows;
    int rc;

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
    // flatten: [0] literal-record counter (k_flatten's partitions only; the lean ones write their lines in place, k_flatten_emit),
    // [1] job counter, [2] work-list length, [4..] look-back state of its partition scan
    const size_t o_flatten = off;
    off += 4 + vb_lookback_words((b.parts_flatten + 8191u) / 8192u, 1);
    const size_t o_draw = off; off += vb_lookback_words(b.parts_draw, 4);
    const size_t o_tile = off; off += vb_lookback_words(b.parts_tile, 1);
    const size_t o_clip = off; off += vb_lookback_words(vb_clip_parts(c.layout.n_clips), 1);
    const size_t o_backdrop = off; off += vb_lookback_words(b.parts_backdrop, 3);
    b.ctl_words = off;

    // the fixed-size intermediates (FRAME_BUFS)
    r->counts = {c.n_tag_words, c.layout.n_paths, n_draw, c.layout.n_clips, n_tiles, (uint32_t)draw_parts, (uint32_t)aligned_bins,
                 b.parts_flatten, b.ctl_words};
    for (int i = 0; i < N_FIXED_BUFS; i++)
        if ((rc = ensure(r, r->fb[i], FRAME_BUFS[i].bytes(r->counts, false)))) return rc;

    // every buffer has its size: the launchers' view of them
    for (int i = 0; i < N_FRAME_BUFS; i++) memcpy((char *)&b + FRAME_BUFS[i].field, &r->fb[i].p, sizeof(void *));
    b.scene = (const uint32_t *)r->cur->scene.p;
    b.ramps = (const uint32_t *)r->cur->ramps.p;
    b.atlas = (const uint8_t *)r->cur->atlas.p;
    b.mask8 = (const uint32_t *)r->mask8.p;
    b.mask16 = (const uint32_t *)r->mask16.p;
    b.view = r->view.on ? (const float *)r->view_coef.p : nullptr;
    // the bindings, and what depends on where the scene lives now: the regions' sources and lengths, the bound gradients' ramps
    b.bound = B;
    if (draw_data_bound(B)) b.dd_src = b.scene + r->cur->layout.draw_data_base;
    if (B.rows[VB_BIND_POINTS].rows) b.pt_src = b.scene + r->cur->layout.path_data_base;
    if (B.rows[VB_BIND_TRANSFORMS].rows) b.xf_src = b.scene + r->cur->layout.transform_base;
    if (B.rows[VB_BIND_STOPS].rows) b.ramps = (const uint32_t *)r->stop_ramps.p;
    b.xf_len = (uint32_t)(std::max(g.len[REGION_BOUND_XF], g.len[REGION_VIEW]) / 6u); // the two are as long when both are present
    b.dd_len = (uint32_t)g.len[REGION_DRAW_DATA];
    b.pd_len = (uint32_t)g.len[REGION_PATH_DATA];
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

FineRows vb_host::fine_rows(const VbConfig &c, const Dest &d) {
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
        if (last >= VB_STAGE_ID_FINE) CK(cudaMemsetAsync(b.ctl + VB_CTL_FINE_QUEUE, 0, 9 * sizeof(uint32_t), st)); // and the flagged queue
        if (first <= VB_STAGE_ID_COARSE && last >= VB_STAGE_ID_COARSE)
            CK(cudaMemsetAsync(b.ctl + VB_CTL_FINE_CLASS, 0, VB_FINE_LISTS * sizeof(uint32_t), st));
        if (first <= VB_STAGE_ID_BACKDROP && last >= VB_STAGE_ID_BACKDROP)
            CK(cudaMemsetAsync(b.lb_backdrop, 0, VB_LB_ZERO_WORDS(b.parts_backdrop) * sizeof(uint32_t), st));
    }
    // path_tiling and coarse both depend on backdrop only (it assigns the segment slices): path_tiling is forked onto the
    // tiling stream and joined again before the next stage, so the two kernels share the GPU. Launch counts are unchanged;
    // with per-stage timing on, the stages stay serial so that each one's events time it alone.
    const bool fork_tiling = !r->timing && first <= VB_STAGE_ID_COARSE && last >= VB_STAGE_ID_PATH_TILING;
    // draw reads pathtag's path table and the transforms, not flatten's output, and clip's depth scan and links read only
    // draw's clip inputs: they are forked onto the tiling stream once the transforms are written, beside flatten, and
    // joined before clip's boxes (which read the path boxes). Launch counts are unchanged. Serial with per-stage timing, with
    // the exchange (draw waits for its second half) and for partial ranges: only whole frames fork, whose fine may follow
    // separately (a host destination's bands after the captured graph).
    const bool fork_draw = !r->timing && !r->xc.enabled && first == VB_STAGE_ID_PATHTAG && last >= VB_STAGE_ID_FINE - 1;
    rec(r, 0);
    for (int s = first; s <= last; s++) {
        switch (s) {
        case VB_STAGE_ID_PATHTAG: launches += vb_launch_pathtag(c, b, st); break;
        case VB_STAGE_ID_FLATTEN: {
            // with the exchange on, this GPU flattens its share of the tag stream (no stripe culling: the lines are for
            // everybody), then the lines and path boxes are exchanged through peer memory (k_exchange.cu)
            // first, inside flatten's stage events, what the bindings (VbBound) and the view make of the scene: the regions past
            // its streams in regions_of's order, the bound transforms before the viewed ones (their source; instances, then
            // transform rows), the draw data (read by draw, coarse and fine) and the path data (read by flatten alone); the bound
            // gradients' ramp rows (read by fine); the visibility mask and the stroke widths' snapshot (read by flatten and
            // damage tracking). Each launcher launches nothing while its binding is unbound.
            launches += vb_launch_instance_transforms(c, b, st);
            launches += vb_launch_bound_transforms(c, b, st);
            if (r->view.on) launches += vb_launch_view_transforms(c, b, st);
            launches += vb_launch_draw_data(c, b, st);
            launches += vb_launch_bound_ramps(c, b, st);
            launches += vb_launch_path_points(c, b, st);
            launches += vb_launch_draw_visibility(c, b, st);
            launches += vb_launch_stroke_widths(c, b, st);
            if (fork_draw) {
                CK(cudaEventRecord(r->draw_fork, st));
                CK(cudaStreamWaitEvent(r->tiling_stream, r->draw_fork, 0));
                launches += vb_launch_draw(c, b, r->tiling_stream);
                launches += vb_launch_clip_links(c, b, r->tiling_stream);
                CK(cudaEventRecord(r->draw_join, r->tiling_stream));
            }
            VbConfig cf = c;
            uint32_t p0 = 0u, p1 = b.parts_flatten;
            if (r->xc.enabled) {
                cf.win_cull = 0u;
                cf.frame_cull = 0u;
                const uint32_t P = b.parts_flatten, G = r->xc.world, k = r->xc.rank;
                p0 = (uint32_t)((uint64_t)P * k / G) & ~7u;
                p1 = k + 1u == G ? P : ((uint32_t)((uint64_t)P * (k + 1u) / G) & ~7u);
            }
            launches += vb_launch_flatten(cf, b, first != 0, p0, p1, st);
            if (r->xc.enabled) launches += vb_launch_exchange_send(c, b, X, st);
            break;
        }
        case VB_STAGE_ID_DRAW:
            // a range that starts here writes them again: the kernels only read the scene's own and the caller's rows, so the
            // words are the same
            if (first == VB_STAGE_ID_DRAW) launches += vb_launch_instance_transforms(c, b, st);
            if (first == VB_STAGE_ID_DRAW) launches += vb_launch_bound_transforms(c, b, st);
            if (r->view.on && first == VB_STAGE_ID_DRAW) launches += vb_launch_view_transforms(c, b, st);
            if (first == VB_STAGE_ID_DRAW) launches += vb_launch_draw_data(c, b, st);
            if (first == VB_STAGE_ID_DRAW) launches += vb_launch_bound_ramps(c, b, st);
            if (r->xc.enabled) // second half of the exchange: my lines and the complete path boxes arrive before draw_leaf reads them
                launches += vb_launch_exchange_recv(c, b, X, st);
            if (fork_draw) CK(cudaStreamWaitEvent(st, r->draw_join, 0)); // launched beside flatten
            else launches += vb_launch_draw(c, b, st);
            break;
        case VB_STAGE_ID_CLIP:
            if (!fork_draw) launches += vb_launch_clip_links(c, b, st); // else launched beside flatten
            launches += vb_launch_clip_bboxes(c, b, st);
            break;
        case VB_STAGE_ID_BINNING: launches += vb_launch_binning(c, b, st); break;
        case VB_STAGE_ID_TILE_ALLOC: launches += vb_launch_tile_alloc(c, b, st); break;
        case VB_STAGE_ID_PATH_COUNT: launches += vb_launch_path_count(c, b, st); break;
        case VB_STAGE_ID_BACKDROP: launches += vb_launch_backdrop(c, b, st); break;
        case VB_STAGE_ID_COARSE:
            // damage tracking: the frame's damaged tiles, from binning's draw boxes, before coarse reads them
            launches += vb_launch_damage(c, b, st);
            // the first frame after an upload that tracking follows: which draw objects the upload changed, as the tables
            // that k_recompose_damage reads
            launches += vb_launch_upload_diff(c, b, st);
            launches += vb_launch_recompose_damage(c, b, st); // the first frame after vb_recompose: what the recompose changed
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
                launches += vb_launch_fine(cb, b, d.out, d.bg, (int)r->params.aa, r->occlusion_cull, band, f.bands == 1u, st);
                if (d.host && (rc = queue_readback(r, c, f, band, d))) return rc;
            }
            break;
        }
        default: return VB_E_INVALID;
        }
        rec(r, s + 1);
    }
    if (last == VB_STAGE_ID_FINE) launches += vb_launch_damage_commit(c, b, st); // after fine: the frame's success is known
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
static void graph_key(vb_renderer *r, int last, const Dest &d, GraphKey *k) {
    memset(k, 0, sizeof *k);
    k->cfg = r->cfg;
    memcpy(&k->bufs, &r->bufs, sizeof k->bufs);
    k->bg = d.bg;
    k->out = d.dev;
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
    graph_key(r, g_last, d, &key);
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
        r->graph_captures++;
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

// The frame's device destination: a registered destination's key, the given pointer, or the renderer's own target (allocated
// for this frame's window).
static int pick_out(vb_renderer *r, Dest *d) {
    if (vb_texture_key(d->dev)) return resolve_destination(r, d);
    int rc = VB_OK;
    if (!d->dev) {
        const VbConfig &c = r->cfg;
        DevBuf &t = d->alt ? r->target_alt : r->target;
        rc = ensure(r, t, (size_t)c.out_pitch_px * 4u * fine_rows(c, *d).dest_rows);
        d->dev = t.p;
    }
    d->out = VbFineOut{};
    d->out.out = (uint32_t *)d->dev;
    return rc;
}

// A frame is enqueued in two steps: everything that may allocate, free or otherwise synchronise with the device (config,
// arenas, the output target), then the launches. vb_group runs step 1 for ALL its renderers before step 2 of any: with the
// exchange on, a renderer's frame contains a kernel that waits for its peers, and a peer that shares the device (tests)
// must not be stuck in a cudaFree behind that kernel.
int vb_host::frame_prepare(vb_renderer *r, const Frame &f) {
    if (!r) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    CK(cudaSetDevice(r->device));
    int rc = prepare(r, &f.params);
    if (rc) return rc;
    r->dest = f.dest;
    if ((rc = pick_out(r, &r->dest)) || (rc = resolve_background(r, f.bg, &r->dest))) return rc;
    return damage_prepare(r);
}
// Enqueue stages first..last of the frame frame_prepare set up. A range from stage 0 starts the frame: the dirty overridden
// images are copied and the hit record and the frame's first event are taken. A range after stage 0 continues the frame and
// adds to its launches. A range that ends at fine completes it: the frame's last event, and the frame is pending.
int vb_host::launch(vb_renderer *r, int first, int last) {
    CK(cudaSetDevice(r->device));
    const uint32_t before = r->launches;
    int rc;
    if (first == 0) {
        if ((rc = refresh_overrides(r))) return rc;
        CK(cudaEventRecord(r->frame_ev[0], r->stream));
        hit_enqueued(r);
    }
    rc = enqueue(r, first, last, r->dest, false);
    if (first != 0) r->launches += before;
    if (rc != VB_OK) hit_forget(r); // a frame enqueued in part
    if (last == VB_N_STAGE_IDS - 1) {
        if (rc == VB_OK) CK(cudaEventRecord(r->frame_ev[1], r->stream));
        r->frame_timed = rc == VB_OK;
        r->frame_pending = rc == VB_OK;
    }
    return rc;
}

// A frame of the renderer's current scene slot, under its current view and over its current background.
Frame vb_host::frame_of(const vb_renderer *r, const vb_params *p, const Dest &d) {
    return Frame{*p, d, r->view, r->bg, (uint32_t)(r->cur - r->slot)};
}

static bool same_view(const View &a, const View &b) { return a.on == b.on && (!a.on || memcmp(a.m, b.m, sizeof a.m) == 0); }
// Enqueue frame f from its scene slot and under its view; the renderer's current slot and view are restored afterwards.
static int issue(vb_renderer *r, const Frame &f) {
    vb_renderer::SceneSlot *const keep = r->cur;
    const View now = r->view;
    const bool other = !same_view(now, f.view);
    r->cur = &r->slot[f.slot];
    int rc = other ? put_view(r, f.view) : VB_OK;
    if (rc == VB_OK) rc = frame_prepare(r, f);
    if (rc == VB_OK) rc = launch(r, 0, VB_N_STAGE_IDS - 1);
    if (other) {
        const int rc2 = put_view(r, now);
        if (rc == VB_OK) rc = rc2;
    }
    r->cur = keep;
    return rc;
}

extern "C" int vb_render_enqueue(vb_renderer *r, const vb_params *p, void *out_device) {
    if (!r || !p) return VB_E_INVALID;
    return issue(r, frame_of(r, p, Dest{out_device}));
}

static void fill_stats(vb_renderer *r, vb_frame_stats *s, uint32_t retries) {
    if (!s) return;
    memset(s, 0, sizeof *s);
    memcpy(s, r->cur->h_bump, sizeof(VbBump));
    s->retries = retries;
    s->kernel_launches = r->launches;
    for_each_buf(r, [&](DevBuf &b) { s->arena_bytes += b.cap; });
    s->arena_bytes += r->fragment_bytes;
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
    fill_stats(r, stats, 0u); // an enqueued frame is not re-run
    hit_finished(r, r->cur->h_bump->failed == 0u);
    if (r->cur->h_bump->failed == 0u) damage_succeeded(r);
    return r->cur->h_bump->failed ? VB_E_BUMP_OVERFLOW : VB_OK;
}

// Wait for frame f, issued last, and for its read-back when it has a host destination.
int vb_host::finish(vb_renderer *r, const Frame &f) {
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    r->frame_pending = false;
    // the band copies were queued behind the fine bands; a re-run after an arena overflow simply copies again
    if (f.dest.host) CK(cudaStreamSynchronize(r->copy_stream));
    return VB_OK;
}
// Issue frame f and wait for it (for the band copies of a frame enqueued in part too).
static int run(vb_renderer *r, const Frame &f) {
    const int rc = issue(r, f);
    const int rc2 = finish(r, f);
    return rc ? rc : rc2;
}

// The grow-and-re-run loop of every entry point. Frame f has finished an attempt (r->cur is its scene slot); while the
// attempt overflowed, grow the arenas and run f again, at most max_retries times. Then report f in *stats.
int vb_host::settle(vb_renderer *r, const Frame &f, vb_frame_stats *stats) {
    uint32_t retries = 0;
    while (r->cur->h_bump->failed != 0u) {
        hit_finished(r, false);
        if (r->xc.enabled) {
            // every attempt of an exchanged frame is a collective step (all GPUs advance their epoch together): grow what
            // overflowed here and let the caller re-issue the frame on every GPU
            grow_arenas(r);
            fill_stats(r, stats, retries);
            r->err = "bump overflow in an exchanged frame: re-issue the frame on every GPU";
            return VB_E_BUMP_OVERFLOW;
        }
        if (retries >= r->max_retries) {
            fill_stats(r, stats, retries);
            r->err = "bump overflow persisted";
            return VB_E_BUMP_OVERFLOW;
        }
        grow_arenas(r);
        retries++;
        const int rc = run(r, f);
        if (rc) return rc;
    }
    fill_stats(r, stats, retries);
    hit_finished(r, true);
    damage_succeeded(r);
    return VB_OK;
}

// One frame, after the streamed frames still in flight, re-run with grown arenas until it fits.
static int render_sync(vb_renderer *r, const vb_params *p, const Dest &d, vb_frame_stats *stats) {
    int rc = drain_stream(r);
    if (rc) return rc;
    const Frame f = frame_of(r, p, d);
    rc = run(r, f);
    return rc ? rc : settle(r, f, stats);
}

extern "C" int vb_render_resident(vb_renderer *r, const vb_params *p, void *out_device, vb_frame_stats *stats) {
    if (!r || !p) return VB_E_INVALID;
    return render_sync(r, p, Dest{out_device}, stats);
}

extern "C" int vb_render_uploaded(vb_renderer *r, const vb_params *p, void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    if (!r || !p || !out) return VB_E_INVALID;
    if (!out_is_device && refuse_key(r, out, "vb_render_uploaded")) return VB_E_INVALID;
    return render_sync(r, p, out_is_device ? Dest{out} : Dest{nullptr, out, false, r->readback_bands}, stats);
}

extern "C" int vb_render(vb_renderer *r, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                         uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, const vb_params *p,
                         void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    if (!r || !p || !out) return VB_E_INVALID;
    if (!out_is_device && refuse_key(r, out, "vb_render")) return VB_E_INVALID;
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

// Frame in ring entry q: wait for its kernels, look at its bump counters, re-run on overflow (together with the younger frame
// enqueued behind it, ring entry `younger`, or -1).
static int check_raster(vb_renderer *r, uint32_t q, int younger) {
    vb_renderer::RingFrame &f = r->ring[q];
    if (!f.pending || f.raster_checked) return VB_OK;
    vb_renderer::SceneSlot *const keep = r->cur;
    CK(cudaEventSynchronize(r->raster_done[f.frame.slot]));
    r->cur = &r->slot[f.frame.slot];
    int rc = VB_OK;
    if (r->cur->h_bump->failed != 0u) {
        CK(cudaStreamSynchronize(r->stream));
        CK(cudaStreamSynchronize(r->copy_stream));
        rc = settle(r, f.frame, &f.stats);
        CK(cudaEventRecord(r->copy_done[q], r->copy_stream));
        vb_renderer::RingFrame *const y = younger >= 0 ? &r->ring[younger] : nullptr;
        if (rc == VB_OK && y && y->pending) {
            r->cur = &r->slot[y->frame.slot];
            if (r->cur->h_bump->failed != 0u) {
                rc = settle(r, y->frame, &y->stats);
                CK(cudaEventRecord(r->raster_done[y->frame.slot], r->stream));
                CK(cudaEventRecord(r->copy_done[younger], r->copy_stream));
                y->raster_checked = true; // its stats are the re-run's
            }
        }
    } else {
        fill_stats(r, &f.stats, 0u);
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
    if (refuse_key(r, out_host, "vb_render_begin")) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    if (stats) memset(stats, 0, sizeof *stats);
    const uint64_t k = r->stream_seq;
    const uint32_t slot = (uint32_t)(k & 1u), q = (uint32_t)(k % 3u), q1 = (uint32_t)((k + 2u) % 3u), q2 = (uint32_t)((k + 1u) % 3u);
    // frame k-2 (same scene slot, same device target) was checked by the previous call; frame k-3 (ring entry q) is complete
    r->cur = &r->slot[slot];
    int rc = upload_on(r, r->upload_stream, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h, false);
    if (rc) return rc;
    CK(cudaEventRecord(r->upload_done[slot], r->upload_stream));
    CK(cudaStreamWaitEvent(r->stream, r->upload_done[slot], 0));
    if (k >= 2u && r->ring[q2].pending) CK(cudaStreamWaitEvent(r->stream, r->copy_done[q2], 0)); // its read-back still reads this target
    // one band: the whole read-back overlaps the next frames, no reason to split fine
    const Frame f = frame_of(r, p, Dest{nullptr, out_host, slot != 0u, 1u});
    rc = issue(r, f);
    if (rc) return rc;
    r->frame_pending = false;
    CK(cudaEventRecord(r->raster_done[slot], r->stream));
    CK(cudaEventRecord(r->copy_done[q], r->copy_stream));
    r->ring[q].pending = true;
    r->ring[q].raster_checked = false;
    r->ring[q].frame = f;
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
    const bool streamed = r->stream_pending;
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
    // the intermediates hold the frame enqueued last (a re-run after an overflow is enqueued anew)
    if (streamed) hit_finished(r, rc == VB_OK);
    return rc;
}

extern "C" int vb_run_stages(vb_renderer *r, const vb_params *p, int first, int last, void *out_device) {
    if (!r || !p || first < 0 || last >= VB_N_STAGE_IDS || first > last) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    hit_forget(r);
    r->dmg.diff.armed = false; // the stages may write the destination: the frame after them is full
    CK(cudaSetDevice(r->device));
    int rc = prepare(r, p);
    if (rc) return rc;
    Dest d{out_device};
    if ((last == VB_STAGE_ID_FINE || vb_texture_key(d.dev)) && (rc = pick_out(r, &d))) return rc;
    if (last == VB_STAGE_ID_FINE && (rc = resolve_background(r, r->bg, &d))) return rc;
    if ((rc = enqueue(r, first, last, d, true))) return rc;
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

// ---- hit testing: vb_hit_test, vb_hit_map ---------------------------------------------------------------------------------
// The answers read the buffers of the frame recorded in r->hit (k_hit.cu); nothing of the frame is written, launched or
// captured, so kernel_launches, the graph key and the next frame are the same with or without hit tests or maps in between.
bool vb_host::device_memory_of(vb_renderer *r, const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeManaged || (a.type == cudaMemoryTypeDevice && a.device == r->device);
}
// The renderer's state checks both calls make, in this order, with `fn` naming the call in vb_last_error.
static int hit_state(vb_renderer *r, const char *fn) {
    auto bad = [&](const char *why) {
        r->err = std::string(fn) + ": " + why;
        return VB_E_INVALID;
    };
    if (r->grouped || r->xc.enabled) return bad("not available for a renderer of a vb_group or with the exchange enabled");
    if (r->frame_pending || r->stream_pending) return bad("a frame is in flight (finish it with vb_frame_finish / vb_readback_wait)");
    if (!r->hit.valid) {
        r->err = std::string(fn) + ": no successful frame since the last scene upload, vb_set_cells, vb_run_stages or vb_debug_* call";
        return VB_E_NO_SCENE;
    }
    if (r->hit.windowed) return bad("the last frame had a bin_row / tile_row window");
    return VB_OK;
}
extern "C" int vb_hit_test(vb_renderer *r, const float *xy, uint32_t n, int32_t *draw_ix, uint32_t on_device) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const char *why) {
        r->err = std::string("vb_hit_test: ") + why;
        return VB_E_INVALID;
    };
    if (n == 0u) return VB_OK;
    if (!xy || !draw_ix) return bad("NULL points or answers");
    if (int rc = hit_state(r, "vb_hit_test")) return rc;
    CK(cudaSetDevice(r->device));
    if (on_device) {
        if (!device_memory_of(r, xy) || !device_memory_of(r, draw_ix)) return bad("on_device: the pointers must be memory of the renderer's device");
        vb_launch_hit_test(r->hit.cfg, r->hit.bufs, xy, n, draw_ix, r->stream);
        CK(cudaGetLastError());
        return VB_OK;
    }
    const size_t xy_bytes = (size_t)n * 2u * sizeof(float);
    int rc = ensure(r, r->hit_io, xy_bytes + (size_t)n * sizeof(int32_t));
    if (rc) return rc;
    float *d_xy = (float *)r->hit_io.p;
    int32_t *d_ix = (int32_t *)((char *)r->hit_io.p + xy_bytes);
    CK(cudaMemcpyAsync(d_xy, xy, xy_bytes, cudaMemcpyHostToDevice, r->stream));
    vb_launch_hit_test(r->hit.cfg, r->hit.bufs, d_xy, n, d_ix, r->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(draw_ix, d_ix, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, r->stream));
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}
extern "C" int vb_hit_map(vb_renderer *r, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, int32_t *draw_ix, size_t pitch_bytes,
                          uint32_t on_device) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const char *why) {
        r->err = std::string("vb_hit_map: ") + why;
        return VB_E_INVALID;
    };
    if (w == 0u || h == 0u) return VB_OK;
    if (!draw_ix) return bad("NULL answers");
    if (int rc = hit_state(r, "vb_hit_map")) return rc;
    const VbConfig &cfg = r->hit.cfg;
    if ((uint64_t)x0 + w > cfg.target_width || (uint64_t)y0 + h > (uint64_t)cfg.n_cells * cfg.target_height)
        return bad("the rectangle does not lie inside the last frame");
    const size_t row = (size_t)w * sizeof(int32_t);
    if (pitch_bytes % sizeof(int32_t) != 0u || pitch_bytes < row) return bad("pitch_bytes must be a multiple of 4 and at least 4 * w");
    if ((size_t)(h - 1u) > (SIZE_MAX - row) / pitch_bytes) return bad("the rows do not fit in the address space");
    CK(cudaSetDevice(r->device));
    if (on_device) {
        if (!device_memory_of(r, draw_ix)) return bad("on_device: draw_ix must be memory of the renderer's device");
        vb_launch_hit_map(cfg, r->hit.bufs, x0, y0, w, h, draw_ix, pitch_bytes, r->stream);
        CK(cudaGetLastError());
        return VB_OK;
    }
    int rc = ensure(r, r->hit_io, row * h);
    if (rc) return rc;
    int32_t *d_ix = (int32_t *)r->hit_io.p;
    vb_launch_hit_map(cfg, r->hit.bufs, x0, y0, w, h, d_ix, row, r->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpy2DAsync(draw_ix, pitch_bytes, d_ix, row, row, h, cudaMemcpyDeviceToHost, r->stream));
    CK(cudaStreamSynchronize(r->stream));
    return VB_OK;
}

// ---- views: vb_set_view --------------------------------------------------------------------------------------------------
// Make v the view of the frames enqueued from now on: its coefficients are written on the renderer's stream, behind every
// frame already enqueued, so those keep theirs. Setting or clearing a view changes the frame's config (and the graph key);
// changing the coefficients does not.
int vb_host::put_view(vb_renderer *r, const View &v) {
    CK(cudaSetDevice(r->device));
    r->view = v;
    if (!v.on) { // no view: nothing of it stays (frames already enqueued may still read the coefficients)
        if (r->view_coef.p) {
            CK(cudaStreamSynchronize(r->stream));
            CK(cudaFree(r->view_coef.p));
            r->view_coef = DevBuf{};
        }
        return VB_OK;
    }
    int rc = ensure(r, r->view_coef, 6 * sizeof(float));
    if (rc) return rc;
    vb_launch_view_set((float *)r->view_coef.p, v.m, r->stream);
    CK(cudaGetLastError());
    return VB_OK;
}
int vb_host::view_of(const double *affine, View *v) {
    v->on = affine != nullptr;
    for (int k = 0; v->on && k < 6; k++) {
        v->m[k] = (float)affine[k]; // Transform::from_kurbo
        if (!isfinite(v->m[k])) return VB_E_INVALID;
    }
    return VB_OK;
}
extern "C" int vb_set_view(vb_renderer *r, const double affine[6]) {
    if (!r) return VB_E_INVALID;
    View v;
    if (view_of(affine, &v)) {
        r->err = "vb_set_view: the coefficients must be finite in f32";
        return VB_E_INVALID;
    }
    if (!same_view(r->view, v)) r->dmg.epoch++;
    return put_view(r, v);
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
