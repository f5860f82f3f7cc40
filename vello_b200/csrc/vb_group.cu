// vb_group.cu -- one frame on several GPUs: vb_group (tile-row stripes, one host thread), the multi-GPU exchange set-up
// (k_exchange.cu) and the CUDA IPC helpers for one process per GPU.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>

#include "vb_renderer.h"
#include "vb_textures.h"

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
extern "C" int vb_group_set_view(vb_group *g, const double affine[6]) {
    if (!g) return VB_E_INVALID;
    View v;
    if (view_of(affine, &v)) {
        g->err = "vb_group_set_view: the coefficients must be finite in f32";
        return VB_E_INVALID;
    }
    // all renderers or none: on a failure the ones already switched get their earlier view back
    std::vector<View> before;
    for (vb_renderer *r : g->subs) before.push_back(r->view);
    for (size_t i = 0; i < g->subs.size(); i++) {
        const int rc = put_view(g->subs[i], v);
        if (rc) {
            g->err = g->subs[i]->err;
            for (size_t j = 0; j <= i; j++) put_view(g->subs[j], before[j]);
            return rc;
        }
    }
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
    if (vb_texture_key(out_device) || vb_texture_key(host_out)) {
        g->err = "a vb_group renders into plain host or device pointers, not into registered destinations or texture keys";
        return VB_E_INVALID;
    }
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
    // device destination: straight into the frame on devices[0] when peer-mapped; otherwise (and for a host destination) the
    // renderer's own target. Without the exchange a host destination's stripe is copied by the frame itself, on the
    // renderer's copy stream.
    std::vector<Frame> fs;
    for (size_t i = 0; i < n; i++) {
        Frame f = frame_of(g->subs[i], p, Dest{});
        f.params.tile_row0 = g->bounds[i];
        f.params.tile_row1 = g->bounds[i + 1];
        if (!host_out && g->peer_ok[i]) f.dest.dev = (char *)frame + (size_t)g->bounds[i] * 16u * pitch;
        if (host_out && !g->exchange) f.dest.host = (char *)host_out + (size_t)g->bounds[i] * 16u * pitch;
        fs.push_back(f);
    }
    int result = VB_OK;
    for (uint32_t attempt = 0;; attempt++) {
        if (g->exchange)
            for (vb_renderer *r : g->subs) vb_exchange_set_bounds(r, g->bounds.data());
        // renderers that share a device (tests) launch the frame in two submissions: up to and including flatten + the
        // sending half of the exchange, then the rest (see k_exchange.cu)
        const bool halves = g->exchange && g->shared_device;
        // phases: 0 = configs and arenas of every renderer, 1 (and 2) = the launches, last = the read-backs of a host
        // destination. A copy into pageable host memory blocks the host until it is done, so it must not be issued before
        // every renderer's frame has been launched (with the exchange on, a frame waits for its peers).
        const int n_launch = halves ? 2 : 1;
        const bool late_copy = host_out != nullptr && g->exchange; // without the exchange every frame queues its own read-back
        for (int phase = 0; phase < 1 + n_launch + (late_copy ? 1 : 0); phase++) {
            for (size_t i = 0; i < n; i++) {
                vb_renderer *r = g->subs[i];
                if (g->bounds[i + 1] <= g->bounds[i]) continue; // more devices than tile rows (never with the exchange on)
                const size_t row0 = (size_t)g->bounds[i] * 16u;
                int rc = VB_OK;
                if (phase == 0) rc = frame_prepare(r, fs[i]);
                else if (phase <= n_launch)
                    rc = launch(r, phase == 2 ? VB_STAGE_ID_DRAW : 0, halves && phase == 1 ? VB_STAGE_ID_FLATTEN : VB_N_STAGE_IDS - 1);
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
            if (g->bounds[i + 1] <= g->bounds[i]) {
                if (stats) memset(&stats[i], 0, sizeof(vb_frame_stats));
                continue;
            }
            const size_t row0 = (size_t)g->bounds[i] * 16u;
            // a stripe that overflowed is re-run by its renderer alone (first frames); with the exchange on, settle only grows
            // the arenas and the frame is re-issued on EVERY device (epochs advance together)
            int rc = finish(r, fs[i]);
            if (rc == VB_OK) rc = settle(r, fs[i], stats ? &stats[i] : nullptr);
            if (rc == VB_E_BUMP_OVERFLOW && g->exchange) {
                redo = true;
                rc = VB_OK;
            }
            if (stats) stats[i].retries += attempt; // the re-issues of an exchanged frame
            g->ms[i] = vb_last_frame_ms(r);
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
        if (attempt >= g->subs[0]->max_retries) {
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

// ---- multi-GPU exchange set-up (k_exchange.cu) ----------------------------------------------------------------------------
// grow_arenas() is declared above; these entry points only manage the arena and the peer table.
extern "C" int vb_exchange_configure(vb_renderer *r, uint32_t rank, uint32_t world, void **arena, size_t *arena_bytes) {
    if (!r || world < 1u || world > 8u || rank >= world) return VB_E_INVALID;
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    if (r->bg.on) {
        r->err = "vb_exchange_configure: not available for a renderer with a background (vb_set_background)";
        return VB_E_INVALID;
    }
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
