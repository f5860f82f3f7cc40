// vb_renderer.h -- the renderer's host state (struct vb_renderer) and the helpers its host files share. Internal to the library.
//
// The host code is split by concern: vb_frame.cu (renderer lifetime, arenas, the frame path, views, hit testing), vb_upload.cu
// (scene uploads, the device resolve, image overrides and textures, cells), vb_compose.cu (fragments, compose, recompose, and the
// bindings to device rows: VbBound, one bind path for every kind), vb_damage.cu (damage tracking), vb_debug.cu (debug downloads
// and uploads) and vb_group.cu (vb_group, the exchange, CUDA IPC). Each helper declared at the end is defined in one of them. They live in
// namespace vb_host, hidden from the shared library's symbol table, so that a host program's own functions of the same names
// cannot interpose on them.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/vello_b200.h"
#include "vb_stages.h"
#include "vb_types.h"

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0; // bytes
};

// Pinned host memory that tables reach the device through (stage_host / stage_copied). It is rewritten only once the last
// copy out of it has run.
struct PinnedStage {
    uint8_t *host = nullptr;
    size_t cap = 0;                 // bytes
    cudaEvent_t copied = nullptr;   // the last copy out of host
};
// The renderer's stages: the rectangles of k_atlas_blit, and the tables of compose and bind. They are separate because compose
// enqueues its blits while its own tables are still being copied.
enum { PIN_BLITS, PIN_COMPOSE, N_PINNED };

// the seven bump-allocated arenas, in the order of VbConfig::lines_size .. ptcl_size (ARENAS below)
enum { ARENA_LINES, ARENA_BINNING, ARENA_TILES, ARENA_SEG_COUNTS, ARENA_SEGMENTS, ARENA_BLEND, ARENA_PTCL, N_ARENAS };
static_assert(offsetof(VbConfig, ptcl_size) - offsetof(VbConfig, lines_size) == (N_ARENAS - 1) * sizeof(uint32_t),
              "VbConfig's arena sizes are consecutive words in ARENA_* order");

// The device buffers prepare sizes for each frame, in vb_renderer::fb (FRAME_BUFS below): the fixed-size intermediates, then
// the bump arenas' buffers (ARENAS) and flatten's two scratch arenas, which ensure_arena sizes.
enum {
    FB_TAG_MONOIDS, FB_PATH_BBOXES, FB_PATH_DRAW, FB_DRAW_MONOIDS, FB_CLIP_INP, FB_CLIP_BBOXES, FB_CLIP_SCRATCH, FB_DRAW_BBOXES,
    FB_BIN_HEADERS, FB_PATHS, FB_TILE_START, FB_CLS_LIST, FB_FLATTEN_PARTS, FB_CTL, N_FIXED_BUFS,
    FB_LINES = N_FIXED_BUFS, FB_INFO_BIN_DATA, FB_TILES, FB_SEG_COUNTS, FB_SEGMENTS, FB_BLEND_SPILL, FB_PTCL, FB_LINE_SCRATCH,
    FB_FLATTEN_JOBS, N_FRAME_BUFS
};
// The counts the fixed-size intermediates of a frame are sized from, set by prepare (vb_renderer::counts).
struct FrameCounts {
    uint32_t tag_words, paths, draws, clips, tiles;
    uint32_t draw_parts;    // partitions of 256 draw objects (binning's and tile_alloc's)
    uint32_t aligned_bins;  // the bins of every cell, rounded up to 256: a partition's stride in bin_headers
    uint32_t flatten_parts; // VbFrameBufs::parts_flatten
    size_t ctl_words;       // VbFrameBufs::ctl_words: the control block, look-back states included
};

// Where a frame's pixels go: a device pointer, a registered destination's key, or the renderer's own target (target_alt when
// `alt`), and optionally a copy of the frame in host memory, read back in `bands` row bands while fine runs. `out` is where
// fine stores, set from `dev` for each attempt by pick_out (dev itself stays the identity of the destination: the graph key's
// and damage tracking's).
struct Dest {
    void *dev = nullptr, *host = nullptr;
    bool alt = false;
    uint32_t bands = 1;
    VbFineOut out{};
    VbFineBg bg{}; // what fine's tiles start from: the frame's background, set for each attempt by resolve_background
};

// A registered destination (vb_register_destination), found by its key in vb_renderer::dests. LINEAR: pixel (x, y) of a frame
// at ptr + y * pitch + texel() * x. ARRAY: at texel (x + x0, y + y0) of a w x h array, written through surf. `format` is the
// texel format alone; `premul` is VB_DEST_PREMULTIPLIED.
struct Destination {
    uint32_t kind = VB_DEST_LINEAR, format = VB_DEST_RGBA8;
    bool premul = false;
    uint32_t texel() const { return format == VB_DEST_RGBA32F ? 16u : format == VB_DEST_RGBA16F ? 8u : 4u; } // bytes
    uint8_t *ptr = nullptr;
    size_t pitch = 0;
    cudaSurfaceObject_t surf = 0;
    uint32_t x0 = 0, y0 = 0;
    size_t w = 0, h = 0;
};
// A background (vb_set_background): the pixels every frame enqueued while it is set starts from, described and checked as a
// registered destination is (destination_of). Pixel (x, y) of cell c of a LINEAR one at ptr + (c * height + y) * pitch + T * x.
struct Background {
    bool on = false;
    Destination d;
};

// key of a captured frame: the inputs of its launches (see enqueue)
struct GraphKey {
    VbConfig cfg;
    VbFrameBufs bufs;
    VbFineBg bg; // the background's descriptor; its pixels are read at replay
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

// A view (vb_set_view): the f32 coefficients every frame enqueued while it is set renders the scene under.
struct View {
    bool on = false;
    float m[6] = {};
};

// Everything a frame needs to be issued again (issue): a re-run renders under the view, over the background and from the scene
// slot the frame was first issued with, even if the renderer's have changed since.
struct Frame {
    vb_params params{};
    Dest dest;
    View view;
    Background bg;
    uint32_t slot = 0;
};

// Composition (vb_compose). A ramp key is one distinct gradient ramp, (stops, interpolation space) compared as every
// resolve compares them (vb_same_ramp); an image key is one atlas slot, (pixels pointer, width, height, hash of the pixels). Fragments hold
// references to the keys of their patches, so de-duplicating a composed scene's ramps and images is a walk over the
// instances' patch lists (stamp / local: the ramp id or atlas slot the key got in the compose numbered stamp).
struct RampKey {
    std::vector<vb_ramp_stop> stops;
    bool premul = false;
    bool self_equal = true; // false when a stop holds a NaN: such a ramp equals no other ramp, itself included
    uint32_t id = 0, refs = 0;
    uint32_t pool = 0;      // its first stop in the renderer's stop pool
    uint64_t stamp = 0;
    uint32_t local = 0;
};
struct ImageKey {
    const void *key = nullptr;
    uint32_t w = 0, h = 0, id = 0, refs = 0;
    uint64_t pixels_hash = 0; // of the pixels read at upload (0 for a NULL or registered-texture key, which are not read)
    uint64_t stamp = 0;
    uint32_t local = 0;
};
// A resident fragment: its streams in one device allocation, back to back behind a header of their word offsets (k_compose.cu
// reads it), followed by a copy of the pixels of each image key it draws. Patch words are as the encoder wrote them.
enum { CMP_TAGS, CMP_PATH_DATA, CMP_DRAW_TAGS, CMP_DRAW_DATA, CMP_TRANSFORMS, CMP_STYLES, CMP_STREAMS };
#define CMP_FROM_OVERRIDE 0xffffffffu // the source of an atlas slot filled from an override (fragment ids start at 1, count up)
// An image's atlas slot in a composition: (image-key id << 32 | pixel source), as in SceneSlot::atlas_keys, and x << 16 | y.
struct ImgPlace {
    uint64_t key;
    uint32_t xy;
};
struct Fragment {
    uint32_t id = 0;
    void *mem = nullptr;
    size_t bytes = 0;
    uint32_t len[CMP_STREAMS] = {}; // tag bytes, path data words, draw tags, draw data words, transforms, style words
    uint32_t n_paths = 0, n_clips = 0, n_open_clips = 0, info = 0;
    struct Ramp { uint32_t dd, extend; RampKey *key; };
    struct Image { uint32_t dd; ImageKey *key; const uint8_t *pixels; }; // pixels: in mem, or nullptr for a NULL / texture key
    std::vector<Ramp> ramps;
    std::vector<Image> images;
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
        // set by vb_compose, cleared by every other upload: what the slot's ramps and atlas were made from, so that a compose
        // regenerates them only when that changes (ramp-key ids in ramp order; (image-key id << 32 | source fragment) in
        // placement order)
        bool composed = false;
        std::vector<uint32_t> ramp_keys;
        std::vector<uint64_t> atlas_keys;
        // the composed scene's instances, for vb_bind_instance_transforms: each one's fragment id and compose-time transform
        std::vector<uint32_t> inst_frag;
        std::vector<CmpXform> inst_xf;
        std::vector<uint32_t> inst_draw; // the exclusive prefix of the instances' draw objects (n + 1), for damage tracking
        // for vb_recompose: the atlas places of the instances' images in patch order, instance k's from inst_img[k] (n + 1)
        std::vector<uint32_t> inst_img;
        std::vector<ImgPlace> img_place;
        // for vb_bind_gradient_stops: the scene's ramp patches in draw-data order, each with its ramp word (relative to the
        // draw data), its stop count, interpolation space and first stop in `stops`, the encoded stops concatenated. Kept by
        // streams installations and vb_compose (have_stops), cleared by packed uploads, whose stops exist only as resolved ramps.
        struct StopPatch { uint32_t dd, n_stops, premul, first; };
        bool have_stops = false;
        std::vector<StopPatch> stop_patches;
        std::vector<vb_ramp_stop> stops;
    } slot[2];
    SceneSlot *cur = slot;
    DevBuf mask8, mask16;

    DevBuf fb[N_FRAME_BUFS]; // the frame's intermediates and arenas (FB_*)
    DevBuf target, target_alt;
    // Renderer::override_image: images (by key) whose pixels come from device memory at the device resolve
    struct Override {
        const uint8_t *src;
        size_t pitch;
        uint32_t w, h;
    };
    std::unordered_map<const void *, Override> overrides;
    std::unordered_map<const void *, Destination> dests; // by key
    DevBuf blit_rects;                  // k_atlas_blit's rectangles, staged through pinned[PIN_BLITS]
    PinnedStage pinned[N_PINNED];
    DevBuf resolve_tmp; // patches, ramp descriptors and stops of vb_scene_upload_streams
    // bump arenas (ARENAS), capacities in elements
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
    FrameCounts counts{}; // of the frame prepare set up last: vb_debug_download returns that much of its intermediates
    vb_params params{};
    Dest dest; // of the frame frame_prepare set up
    uint32_t launches = 0;
    VbFrameBufs bufs{};           // the buffers of the frame prepare set up, as the launchers take them
    bool use_graph = true;        // replay whole frames as CUDA graphs (see enqueue)
    GraphSlot graphs[4];
    uint32_t graph_next = 0;
    uint64_t graph_captures = 0;  // whole-frame graphs instantiated (vb_debug_graph_captures)
    // the view of the frames enqueued from now on; its coefficients reach view_coef in stream order (put_view)
    View view;
    DevBuf view_coef;
    Background bg; // of the frames enqueued from now on (vb_set_background); an array's surface object is the renderer's
    uint32_t readback_bands = 8; // fine launches per frame when the pixels go to the host (vb_render); 1 while streaming
    uint32_t occlusion_cull = 1; // fine starts each tile at its last opaque full-tile cover
    // path_tiling runs on its own stream beside coarse: forked after backdrop, joined before fine (enqueue_direct). Earlier in
    // the frame, draw and clip's links run on the same stream beside flatten: forked after the transforms, joined before clip's
    // boxes (draw_fork / draw_join).
    cudaStream_t tiling_stream = nullptr;
    cudaEvent_t tiling_fork = nullptr, tiling_join = nullptr, draw_fork = nullptr, draw_join = nullptr;
    cudaEvent_t ev[VB_N_STAGE_IDS + 1]{};
    cudaEvent_t frame_ev[2]{}; // around every whole frame (vb_last_frame_ms: the signal stripe balancing uses)
    bool frame_timed = false;
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
        Frame frame;
        vb_frame_stats stats{};
    } ring[3];
    uint64_t stream_seq = 0;

    // hit testing (vb_hit_test, vb_hit_map): the config and buffers of a frame, taken when it is enqueued (hit_enq) and handed to `hit` once
    // it is known to have succeeded. `hit` stays valid until something rewrites what the answers read: the next frame, a scene
    // upload, vb_set_cells, vb_run_stages, vb_debug_upload or vb_debug_limit_arena.
    struct HitFrame {
        bool valid = false;
        bool windowed = false; // rendered with a bin_row / tile_row window
        VbConfig cfg{};
        VbFrameBufs bufs{};
    } hit, hit_enq;
    DevBuf hit_io; // the host forms' points and answers, and maps

    // composition (vb_fragment_upload / vb_compose): the resident fragments by id, and the keys their ramps and images are
    // de-duplicated by across fragments
    std::unordered_map<uint32_t, std::unique_ptr<Fragment>> fragments;
    uint32_t next_fragment = 1;
    size_t fragment_bytes = 0;
    std::unordered_map<uint64_t, std::vector<RampKey *>> ramp_by_hash; // ramps whose stops compare equal to themselves
    std::unordered_map<uint32_t, std::unique_ptr<RampKey>> ramp_keys;
    uint32_t next_ramp_key = 1;
    DevBuf stop_pool;      // the stops of every ramp key, RampKey::pool apart
    uint32_t pool_used = 0; // stops
    std::map<std::tuple<const void *, uint32_t, uint32_t, uint64_t>, std::unique_ptr<ImageKey>> image_keys;
    // freed fragments whose memory composes already enqueued may still read: released once `done` has completed
    struct FreedFragment { void *mem; size_t bytes; cudaEvent_t done; };
    std::vector<FreedFragment> freed;
    uint32_t next_image_key = 1;
    uint64_t compose_seq = 0;
    DevBuf compose_tmp;                  // compose's tables, staged through pinned[PIN_COMPOSE]
    DevBuf paths_tmp;                    // the scratch of vb_fragment_from_device_paths (DpArgs, k_device_paths.cu)
    DevBuf dashes_tmp;                   // the scratch of vb_fragment_from_device_dashes' walk (DdArgs, k_device_dashes.cu)
    DevBuf dashes_mid;                   // its intermediate of sub-rings, which k_device_paths.cu encodes
    // What is bound to device rows (vb_bind_*, vb_compose.cu), with the device tables the bindings made at bind time (VbBound,
    // vb_stages.h), which point into the buffers below. Every scene installation unbinds (set_scene).
    //  - inst_tables: [prefix of the instances' transform counts (n + 1)] [compose-time transforms (n)] [the fragments'
    //    untransformed transforms] [the instances' draw prefix (n + 1)]
    //  - dd_slots: one word per draw-data word of the scene (VbBound::dd_slots, k_colors.cu), while colours, stops or opacity
    //    are bound
    //  - point_slots: the first point of each path (layout.n_paths + 1 words), then the bind-time flag of a 16-bit segment
    //  - stop_tables: [each bound gradient's ramp word in the draw data] [the gradients (RsRamp)] [their encoded stops] [per
    //    draw object its gradient or VB_COLOR_NONE]; stop_ramps: the scene's ramps, then a row per bound gradient (k_resolve.cu)
    //  - xform_ranges: each path's transform range {t_lo, t_hi} (layout.n_paths uint2, k_points.cu)
    //  - vis_mask: the bit mask (vb_vis_words) each frame packs the visibility rows into (k_visibility.cu)
    //  - width_snap: the snapshot (vb_width_entries floats) each frame reads the stroke-width rows into (k_widths.cu)
    VbBound bound{};
    DevBuf inst_tables, dd_slots, point_slots, stop_tables, stop_ramps, xform_ranges, vis_mask, width_snap;

    // damage tracking (vb_set_damage_tracking; k_damage.cu). `epoch` counts what makes the next frame a full one: a scene
    // installation, a binding or unbinding, vb_set_cells, a new view, switching tracking on. A frame is incremental when it
    // matches `base`, the last successful frame, in epoch, size, AA, base colour and device destination. The device keeps the
    // base's snapshot (dmg_snap) and advances it itself, so base changes only when the host learns that a frame succeeded.
    struct DamageFrame {
        uint32_t mode = VB_DMG_OFF;
        bool can_base = false; // one cell, no window, device destination: the frame can be the next one's base
        uint32_t w = 0, h = 0, aa = 0, base_color = 0;
        const void *dest = nullptr;
        uint64_t epoch = 0;
    };
    struct Damage {
        bool on = false;
        uint64_t epoch = 0;
        bool have_base = false, have_last = false;
        bool rects = false;      // vb_add_damage since the last successful frame (dirty overrides then do not force a full frame)
        bool force_full = false; // dirty overrides without rectangles: the frame and its re-runs are full
        DamageFrame base, frame, last; // frame: the one prepared last; last: the last successful one
        // A draw-object diff that tracking follows, of n_old instances (old_draws draw objects) of the base frame's scene against
        // n_new (new_draws) of the next one: a vb_recompose, or with `upload` an upload under vb_set_upload_diff (one draw object
        // per instance; the frame builds the tables, k_upload_diff.cu). `pending` from diff_begin until the installation
        // (set_scene), then `armed` for the next frame of epoch `epoch`, which is incremental against `base` and runs
        // k_recompose_damage on the base frame's boxes and the tables in dmg_diff; consumed when a frame succeeds.
        struct Diff {
            bool pending = false, armed = false, upload = false;
            uint64_t epoch = 0;
            uint32_t n_old = 0, n_new = 0, old_draws = 0, new_draws = 0;
            size_t o_boxes = 0, o_tables = 0;
        } diff;
    } dmg;
    DevBuf dmg_mask, dmg_pending, dmg_snap; // VbDamage::mask, pending and snap
    DevBuf dmg_diff; // the diff's buffer: [the base frame's draw boxes, at o_boxes] [the tables, at o_tables] (VbDamage)
    // upload diff (vb_set_upload_diff): the switch; and the spare scene, ramps and atlas buffers an upload that tracking follows
    // writes, while the current slot's (the base frame's scene) are kept and swapped into the spare set. The diff's buffer is laid
    // out by vb_udiff_layout, behind a head (VbUdiff) written from ud_head.
    bool upload_diff = false;
    DevBuf spare_scene, spare_ramps, spare_atlas;
    VbUdiff ud_head{};

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
                           &r->mask8, &r->mask16, &r->cell_draw, &r->target, &r->target_alt, &r->resolve_tmp, &r->blit_rects, &r->xc.arena,
                           &r->view_coef, &r->hit_io, &r->stop_pool, &r->compose_tmp, &r->paths_tmp, &r->dashes_tmp, &r->dashes_mid, &r->inst_tables, &r->dd_slots, &r->point_slots,
                           &r->stop_tables, &r->stop_ramps, &r->xform_ranges, &r->vis_mask, &r->width_snap,
                           &r->dmg_mask, &r->dmg_pending, &r->dmg_snap, &r->dmg_diff, &r->spare_scene, &r->spare_ramps, &r->spare_atlas};
    for (DevBuf *b : all) f(*b);
    for (DevBuf &b : r->fb) f(b);
}

#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) {                                                                  \
            r->err = std::string(#call) + ": " + cudaGetErrorString(e_);                          \
            return VB_E_CUDA;                                                                     \
        }                                                                                         \
    } while (0)

// One entry per frame buffer (FB_*): its name, where its pointer goes in VbFrameBufs and, for a fixed-size intermediate, its
// size in a frame of counts `n`: the bytes prepare allocates, or with `download` the bytes vb_debug_download returns by that
// name (for a downloadable one). The arenas' buffers have no size here: ensure_arena sizes them from the arenas' capacities.
struct FrameBufDesc {
    const char *name;
    size_t field; // offsetof(VbFrameBufs, ...)
    bool downloadable;
    size_t (*bytes)(const FrameCounts &n, bool download);
};

// One entry per bump arena: the name vb_debug_limit_arena takes, the buffer (FB_*), its element size and its VbBump counter.
// The special cases are in arena_offset, arena_need, ensure_arena and the first guesses of prepare.
using BumpCounter = uint32_t VbBump::*;
struct ArenaDesc {
    const char *name;
    int buf;
    size_t elem_bytes;
    BumpCounter counter;
};

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

namespace vb_host __attribute__((visibility("hidden"))) {

// Transforms of a scene: the stream from layout.transform_base to style_base (0 for a layout that does not fit the scene).
inline uint32_t n_transforms(const VbLayout &L, size_t scene_words) {
    if (L.style_base < L.transform_base || L.style_base > scene_words) return 0u;
    return (L.style_base - L.transform_base) / 6u;
}
// Draw-data words of a scene: the stream from layout.draw_data_base to transform_base (0 for a layout that does not fit the scene).
inline uint32_t n_draw_data(const VbLayout &L, size_t scene_words) {
    if (L.transform_base < L.draw_data_base || L.transform_base > scene_words) return 0u;
    return L.transform_base - L.draw_data_base;
}
// Path-data words of a scene: the stream from layout.path_data_base to draw_tag_base (0 for a layout that does not fit the scene).
inline uint32_t n_path_data(const VbLayout &L, size_t scene_words) {
    if (L.draw_tag_base < L.path_data_base || L.draw_tag_base > scene_words) return 0u;
    return L.draw_tag_base - L.path_data_base;
}
// Whether anything of the current scene is bound to device rows (VbBound). Such frames keep a damage snapshot, and are no base
// for an upload diff.
inline bool any_binding(const VbBound &b) {
    for (const VbRows &k : b.rows)
        if (k.rows) return true;
    return false;
}
// Whether frames read their draw data from the region past the scene's streams: with bound colours, bound gradient stops or
// bound opacity.
inline bool draw_data_bound(const VbBound &b) {
    return b.rows[VB_BIND_COLORS].rows || b.rows[VB_BIND_STOPS].rows || b.rows[VB_BIND_OPACITY].rows;
}

// The regions frames write past a scene's words, in this order, each present or not: the bound transforms (bound instance
// transforms, k_compose.cu, and bound transforms, k_transforms.cu, share it), the viewed transforms (k_view.cu), the bound
// draw data (bound colours, stops or opacity, k_colors.cu) and the bound path data (bound points, k_points.cu). This is the one place
// that knows the order: prepare places a frame's regions with it, scene allocations are sized with it, and the bind calls
// check 32-bit word offsets with it.
enum { REGION_BOUND_XF, REGION_VIEW, REGION_DRAW_DATA, REGION_PATH_DATA, N_REGIONS };
struct Regions {
    uint64_t base[N_REGIONS]; // each region's first word
    uint64_t len[N_REGIONS];  // its words, 0 when absent
    uint64_t words;           // the scene's words and its present regions': the frame's scene_words
    size_t bytes;             // the scene slot's allocation: those words, then slack
};
inline Regions regions_of(const VbLayout &L, size_t scene_words, bool bound_xf, bool view, bool draw_data, bool path_data) {
    const uint64_t xf = 6u * (uint64_t)n_transforms(L, scene_words);
    const uint64_t full[N_REGIONS] = {xf, xf, n_draw_data(L, scene_words), n_path_data(L, scene_words)};
    const bool on[N_REGIONS] = {bound_xf, view, draw_data, path_data};
    Regions g;
    g.words = scene_words;
    for (int i = 0; i < N_REGIONS; i++) {
        g.base[i] = g.words;
        g.len[i] = on[i] ? full[i] : 0u;
        g.words += g.len[i];
    }
    g.bytes = g.words * 4u + 64u;
    return g;
}

// vb_frame.cu
int ensure(vb_renderer *r, DevBuf &b, size_t bytes);
int stage_host(vb_renderer *r, PinnedStage &s, size_t bytes, uint8_t **host);
int stage_copied(vb_renderer *r, PinnedStage &s);
void hit_forget(vb_renderer *r);
extern const FrameBufDesc FRAME_BUFS[N_FRAME_BUFS];
extern const ArenaDesc ARENAS[N_ARENAS];
int arena_index(const char *name);
uint64_t ptcl_static(const VbConfig &c);
size_t arena_offset(const vb_renderer *r, int a);
uint64_t arena_need(const vb_renderer *r, int a);
int ensure_arena(vb_renderer *r, int a);
uint32_t grow(uint32_t need);
int drain_stream(vb_renderer *r);
FineRows fine_rows(const VbConfig &c, const Dest &d);
int frame_prepare(vb_renderer *r, const Frame &f);
int launch(vb_renderer *r, int first, int last);
Frame frame_of(const vb_renderer *r, const vb_params *p, const Dest &d);
int finish(vb_renderer *r, const Frame &f);
int settle(vb_renderer *r, const Frame &f, vb_frame_stats *stats);
bool device_memory_of(vb_renderer *r, const void *p);
int put_view(vb_renderer *r, const View &v);
int view_of(const double *affine, View *v);

// vb_upload.cu
void drop_registrations(vb_renderer *r);
// a registered destination's key: where fine stores (d->out), after the frame-time checks
int resolve_destination(vb_renderer *r, Dest *d);
// The checks vb_register_destination and vb_set_background make of a descriptor (`who` names the call in vb_last_error), and the
// Destination it describes, with a new surface object for an array.
int destination_of(vb_renderer *r, const vb_destination *d, const char *who, Destination *out);
// what fine's tiles start from in the frame r prepared (d->bg): the background bg, after the frame-time checks, or the base colour
int resolve_background(vb_renderer *r, const Background &bg, Dest *d);
void set_scene(vb_renderer *r, const VbLayout &L, size_t scene_words, uint32_t n_ramps, uint32_t atlas_w, uint32_t atlas_h,
               std::vector<vb_renderer::SceneSlot::OverridePlace> overridden, bool composed);
// diff: the upload may be diffed against the base frame's scene (vb_set_upload_diff); not for streamed frames
int upload_on(vb_renderer *r, cudaStream_t st, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
              uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, bool diff);
int enqueue_blits(vb_renderer *r, std::vector<VbBlitRect> &rects, void *atlas, uint32_t atlas_w);
int refresh_overrides(vb_renderer *r);
int check_streams(vb_renderer *r, const vb_encoding_streams *e, const char *who);
int image_source(vb_renderer *r, const char *who, const void *key, uint32_t w, uint32_t h, uint32_t x, uint32_t y,
                 std::vector<VbBlitRect> &blits, std::vector<vb_renderer::SceneSlot::OverridePlace> &over, bool *overridden);

// vb_damage.cu
int damage_prepare(vb_renderer *r);
void damage_succeeded(vb_renderer *r);
// Can the next installation be diffed against the scene the base frame rendered? What each diff source needs besides, it checks.
bool base_diffable(const vb_renderer *r);
// Begin the diff of the next installation (dmg.diff): n_old instances of the current scene's draw objects against n_new of
// new_draws; with `upload`, one draw object per instance. The caller stages the tables, or an upload's head and records.
int diff_begin(vb_renderer *r, cudaStream_t st, bool upload, uint32_t n_old, uint32_t n_new, uint32_t new_draws);

} // namespace vb_host
using namespace vb_host;
