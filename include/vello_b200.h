/* vello_b200.h -- C ABI of libvello_b200.so: a Hopper (sm_90a) drop-in for the GPU compute
 * path behind vello's `Renderer::render_to_texture`.
 *
 * What each entry point replaces in the reference (linebender/vello @ 3fabef93):
 *
 *   vb_renderer_new / _free   Renderer::new(&Device, RendererOptions)          vello/src/lib.rs:432-458
 *                             (shader registry + pipeline build: shaders.rs:48-274, wgpu_engine.rs:163-246)
 *   vb_render                 Renderer::render_to_texture(dev, queue, &scene, &tex, &RenderParams)
 *                                                                             vello/src/lib.rs:474-515
 *                             = Render::render_encoding_coarse + record_fine   vello/src/render.rs:135-629
 *                             + WgpuEngine::run_recording                      vello/src/wgpu_engine.rs:380-780
 *                             The inputs are exactly what crosses that seam: the packed scene bytes and
 *                             `Layout` from Resolver::resolve (vello_encoding/src/resolve.rs:183-399), the
 *                             gradient ramps (ramp_cache.rs:12,119-155), the image atlas and RenderParams
 *                             (lib.rs:357-369).
 *   vb_scene_upload           the `upload("vello.scene")` / ramps / atlas uploads    render.rs:149-232
 *   vb_render_resident        the 16-18 dispatches + fine, scene already on the device
 *   vb_frame_stats            Renderer::render_to_texture_async's bump readback  lib.rs:753-763 (the
 *                             reference leaves "re-run on overflow" as a TODO; here it is implemented)
 *   vb_run_stages / vb_debug_*   the operator seam `fn(u32 n_wg, &[CpuBinding])`  wgpu_engine.rs:57-61,
 *                             vello_shaders/src/cpu.rs:57-62 -- used by the stage-level parity tests
 *
 * Threading: one host thread per vb_renderer (mirrors `&mut self`; Renderer is Send, not Sync,
 * lib.rs:351-352). All pointers are plain host or device pointers; no torch / wgpu types.
 * Errors: 0 = ok, negative = error (vb_strerror). Unlike the reference, bump-arena overflow is
 * handled (grow and re-run) and, if it persists, REPORTED (VB_E_BUMP_OVERFLOW) instead of silently
 * leaving the texture unwritten (shared/bump.wgsl:5-9, fine.wgsl:1070-1074).
 */
#ifndef VELLO_B200_H
#define VELLO_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vb_renderer vb_renderer;

typedef struct {
    int32_t device;        /* CUDA device ordinal */
    uint32_t timing;       /* 1: record per-stage CUDA events (adds launch gaps; for profiling) */
    uint32_t max_retries;  /* grow-and-re-run attempts on bump overflow (0 -> default 6) */
    uint32_t reserved;
} vb_options;

/* == vello_encoding::Layout (resolve.rs:16-39); offsets in u32 words */
typedef struct {
    uint32_t n_draw_objects, n_paths, n_clips, bin_data_start;
    uint32_t path_tag_base, path_data_base, draw_tag_base, draw_data_base;
    uint32_t transform_base, style_base;
} vb_layout;

/* == vello::RenderParams (lib.rs:357-369) + the stripe window extension */
typedef struct {
    uint32_t base_color;  /* premultiplied RGBA8, r in the low byte (config.rs:183) */
    uint32_t width, height;
    uint32_t aa;          /* AaConfig: 0 Area, 1 Msaa8, 2 Msaa16 (lib.rs:175-193) */
    uint32_t bin_row0, bin_row1; /* render only bin rows [bin_row0, bin_row1) (256 px each); 0,0 = all.
                                    The output buffer then holds rows bin_row0*256 .. min(bin_row1*256, height). */
    uint32_t tile_row0, tile_row1; /* finer stripe window in TILE rows (16 px each), used when tile_row1 > tile_row0 (it then
                                    takes precedence over bin_row*): the cost-balanced stripes of vb_group / the multi-GPU
                                    bench. The output buffer holds rows tile_row0*16 .. min(tile_row1*16, height). */
} vb_params;

enum {
    VB_STAGE_ID_PATHTAG = 0, VB_STAGE_ID_FLATTEN, VB_STAGE_ID_DRAW, VB_STAGE_ID_CLIP, VB_STAGE_ID_BINNING,
    VB_STAGE_ID_TILE_ALLOC, VB_STAGE_ID_PATH_COUNT, VB_STAGE_ID_BACKDROP, VB_STAGE_ID_COARSE, VB_STAGE_ID_PATH_TILING,
    VB_STAGE_ID_FINE, VB_N_STAGE_IDS
};

typedef struct {
    /* == BumpAllocators (config.rs:24-37) after the frame */
    uint32_t failed, binning, ptcl, tile, seg_counts, segments, blend, lines;
    uint32_t retries;             /* re-runs this frame needed because an arena was too small */
    uint32_t kernel_launches;     /* kernels launched for the final (successful) attempt */
    float stage_ms[VB_N_STAGE_IDS]; /* only when options.timing */
    float total_ms;               /* device time of the final attempt (events), only when options.timing */
    uint64_t arena_bytes;         /* device memory currently held by the renderer */
} vb_frame_stats;

#define VB_OK 0
#define VB_E_INVALID (-1)
#define VB_E_CUDA (-2)
#define VB_E_BUMP_OVERFLOW (-3)
#define VB_E_NO_SCENE (-4)
#define VB_E_UNKNOWN_BUFFER (-5)

int vb_renderer_new(const vb_options *, vb_renderer **);
void vb_renderer_free(vb_renderer *);
const char *vb_strerror(int);
const char *vb_last_error(vb_renderer *);

/* Copy the packed scene + resources to the device (async on the renderer's stream). `scene` etc. are
 * HOST pointers; ramps = ramp_h rows of ramp_w (=512) premultiplied RGBA8 texels; atlas = RGBA8. */
int vb_scene_upload(vb_renderer *, const uint8_t *scene, size_t scene_len, const vb_layout *, const uint32_t *ramps,
                    uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas_rgba8, uint32_t atlas_w, uint32_t atlas_h);

/* Render the uploaded scene. `out` is a DEVICE pointer (RGBA8, un-premultiplied, pitch 4*width) or NULL
 * to render into the renderer's own target (see vb_target). Blocks until the frame is complete and
 * arenas were large enough (re-running if not). */
int vb_render_resident(vb_renderer *, const vb_params *, void *out_device, vb_frame_stats *);

/* Asynchronous variant for pipelined use / benchmarks: enqueue one attempt and return. The frame is
 * valid iff the following vb_frame_finish returns VB_OK with stats.failed == 0. */
int vb_render_enqueue(vb_renderer *, const vb_params *, void *out_device);
int vb_frame_finish(vb_renderer *, vb_frame_stats *);

/* One call = upload + render + (if out_is_device == 0) copy the pixels back to the HOST pointer `out`. */
int vb_render(vb_renderer *, const uint8_t *scene, size_t scene_len, const vb_layout *, const uint32_t *ramps, uint32_t ramp_w,
              uint32_t ramp_h, const uint8_t *atlas_rgba8, uint32_t atlas_w, uint32_t atlas_h, const vb_params *, void *out,
              uint32_t out_is_device, vb_frame_stats *);

/* Streaming form of vb_render for back-to-back frames with HOST buffers (a viewer / exporter reading every frame back,
 * as vello's headless examples do with a mapped read-back buffer, examples/headless/src/main.rs:188-210). Three frames are in
 * flight: the call uploads frame k's scene (its own stream, second scene slot), enqueues its rasterisation and read-back and
 * returns once frame k-1 is known to have rasterised without an arena overflow and frame k-2's pixels are in ITS out_host, so
 * upload(k+1), raster(k) and read-back(k-1) overlap and a frame costs max(raster, read-back). `stats` describes frame k-2
 * (zeros while there is none). vb_readback_wait completes everything still in flight. Use THREE alternating out_host buffers
 * (a buffer may be reused once the call two frames later has returned). */
int vb_render_begin(vb_renderer *, const uint8_t *scene, size_t scene_len, const vb_layout *, const uint32_t *ramps, uint32_t ramp_w,
                    uint32_t ramp_h, const uint8_t *atlas_rgba8, uint32_t atlas_w, uint32_t atlas_h, const vb_params *, void *out_host,
                    vb_frame_stats *);
int vb_readback_wait(vb_renderer *);
/* vb_render with a host destination launches fine in `n` bands of tile rows (1..8, default 8) and copies each band back
 * while the next one rasterises. Tuning knob; vb_render_begin always uses one band. */
int vb_set_readback_bands(vb_renderer *, uint32_t n);
/* Whole frames are replayed as CUDA graphs (one submission instead of ~20 launches; captured again whenever an arena,
 * the scene layout, the frame size or the window changes). On by default; 0 launches every kernel individually.
 * Environment: VELLO_B200_NO_GRAPH=1 disables it at renderer creation. */
int vb_set_cuda_graph(vb_renderer *, int on);
/* Switch the per-stage CUDA events of vb_options.timing on or off for the following frames (on: plain launches, no graph). */
int vb_set_timing(vb_renderer *, int on);

/* The renderer-owned target of the last frame (device pointer) and its size in bytes. */
void *vb_target(vb_renderer *, size_t *bytes);
/* Copy `bytes` from a device pointer to a host pointer on the renderer's stream, then synchronise. */
int vb_copy_to_host(vb_renderer *, const void *src_device, void *dst_host, size_t bytes);
/* cudaStream_t the renderer enqueues on (for event timing by the caller). Writes to an overridden image's device pixels
 * (vb_override_image) that are enqueued on this stream before the copying call are ordered before the copy. */
void *vb_stream(vb_renderer *);

/* ---- stage-level access (parity tests; mirrors the reference's CPU-shader operator seam) ----
 * SURVEY.md 8(b) sketched one entry point per stage, `vb_stage_<name>(renderer, n_wg, bindings, n)`, 1:1 with the reference's
 * `fn(u32 n_wg, &[CpuBinding])` (wgpu_engine.rs:57-61). That shape does not fit this implementation -- stages are fused
 * (pathtag_reduce / reduce2 / scan1 / scan are ONE kernel, draw_reduce + draw_leaf another), grids are derived on the device,
 * and the bindings are renderer-owned arenas -- so the seam is instead: vb_run_stages(first..last) over the renderer's own
 * buffers + vb_debug_download / vb_debug_upload of any buffer by its Appendix-B name. A stage range may be run once per
 * zeroing of the control block (i.e. once after a range that started at stage 0). */
/* Run stages first..last (VB_STAGE_ID_*) of the uploaded scene, one attempt, synchronously. */
int vb_run_stages(vb_renderer *, const vb_params *, int first, int last, void *out_device);
/* Copy an intermediate buffer to the host: "tag_monoids","path_bboxes","lines","draw_monoids",
 * "info_bin_data","clip_inp","clip_bboxes","draw_bboxes","bin_headers","paths","tiles","seg_counts",
 * "segments","ptcl","blend_spill","bump","config", and the guard regions of vb_debug_limit_arena ("<arena>.guard", empty
 * while the arena has no limit). Returns bytes available in *bytes; copies min(cap, bytes). */
int vb_debug_download(vb_renderer *, const char *name, void *dst, size_t cap, size_t *bytes);
/* Overwrite an intermediate buffer from the host ("lines" also sets bump.lines; "path_bboxes"). */
int vb_debug_upload(vb_renderer *, const char *name, const void *src, size_t bytes);
/* Test-only capacity limit of one bump arena, to drive the overflow / grow-and-re-run path at a chosen boundary. `arena`:
 * "lines", "binning", "tiles", "seg_counts", "segments", "blend" or "ptcl"; `limit` in the units of the matching
 * VbConfig::*_size (ptcl: words of the whole arena, static area included); UINT32_MAX clears it. The kernels then see
 * min(capacity, limit); the allocation is unchanged and its bytes past the limit become a guard region, filled with
 * VB_GUARD_BYTE when the limit is set (after the renderer's streams are synchronised) and downloadable as "<arena>.guard"
 * (for "lines" also "line_scratch.guard" and "flatten_jobs.guard"). A limit lasts until an attempt overflows it: growing
 * the arenas after that attempt drops it. vb_run_stages never grows, so there it stays until cleared. VB_E_INVALID for a
 * limit of 0, above the current allocation, or (ptcl) below the static area of the last frame's tiles. */
int vb_debug_limit_arena(vb_renderer *, const char *arena, uint32_t limit);
#define VB_GUARD_BYTE 0xA5

/* Traffic statistics of the last frame's `fine` (for the roofline): PTCL words its interpreters read,
 * segments referenced by CMD_FILL, number of CMD_FILL commands. */
/* fine starts every tile at its last opaque full-tile cover (CMD_SOLID + CMD_COLOR with alpha 255 outside any clip);
 * commands before it cannot reach the output, so pixels are identical. On by default; 0 executes every command, as
 * vello_shaders/shader/fine.wgsl:1064-1398 does. No counterpart in the reference (an addition, like early-z). */
int vb_set_occlusion_cull(vb_renderer *, int on);

int vb_debug_fine_traffic(vb_renderer *, uint64_t *ptcl_words, uint64_t *segment_refs, uint64_t *fill_cmds);

/* ---- batches: many scenes of one size in one pass (an addition; vello has no batch API) ----
 * Split the uploaded scene's draw objects into n_cells contiguous ranges (cells): draw_offsets[0] = 0 <= ... <= draw_offsets[n_cells]
 * = layout.n_draw_objects (n_cells + 1 entries; vb_scene_batch builds such a scene and its offsets). The following frames of
 * that scene (vb_render_resident, vb_render_enqueue, vb_render_uploaded, vb_run_stages) render cell c, alone, into a
 * params.width x params.height frame at byte offset c * 4 * width * height of the destination: n_cells frames back to back,
 * i.e. an [n_cells, height, width, 4] RGBA8 buffer. Every cell shares the params (size, AA, base colour); no cell's geometry
 * reaches another's frame, and a cell's pixels are the ones its scene renders alone. Any scene upload resets the renderer to
 * one cell; n_cells = 1 ({0, n_draw_objects}) is no batch. VB_E_INVALID (vb_last_error says why): offsets that do not start
 * at 0, decrease, or do not end at n_draw_objects; a cell whose BEGIN_CLIP / END_CLIP do not balance; a renderer of a vb_group
 * or with the exchange enabled; and, at the frame, bin_row / tile_row windows or a batch larger than the arenas can index. */
int vb_set_cells(vb_renderer *, const uint32_t *draw_offsets, uint32_t n_cells);

/* ---- Resolver::resolve on the DEVICE (vello_encoding/src/resolve.rs:183-399, ramp_cache.rs:119-155) ----
 * Instead of a packed scene the caller hands over the six streams of a vello_encoding::Encoding (encoding.rs:22-48) and its
 * late-bound patches (resolve.rs:560-590): each stream is copied straight to its Layout offset inside the packed buffer in
 * device memory, and a kernel finishes the job there -- tag padding, the trailing PATH / END_CLIP tags of unclosed clips, the
 * ramp-id and atlas-position patches, and the gradient ramps themselves (one thread per texel). The images go into the atlas
 * with one 2-D copy each from host memory, except those with an override (vb_override_image below), which come from device
 * memory with one k_atlas_blit launch for all of them. Only sizes, the ramp de-duplication and the atlas shelf placement stay on the host. The resulting
 * device buffers are byte-identical to what vb_scene_upload receives from the host-side resolve (tests/test_gpu_parity.py).
 * Glyph runs are not part of this path (they are resolved to outlines above the boundary). */
typedef struct { float offset, r, g, b, a; } vb_ramp_stop; /* straight-alpha colour */
typedef struct {
    uint32_t draw_data_offset; /* word in the draw-data stream that receives (ramp id << 2) | extend */
    uint32_t extend, premul_interp, n_stops;
    const vb_ramp_stop *stops;
} vb_ramp_patch;
typedef struct {
    uint32_t draw_data_offset; /* word that receives (atlas x << 16) | atlas y */
    uint32_t width, height;
    const uint8_t *pixels; /* RGBA8 / BGRA8 rows, width * 4 bytes each; identical pointers share one atlas slot */
} vb_image_patch;
typedef struct {
    const uint8_t *path_tags; uint32_t n_path_tags;
    const uint32_t *path_data; uint32_t n_path_data;   /* 32-bit words */
    const uint32_t *draw_tags; uint32_t n_draw_tags;
    const uint32_t *draw_data; uint32_t n_draw_data;
    const float *transforms; uint32_t n_transforms;    /* 6 floats each (math.rs:9-17) */
    const uint32_t *styles; uint32_t n_styles;         /* 2 words each (path.rs:11-69) */
    uint32_t n_paths, n_clips, n_open_clips;
    const vb_ramp_patch *ramp_patches; uint32_t n_ramp_patches;
    const vb_image_patch *image_patches; uint32_t n_image_patches;
} vb_encoding_streams;
/* Resolve + upload; afterwards the renderer holds the scene exactly as after vb_scene_upload. *layout_out (optional) = the Layout. */
int vb_scene_upload_streams(vb_renderer *, const vb_encoding_streams *, vb_layout *layout_out);
/* Render the uploaded scene and deliver the pixels like vb_render does (host pointer with out_is_device == 0, device otherwise). */
int vb_render_uploaded(vb_renderer *, const vb_params *, void *out, uint32_t out_is_device, vb_frame_stats *);

/* ---- images drawn from device memory: Renderer::override_image / mark_override_image_dirty (vello/src/lib.rs:536-603) ----
 * An image is named by its key: the `pixels` pointer of its vb_image / vb_image_patch (the atlas already shares one slot per
 * key, like vello's blob id). With an override, every image of that key (and these dimensions) is copied into its atlas slot
 * from `device_pixels` by the device resolve (vb_scene_upload_streams / vb_scene_upload_device) with one k_atlas_blit for all
 * overridden images, instead of from the key's host memory. device_pixels: RGBA8 / BGRA8 rows (the vb_image's format decides),
 * row_pitch_bytes apart, in memory of the renderer's device (or managed memory); pointer and pitch multiples of 4, pitch >=
 * 4 * width, no dimension 0 -- else VB_E_INVALID (vb_last_error says why). device_pixels NULL removes the override.
 * Setting an override marks the image dirty.
 *
 * vello's semantics: the device resolve records where each overridden image sits in this renderer's atlas. A dirty image is
 * copied again in front of the next frame rendered from that scene (on vb_stream, before every kernel of the frame and outside
 * any captured graph; the atlas does not move, so frames keep replaying); a frame with nothing dirty enqueues nothing extra and
 * its kernel_launches do not count the copy. An image that is not marked dirty keeps the pixels copied last. Removing an override,
 * or giving it another size, takes effect at the next device resolve. The caller finishes or orders its writes to device_pixels
 * (e.g. on vb_stream, or with a stream synchronisation) before the call that copies them: vb_scene_upload_streams, or the next
 * frame after vb_mark_override_image_dirty. Because the copy precedes the frame's kernels in stream order, a frame may draw its
 * own destination buffer (e.g. the previous frame) as an image: it reads the old contents.
 * The device resolve returns VB_E_INVALID when an override's size differs from its image's. Caller-packed atlases
 * (vb_scene_upload, vb_render, vb_render_begin) and vb_group ignore overrides. */
int vb_override_image(vb_renderer *, const void *key, uint32_t width, uint32_t height, const void *device_pixels, size_t row_pitch_bytes);
/* Recopy the overridden image `key` before the next frame that renders from this renderer's atlas. VB_E_INVALID: no override. */
int vb_mark_override_image_dirty(vb_renderer *, const void *key);

/* ---- one frame on several GPUs of one box (SURVEY.md 8e, north_star: "a single frame shards across the GPUs by stripes") ----
 * The frame is cut into horizontal stripes of tile rows, one per device; every device runs the element stages on the scene and
 * the tile stages on its stripe (no winding seam exists between horizontal stripes, DESIGN.md 6), and `fine` on device k stores
 * its pixels STRAIGHT INTO THE FRAME BUFFER ON DEVICE 0 through NVLink peer mapping (no gather pass, no staging copy); with a
 * host destination every device reads its own stripe back over its own PCIe link instead. Stripe boundaries follow the measured
 * per-device frame times of the previous frames (cost balancing). One host thread drives all devices.
 *
 * Single process: vb_group. One process per GPU (torchrun): each rank owns a plain vb_renderer, rank 0 exports its frame buffer
 * with vb_ipc_export and the others map it with vb_ipc_open and pass `mapped + stripe offset` as out_device. */
typedef struct vb_group vb_group;
/* devices[]: CUDA ordinals, the first one owns the assembled frame (the same ordinal may be listed twice: two renderers share
 * that GPU; used by the single-GPU tests). opt->device is ignored. */
int vb_group_new(const int32_t *devices, uint32_t n_devices, const vb_options *opt, vb_group **out);
void vb_group_free(vb_group *);
uint32_t vb_group_size(const vb_group *);
vb_renderer *vb_group_renderer(vb_group *, uint32_t i); /* the i-th device's renderer (statistics, debugging) */
const char *vb_group_last_error(vb_group *);
/* Same arguments as vb_render; p->bin_row* / tile_row* must be 0 (the group chooses the stripes). `out`: host pointer, or a
 * device pointer ON devices[0] when out_is_device != 0, or NULL to leave the frame in the group's own buffer on devices[0]
 * (vb_group_frame). stats: array of vb_group_size() entries or NULL. */
int vb_group_render(vb_group *, const uint8_t *scene, size_t scene_len, const vb_layout *, const uint32_t *ramps, uint32_t ramp_w,
                    uint32_t ramp_h, const uint8_t *atlas_rgba8, uint32_t atlas_w, uint32_t atlas_h, const vb_params *, void *out,
                    uint32_t out_is_device, vb_frame_stats *stats);
int vb_group_scene_upload(vb_group *, const uint8_t *scene, size_t scene_len, const vb_layout *, const uint32_t *ramps, uint32_t ramp_w,
                          uint32_t ramp_h, const uint8_t *atlas_rgba8, uint32_t atlas_w, uint32_t atlas_h);
int vb_group_render_resident(vb_group *, const vb_params *, void *out_device, vb_frame_stats *stats);
void *vb_group_frame(vb_group *, size_t *bytes);
/* tile-row boundaries in use (n_devices + 1 entries) and the device times (ms) of the last frame (n_devices entries) */
int vb_group_stripes(vb_group *, uint32_t *boundaries, float *device_ms);
int vb_group_set_balancing(vb_group *, int on); /* default on */

/* ---- flatten sharded across the GPUs (SURVEY.md 8e option B) ----
 * By default every GPU of a multi-GPU frame flattens the whole scene (culled to its stripe). With the exchange enabled GPU k
 * flattens only its 1/G share of the tag stream and the GPUs trade results through peer memory inside the frame, without host
 * or NCCL involvement: lines are routed to the stripes they touch and PULLED by their owners, partial path boxes are combined,
 * the GPUs synchronise through epoch flags in each other's exchange arena (k_exchange.cu). Set-up, per renderer, after the
 * scene has been uploaded:
 *   vb_exchange_configure(r, rank, world, &arena, &bytes)   allocate my arena (fixed size; export it with vb_ipc_export across processes)
 *   vb_exchange_attach(r, peer, peer_arena)                 for every other rank: its arena as seen from this device
 *   vb_exchange_set_bounds(r, rows)                         the world + 1 tile-row boundaries of the stripes (same on every rank)
 *   vb_exchange_enable(r, 1)
 * then render with tile_row0/1 = rows[rank], rows[rank + 1] as before. All ranks must render the SAME sequence of frames
 * (every attempt advances an epoch): a frame that overflows an arena returns VB_E_BUMP_OVERFLOW after growing it instead of
 * re-running on its own, and the caller re-issues that frame on EVERY rank. A peer that never shows up turns into a failed
 * frame after ~2 s (VB_STAGE_EXCHANGE in stats.failed), never into a hung GPU. vb_group does all of this itself
 * (vb_group_set_exchange). */
int vb_exchange_configure(vb_renderer *, uint32_t rank, uint32_t world, void **arena, size_t *arena_bytes);
int vb_exchange_attach(vb_renderer *, uint32_t peer_rank, void *peer_arena);
int vb_exchange_set_bounds(vb_renderer *, const uint32_t *tile_row_bounds);
int vb_exchange_enable(vb_renderer *, int on);
int vb_group_set_exchange(vb_group *, int on);

/* CUDA IPC helpers for the one-process-per-GPU arrangement (64-byte handles, exchanged by the caller, e.g. over torch.distributed) */
int vb_frame_alloc(vb_renderer *, size_t bytes, void **device_ptr);  /* cudaMalloc on the renderer's device */
int vb_frame_free(vb_renderer *, void *device_ptr);
int vb_ipc_export(vb_renderer *, void *device_ptr, uint8_t handle[64]);
int vb_ipc_open(vb_renderer *, const uint8_t handle[64], void **device_ptr); /* enables peer access to the exporting device */
int vb_ipc_close(vb_renderer *, void *device_ptr);
/* device time of the last completed frame of this renderer in ms (events around the frame; 0 until a frame completed) */
float vb_last_frame_ms(vb_renderer *);

#ifdef __cplusplus
}
#endif
#endif
