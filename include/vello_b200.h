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

/* Render the uploaded scene. `out` is a DEVICE pointer (RGBA8, un-premultiplied, pitch 4*width), the key of a registered
 * destination (vb_register_destination: a pitched buffer or a CUDA array, RGBA8, BGRA8, RGBA16F or RGBA32F), or NULL to render into the
 * renderer's own target (see vb_target). Blocks until the frame is complete and arenas were large enough (re-running if not). */
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

/* ---- views: pan and zoom a resident scene without uploading it again (an addition; vello re-encodes the scene) ----
 * Render the uploaded scene under a view: frames enqueued after this call render what
 * Scene::new().append(&scene, Some(view)) would render (encoding.rs:94-174). affine = kurbo Affine coefficients
 * [a b c d e f], converted to f32 like Transform::from_kurbo. NULL clears the view. Non-finite coefficients (in f32):
 * VB_E_INVALID.
 *  - A view lasts until it is changed or cleared. It survives scene uploads: it belongs to the viewer, not to the scene.
 *  - It applies to every frame the renderer renders: vb_render_resident, vb_render_enqueue, vb_render_uploaded, vb_render,
 *    vb_render_begin, vb_run_stages, batches (every cell, each in its own frame), bin_row / tile_row windows and vb_group
 *    (vb_group_set_view).
 *  - It applies in stream order: a frame already enqueued (e.g. the frames in flight of vb_render_begin) keeps the view it was
 *    enqueued with, also when it is re-run after an arena overflow.
 *  - The viewed transforms are written by the frame itself into renderer-owned memory past the scene (one extra kernel);
 *    the uploaded bytes are never modified. Changing the coefficients replays a captured frame graph; setting or clearing
 *    a view captures again. Room for the viewed transforms is taken only while a view is set (the first viewed frame after an
 *    upload without it moves the scene and waits for the renderer's streams); clearing the view waits for the frames already
 *    enqueued and frees what the view held.
 *  - Setting any view, the identity included, switches on frame culling: flatten emits no lines for a tag whose hull (grown
 *    by the stroke's reach) lies above, below or right of the frame (or the window), so a zoomed-in frame flattens fewer
 *    lines. Pixels are those of the unculled frame. With the exchange (vb_exchange_enable) flatten does not cull; the view
 *    still applies. NULL restores the unviewed pipeline exactly. */
int vb_set_view(vb_renderer *, const double affine[6]);
int vb_debug_graph_captures(vb_renderer *, uint64_t *captures); /* test-only: whole-frame graphs instantiated so far */

/* ---- hit testing: the topmost draw object under each point of the last frame (an addition; vello's applications hit-test on
 * the host against their own geometry) ----
 * For each of the n points xy[2k], xy[2k + 1] writes draw_ix[k]: the index of the LAST draw object in draw order whose path
 * covers the point in the renderer's last frame that completed successfully, or -1.
 *  - Points are f32 pixel coordinates of that frame: x right, y down, pixel (i, j) covers [i, i+1) x [j, j+1). In a batch
 *    (vb_set_cells) the frame is the tall [n_cells * height, width] one: a point of cell c has y in [c * height, (c+1) * height).
 *  - Covering is geometric and exact: the winding number of the draw's flattened outline (the frame's own lines, so a view
 *    and flatten's tolerance are those on screen; strokes are their outlines) at the point is nonzero, or odd under the
 *    even-odd rule, and the point lies inside the clip path of every enclosing BEGIN_CLIP (each with its own fill rule).
 *    Brush alpha, layer alpha and blend modes do not matter: a transparent fill is hit, an image or a blurred rectangle
 *    anywhere in the rectangle it is drawn in. Colour never matters, so bound draw colours (vb_bind_draw_colors) do not change
 *    the answers, nor do bound gradient stops (vb_bind_gradient_stops). Bound path points (vb_bind_path_points) are part of the frame's geometry: the answers follow the points the
 *    frame read, and so are bound transforms (vb_bind_transforms): the answers follow the transforms the frame read. A point exactly on a line is decided by the half-open rules of the tile walk
 *    (tests/tile_walk_ref.py): deterministic, with no promise of the side.
 *  - BEGIN_CLIP / END_CLIP objects are never returned. Points outside the frame and NaN points give -1. Indices are the
 *    scene's draw-object indices (vb_scene_n_draw_objects / Scene.n_draw_objects; global in a batch: cell c's draws are
 *    draw_offsets[c] .. draw_offsets[c + 1]).
 *  - on_device == 0: host pointers; synchronous (the points go through a renderer-owned device buffer). on_device != 0: both
 *    are pointers to memory of the renderer's device; the work is enqueued on vb_stream and the call returns (order the
 *    points' writes before the call, and read the answers after synchronising with vb_stream).
 *  - The answers come from the frame's buffers as its kernels left them; hit tests write nothing of the frame, launch nothing
 *    of it and capture no graph: kernel_launches, graph captures and the next frame's pixels are the same with or without them.
 *    vb_set_view does not change the answers: they stay those of the frame rendered last until the next frame. A frame that
 *    was re-run after an arena overflow answers from the attempt that succeeded.
 * n = 0: nothing happens, VB_OK. VB_E_NO_SCENE: no successful frame since the last scene upload (any form), vb_set_cells,
 * vb_run_stages, vb_debug_upload or vb_debug_limit_arena (each rewrites something the answers read), or the last frame failed.
 * VB_E_INVALID (vb_last_error says why): NULL pointers; device pointers of another device (on_device); the last frame had a
 * bin_row / tile_row window; a renderer of a vb_group or with the exchange enabled; a frame enqueued and not finished
 * (vb_render_enqueue until vb_frame_finish, vb_render_begin until vb_readback_wait). */
int vb_hit_test(vb_renderer *, const float *xy, uint32_t n, int32_t *draw_ix, uint32_t on_device);
/* Hit maps: vb_hit_test's answer at every pixel centre of a rectangle of the same frame. Row j, column i of the output, at
 * (char *)draw_ix + j * pitch_bytes + 4 * i, is the answer for the point (x0 + i + 0.5f, y0 + j + 0.5f), equal int for int;
 * only those h rows of w values are written. Everything above carries over: the frame, its state rules and error codes, the
 * tall frame of a batch, on_device (draw_ix alone is the pointer checked), and a map leaves the frame alone as a hit test
 * does. Like hit tests, maps do not depend on colour, bound draw colours included. One CTA per 16 x 16 tile reads the tile's draw
 * list and segments once for its 256 pixels (DESIGN.md §1, "Hit maps").
 * w = 0 or h = 0: nothing happens, VB_OK. VB_E_INVALID also for NULL draw_ix; a rectangle not inside the last frame
 * (x0 + w > width or y0 + h > n_cells * height); pitch_bytes not a multiple of 4 or below 4 * w. */
int vb_hit_map(vb_renderer *, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, int32_t *draw_ix, size_t pitch_bytes,
               uint32_t on_device);

/* The renderer-owned target of the last frame (device pointer) and its size in bytes. */
void *vb_target(vb_renderer *, size_t *bytes);
/* Copy `bytes` from a device pointer to a host pointer on the renderer's stream, then synchronise. */
int vb_copy_to_host(vb_renderer *, const void *src_device, void *dst_host, size_t bytes);
/* ---- registered destinations: frames straight into CUDA arrays (interop images) and pitched buffers (an addition) ----
 * vello's render_to_texture writes a storage texture. A Vulkan or GL image imported into CUDA is a CUDA array, not a device
 * pointer: cudaImportExternalMemory, cudaExternalMemoryGetMappedMipmappedArray (with cudaArraySurfaceLoadStore), then
 * cudaGetMipmappedArrayLevel(.., 0). vb_register_destination turns such an array, or linear device memory at any row pitch,
 * into a key, which goes wherever a device destination pointer goes: vb_render_resident, vb_render_enqueue / vb_frame_finish,
 * vb_render_uploaded, vb_render and vb_render_scene with out_is_device = 1, and vb_run_stages.
 *  - Pixel (px, py) of a frame lands at texel (x + px, y + py) of the array, or at ptr + py * row_pitch_bytes + T * px, where
 *    the texel size T is 4 (RGBA8, BGRA8), 8 (RGBA16F) or 16 (RGBA32F).
 *  - Values: let c be fine's premultiplied f32 pixel and clamp01(v) = fminf(1, fmaxf(0, v)) (NaN gives 0). With straight
 *    alpha (the default, vello's) a texel is clamp01(c.rgb * (1 / fmaxf(c.a, 1e-6f))) and clamp01(c.a); with
 *    VB_DEST_PREMULTIPLIED in format (for the compositors that take premultiplied pixels) it is clamp01(c). RGBA8 and BGRA8
 *    store floor(0.5 + 255 * value) of those (the RGBA8 straight bytes are exactly a plain pointer's), with r and b swapped
 *    for BGRA8; RGBA16F stores them rounded to the nearest half (ties to even); RGBA32F stores them as they are. No colour
 *    conversion is done: an _SRGB or a float image receives vello's sRGB-encoded values as they are.
 *  - What the float formats add: coverage at edges, blurs, filtered images and translucent overlaps keep their f32 values.
 *    Layers (the blend stack), gradient ramps and images are 8-bit inside fine, as in vello, so a flat gradient fill or an
 *    unscaled image gains nothing.
 *  - A destination holds the whole frame, so a bin_row / tile_row window writes only its rows, at their own rows of the
 *    destination. (A plain pointer differs: its first row is the window's first row.)
 *  - Damage tracking: a frame into the same key as the last successful frame can be incremental, writing only its damaged
 *    tiles into the destination. Whole-frame graphs are keyed by the key like a pointer.
 *  - Keys come from the same reserved, inaccessible address range as vb_register_texture's keys: no buffer has a key's
 *    address, a key is never handed out twice, and a key used as an image key reads as an unregistered texture key does.
 * VB_E_INVALID (vb_last_error says why), each checked on the host before anything is enqueued:
 *  - registering: NULL arguments; an unknown kind, format or flag bit; a renderer of a vb_group or with the exchange
 *    configured; LINEAR: ptr NULL, not a multiple of the texel size T, or not device or managed memory of the renderer's
 *    device; a row pitch that is not a multiple of T or is 2^34 bytes or more; ARRAY: not a 2-D array (1-D, layered,
 *    cubemap, 3-D), channels that do not match the format (four 8-bit cudaChannelFormatKindUnsigned ones for RGBA8 and
 *    BGRA8, four 16-bit cudaChannelFormatKindFloat ones for RGBA16F, four 32-bit ones for RGBA32F), no
 *    cudaArraySurfaceLoadStore flag;
 *  - a frame into a key: the key is unregistered, another renderer's or a texture key; the frame does not fit (x + width or
 *    y + its last row past the array's extent, a row pitch below T * width); a batch (vb_set_cells with more than one cell);
 *  - a key where a host pointer or a plain device pointer is needed: vb_render / vb_render_uploaded / vb_render_scene with
 *    out_is_device = 0, vb_render_begin's out_host, vb_copy_to_host, image pixels (vb_override_image, vb_register_texture),
 *    vb_group destinations.
 * The caller keeps the memory or array alive and on the renderer's device while the key is registered. No CUDA call tells
 * cheaply which device an array belongs to, so an array of another device is a caller error, as a freed pointer is.
 * vb_unregister_destination returns once the frames already enqueued into the key have completed; VB_E_INVALID for a key that
 * is not a destination of this renderer. vb_renderer_free releases the destinations still registered. */
#define VB_DEST_LINEAR 0 /* device memory, row_pitch_bytes apart */
#define VB_DEST_ARRAY 1  /* a 2-D CUDA array (cudaArray_t / CUarray), written through a surface object */
#define VB_DEST_RGBA8 0  /* byte order of a stored pixel: vello's Rgba8Unorm (r in the low byte) */
#define VB_DEST_BGRA8 1  /* b, g, r, a */
#define VB_DEST_RGBA16F 2 /* four IEEE half floats r, g, b, a: 8 bytes a texel */
#define VB_DEST_RGBA32F 3 /* four floats r, g, b, a: 16 bytes a texel */
#define VB_DEST_PREMULTIPLIED 0x100 /* OR'd into format: premultiplied alpha instead of straight */
typedef struct {
    uint32_t kind, format;
    void *ptr;              /* LINEAR: where pixel (0, 0) of a frame goes */
    size_t row_pitch_bytes; /* LINEAR */
    void *array;            /* ARRAY: level-0 array of the renderer's device */
    uint32_t x, y;          /* ARRAY: the texel pixel (0, 0) of a frame lands on */
} vb_destination;
int vb_register_destination(vb_renderer *, const vb_destination *, void **key_out);
int vb_unregister_destination(vb_renderer *, void *key);

/* ---- backgrounds: frames drawn over the pixels of a device buffer or a CUDA array (an addition) ----
 * vello's render_to_texture starts every pixel at the base colour: the destination is overwritten, never drawn on. With a
 * background set, every frame enqueued from then on starts pixel (x, y) at the background's value instead, and the base colour
 * is ignored: 2-D content over a 3-D view or a video frame without a second image and a blend, annotations drawn over a batch
 * of images, a cached static layer under a few moving objects. The descriptor is a vb_destination:
 *  - LINEAR: pixel (x, y) at ptr + y * row_pitch_bytes + T * x (T as for destinations: 4, 8 or 16). With vb_set_cells and
 *    n_cells > 1, cell c's pixel (x, y) at ptr + (c * height + y) * row_pitch_bytes + T * x, so an [N, H, W, 4] tensor works.
 *    ARRAY: texel (background->x + x, background->y + y) of a 2-D CUDA array, read through a surface object.
 *  - format: VB_DEST_RGBA8, VB_DEST_BGRA8, VB_DEST_RGBA16F or VB_DEST_RGBA32F, optionally OR'd with VB_DEST_PREMULTIPLIED.
 *  - Like a destination, a background holds the whole frame: a bin_row / tile_row window or a read-back band reads its rows.
 * The load, per pixel: each channel as f32 (byte / 255.0f for the 8-bit formats, with r and b swapped back for BGRA8; the half
 * converted exactly; the float as stored), then clamp01 (fminf(1, fmaxf(0, v)), the store's clamp: NaN gives 0), then for
 * straight alpha (r * a, g * a, b * a, a), each product rounded on its own; premultiplied values are taken as they are. The
 * store, layers, blend modes and luminance masks are unchanged: the background is the bottom of the blend stack, as the base
 * colour was. So:
 *  - a premultiplied RGBA8 background filled with the base colour's bytes renders byte for byte the frame without one;
 *  - a tile whose command list starts with an opaque cover of the whole tile does not read the background (fine skips the
 *    load), and vb_set_occlusion_cull does not change the pixels;
 *  - with an empty scene, a premultiplied background stored into a destination of the same format comes back bit for bit
 *    (float texels: those already in [0, 1], with -0 read as +0); a straight texel with alpha 0 loses its colour.
 * Scope: every single-renderer frame (vb_render_resident, vb_render_enqueue / vb_frame_finish, vb_render_uploaded, vb_render,
 * vb_render_scene, vb_render_begin, whose destination is host memory, and vb_run_stages ranges that contain fine). The
 * background may be the frame's destination itself (the same pointer or array): each pixel is read and then written by the
 * same thread, and no other thread touches it. A background is renderer state, like a view: it survives uploads, compose,
 * recompose, bindings and vb_set_cells. A frame keeps the background it was issued with, when it is re-run after an arena
 * overflow and when vb_set_background is called while it is in flight. Whole-frame graphs are keyed by the descriptor, not
 * the pixels: new contents replay the captured graph. A frame with a background is full under damage tracking and is no base
 * for the next frame, which is full as well. Hit tests and hit maps answer from geometry and do not depend on it.
 * NULL clears the background. VB_E_INVALID (vb_last_error says why):
 *  - setting: everything vb_register_destination refuses for the same descriptor (an unknown kind, format or flag bit; a
 *    renderer of a vb_group or with the exchange configured; LINEAR: ptr NULL, misaligned, a texture or destination key, or
 *    not device or managed memory of the renderer's device; a bad row pitch; ARRAY: not a 2-D array, channels that do not
 *    match the format, no cudaArraySurfaceLoadStore); vb_exchange_configure refuses a renderer with a background;
 *  - a frame the background cannot cover: a row pitch below T * width, an array too small for the frame at its origin, an
 *    array background with more than one cell.
 * The caller keeps the memory or array alive and its pixels unchanged until the frames that read it have completed. A LINEAR
 * background must hold every row of every cell a frame reads (the descriptor has no height to check it by). Clearing the
 * background, or replacing an array background, returns once the frames that read the old array have completed (streamed
 * frames included); the renderer's surface object is destroyed then. If completing them fails (a streamed frame's error is
 * returned), the renderer is left without a background. */
int vb_set_background(vb_renderer *, const vb_destination *background);

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
 * "segments","ptcl","blend_spill","bump","config"; "transforms", "draw_data" and "path_data", the transform, draw-data and
 * path-data words the last frame read (its bound or viewed region, else the scene's own stream); and the guard regions of vb_debug_limit_arena
 * ("<arena>.guard", empty while the arena has no limit). Test-only, flatten's own state after the last attempt: "flatten_counters" (3 x u32:
 * literal line records, deferred jobs, partitions on the general tag kernel's work list), "line_scratch" (32 B literal
 * records) and "flatten_jobs" (96 B job records), each up to its counter and at most its capacity.
 * Returns bytes available in *bytes; copies min(cap, bytes). */
int vb_debug_download(vb_renderer *, const char *name, void *dst, size_t cap, size_t *bytes);
/* Overwrite an intermediate buffer from the host: "lines" (also sets bump.lines), "tiles" (also sets bump.tile), "path_bboxes",
 * "paths" (exactly layout.n_draw_objects records, else VB_E_INVALID). "lines" and "tiles" grow their arena when `bytes` exceeds
 * it. Growing frees the arena without copying, and the control block, which holds the bump counters and backdrop's look-back
 * state sized from the tile capacity, is only set up anew by a vb_run_stages range that starts at stage 0. So to run
 * backdrop on uploaded tiles: upload them once (to grow the arena), run pathtag..path_count, upload "paths" and "tiles"
 * again, then run backdrop alone. */
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
/* Test-only: the decoupled look-back every scan kernel uses, run alone on the renderer's device over n_parts partitions of one
 * warp each. Partitions take tickets in launch order; partition p waits delay_ns[p] (NULL: none; each at most
 * VB_LOOKBACK_MAX_DELAY_NS) before it publishes agg[p], so that its successors publish aggregates only and later partitions
 * combine whole windows of them. Writes every partition's exclusive prefix to excl[p]. agg and excl hold K words per
 * partition, K by `op`: VB_LOOKBACK_SUM1 (a sum, K = 1), VB_LOOKBACK_SUM5 (a field-wise sum, K = 5), VB_LOOKBACK_BACKDROP
 * (backdrop's segmented sum {crossings, row start seen, backdrop since it}, K = 3), VB_LOOKBACK_AFFINE (x -> a x + b mod
 * 2^32 stored as {a - 1, b}, applied in partition order, K = 2). VB_E_INVALID for another op, n_parts outside
 * 1..VB_LOOKBACK_MAX_PARTS or a longer delay. Synchronous. */
int vb_debug_lookback(vb_renderer *, int op, uint32_t n_parts, const uint32_t *agg, const uint32_t *delay_ns, uint32_t *excl);
#define VB_LOOKBACK_SUM1 0
#define VB_LOOKBACK_SUM5 1
#define VB_LOOKBACK_BACKDROP 2
#define VB_LOOKBACK_AFFINE 3
#define VB_LOOKBACK_MAX_PARTS 65536u
#define VB_LOOKBACK_MAX_DELAY_NS 1000000u

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
 * Glyph runs are not part of this path (they are resolved to outlines above the boundary).
 * Atlas limit (every resolve: vb_scene_resolve, this one, vb_fragment_upload, vb_compose / vb_recompose): the draw data holds
 * an image's atlas place and size as 16-bit fields, so an image with a side over 65535 texels, or one the 2048-wide shelves
 * would place below row 65535, is refused with VB_E_INVALID (vb_last_error says why where the call has a renderer) and the
 * renderer's scene is left as it was; vb_register_texture refuses a side over 65535 too. */
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

/* ---- composition: frames built on the device from resident fragments (an addition; vello builds every frame on the host as
 * Scene::new() + scene.append(&fragment, Some(transform)) per fragment, vello/src/scene.rs:464-469, encoding.rs:94-174) ----
 * vb_fragment_upload copies a fragment's streams (the vb_encoding_streams of vb_scene_upload_streams) into one renderer-owned
 * device allocation, together with the host pixels of its images (one copy per key, as the device resolve keys them: the
 * `pixels` pointer and the size) and its gradient stops. Synchronous; the caller's memory is not needed afterwards, so a key's
 * address may later hold other pixels: images of different fragments share an atlas slot only when their pointer, size AND
 * pixels (a 64-bit hash taken at upload) agree. Registered texture keys are never read (their pixels exist only in device
 * memory) and NULL keys give a zero region, as in a resolve; both are one image per pointer.
 * *fragment_out receives its id; ids are never reused.
 * vb_fragment_free returns at once: the fragment's id is invalid from then on, and its memory is released once the work
 * already enqueued that reads it has finished (checked at the next vb_fragment_* / vb_compose call). A composed scene is a
 * copy: it does not change.
 * vb_compose makes the renderer's current scene exactly
 *     s = Scene::new(); for k: s.append(&fragment[inst[k].fragment], inst[k].has_transform ? Some(T_k) : None); resolve(s)
 * without reading stream, stop or pixel data from the host: the packed scene, the Layout (*layout_out, optional), the ramps
 * and the atlas are byte-identical to vb_scene_append + vb_scene_resolve of those scenes (ramp de-duplication by (stops,
 * interpolation space) across fragments, one atlas slot per image key in first-seen order, the trailing PATH / END_CLIP tags
 * of open clips, the f32 transform product of Encoding::append). transform = kurbo Affine [a b c d e f], converted to f32
 * like Transform::from_kurbo. draw_offsets (n + 1 entries, or NULL): draw_offsets[k] = the draw-object index of instance k's
 * first draw, draw_offsets[n] = the total before the trailing END_CLIPs; a vb_hit_test answer i belongs to the instance k
 * with draw_offsets[k] <= i < draw_offsets[k + 1].
 *  - Afterwards the renderer is as after any scene upload: frames render the composed scene, a view applies on top, vb_set_cells
 *    may split it, vb_hit_test answers VB_E_NO_SCENE until the next frame, and overridden images refresh when marked dirty.
 *  - Images: a key with an override on this renderer (vb_override_image) is copied from the override's device memory (a size
 *    mismatch is VB_E_INVALID); any other from its fragment's copy; a registered texture key without an override is VB_E_INVALID.
 *  - Asynchronous: the work is enqueued on vb_stream and the call returns without waiting, except when the scene, ramp or atlas
 *    buffers have to grow. Streamed frames still in flight (vb_render_begin) are completed first.
 *  - The ramps are regenerated only when the ordered list of distinct ramps changes, the atlas only when the ordered list of
 *    placed images changes or an override applies. A compose that changes only transforms keeps the layout and the buffers,
 *    so the captured frame graph replays.
 *  - n = 0 composes the empty scene.
 * VB_E_INVALID (vb_last_error says why), with the previous scene left as it was: NULL pointers; an unknown or freed fragment;
 * a transform that is not finite in f32; a scene past 32-bit word offsets; a renderer of a vb_group or with the exchange
 * enabled; a call between vb_render_enqueue and vb_frame_finish. */
typedef struct {
    uint32_t fragment;      /* id from vb_fragment_upload */
    uint32_t has_transform; /* 0: Encoding::append(&frag, None); 1: Some(transform) */
    double transform[6];    /* kurbo Affine [a b c d e f], converted to f32 like Transform::from_kurbo */
} vb_instance;
int vb_fragment_upload(vb_renderer *, const vb_encoding_streams *, uint32_t *fragment_out);
int vb_fragment_free(vb_renderer *, uint32_t fragment);
/* A fragment built on the device from ragged arrays in device memory (an addition; no vello counterpart): polygons a model
 * predicts, a time series that grows, a simulation's outlines or a filtered map layer, in the points / offsets layout of
 * GeoArrow, shapely and ragged tensors, with no host loop over their rows and no copy to the host. Path i is rings
 * path_offsets[i] .. path_offsets[i + 1] - 1 (path_offsets NULL: ring i alone, n_paths = n_rings); ring r is points
 * ring_offsets[r] .. ring_offsets[r + 1] - 1, each an (x, y) f32 pair point_pitch_bytes apart; path i's colour is the
 * straight-alpha r g b a f32 row i, color_pitch_bytes apart. The fragment is word for word what vb_fragment_upload receives from
 * a fresh Scene that, for each path i in order, calls
 *     fill(fill_rule, IDENTITY, Color(colors[i]), None, shape_i)      kind 0
 *     stroke(Stroke{width, join, miter_limit, start_cap, end_cap}, IDENTITY, Color(colors[i]), None, shape_i)   kind 1
 * where shape_i is, for each ring of path i, M p_first, L p for every following point, then Z (fills always; strokes when
 * `closed`). So the encoders' rules hold: a point EPS-close (1e-12) to the last kept one writes nothing, a ring of fewer than
 * two distinct points writes nothing, a ring closes with a line when its last kept point differs bit for bit from its first,
 * strokes end each ring with a cap marker, and a path whose rings all write nothing draws nothing. Its one TRANSFORM (identity)
 * and STYLE come first when n_paths > 0; n_paths = 0 is the empty fragment. join and caps are vb_stroke's (VB_JOIN_*,
 * VB_CAP_*, vello_b200_scene.h); dashes, brushes other than one colour per path, and clips are not part of it (curves are
 * vb_fragment_from_device_curves, below).
 * *n_draw_objects_out (optional) receives the fragment's draw objects; draw_index (optional, n_paths int32 entries, device
 * memory) receives path i's draw object within the fragment, or -1 for a path that draws nothing. Which path-data rows a
 * point lands in depends on the points dropped, so bind points of such a fragment (vb_bind_path_points) only with rows made
 * from its own encoding.
 *  - The result is an ordinary fragment: vb_compose and vb_recompose take it beside uploaded ones, instance transforms, views,
 *    hit tests and every binding apply, vb_fragment_free frees it, and its id is never reused. A base layer uploaded once and
 *    an overlay rebuilt from device arrays every frame are one vb_compose([base, overlay]).
 *  - The arrays are read on vb_stream: order the writes to them before the call (on vb_stream, or with a synchronisation).
 *    The call is synchronous like vb_fragment_upload: the streams' lengths depend on the data, so after its kernels it reads
 *    the totals back and synchronises vb_stream once. The allocation is sized for the worst case of the counts (a tag and two
 *    words per point, a closing line and a cap marker per ring, a PATH tag and a draw object per path).
 *  - A compose whose stream lengths differ from the last one's captures its frame graph anew (DESIGN.md gives the cost).
 * VB_E_INVALID (vb_last_error says why), with no fragment made and the renderer as it was: NULL pointers where a count is not
 * zero, or path_offsets NULL with n_paths != n_rings; an array that is not 4-byte aligned device or managed memory of the
 * renderer's device; a point pitch below 8 or a colour pitch below 16 bytes, a pitch that is not a multiple of 4 or is 4 GiB
 * or more; a count past int32; a bad kind, fill rule, join or cap; a width that is not finite and > 0, or a miter limit that
 * is not finite; a worst case past 32-bit word offsets; a renderer of a vb_group or with the exchange; a call between
 * vb_render_enqueue and vb_frame_finish. Checked on the device, naming the first offending row: ring_offsets not starting
 * at 0, decreasing, or not ending at n_points; path_offsets likewise over the rings; a coordinate or a colour component that
 * is not finite. */
typedef struct {
    const float *points;       uint32_t n_points;  size_t point_pitch_bytes; /* x y f32 rows */
    const int32_t *ring_offsets; uint32_t n_rings;  /* n_rings + 1 entries */
    const int32_t *path_offsets; uint32_t n_paths;  /* n_paths + 1 entries over rings; NULL: one ring per path (n_paths = n_rings) */
    const float *colors;       size_t color_pitch_bytes; /* n_paths rows of straight-alpha sRGB r g b a */
    uint32_t kind;             /* 0 fill, 1 stroke */
    uint32_t fill_rule;        /* fills: 0 non-zero, 1 even-odd (VB_FILL_NON_ZERO / VB_FILL_EVEN_ODD) */
    float width, miter_limit;  uint32_t join, start_cap, end_cap, closed; /* strokes: kurbo Stroke without dashes */
    int32_t *draw_index;       /* optional out, n_paths entries: path i's draw object in the fragment, or -1 */
} vb_device_paths;
int vb_fragment_from_device_paths(vb_renderer *, const vb_device_paths *, uint32_t *fragment_out, uint32_t *n_draw_objects_out);
/* vb_fragment_from_device_curves: vb_fragment_from_device_paths of quadratic and cubic Bézier paths (an addition; no vello
 * counterpart): glyph outlines (TrueType quadratics, CFF cubics), the control points a vector-graphics model outputs, circle
 * and ellipse markers, splines. point_kinds holds one byte per point (n_points, device or managed memory of the renderer's
 * device, any alignment): 0 on-curve, 1 off-curve. Within a ring each on-curve point after the first ends one segment, chosen
 * by the k off-curve points in front of it: k = 0 L e, k = 1 Q c e, k = 2 C c1 c2 e. The fragment is word for word what
 * vb_fragment_upload receives from the Scene loop above, shape_i being, for each ring of path i, M p_first, those segments in
 * order, then Z (fills always; strokes when `closed`). A curved closing segment repeats the first point as its end: Z then adds
 * no line, the points being equal bit for bit. point_kinds NULL is vb_fragment_from_device_paths. The encoders' rules hold bit
 * for bit:
 *  - before a ring's first kept segment, a segment is kept when one of its points is EPS-far (1e-12 in x or y) from the ring's
 *    first point (start_tangent_for_line / _quad / _curve); that segment gives the start tangent's end (a line: p0 + 1/3 (e -
 *    p0); a quad: c + 1/3 (p0 - c), or c + 1/3 (e - c) when c is EPS-close to p0; a cubic: the first of c1, c2, e EPS-far from
 *    p0). This is not the span test: with p0.x = 0, c.x = 8e-13 and e.x = -8e-13 the quad is dropped;
 *  - after it, a segment is kept when the span of the last kept end point and the segment's points exceeds EPS in x or y;
 *  - the closing line, the cap markers, SUBPATH_END, the PATH tag, the draw object and draw_index are as above, the last kept
 *    end point standing for the last kept point.
 * The worst case of the allocation does not change: a kept segment's points write two words each, and its tag belongs to its
 * end point. Which path-data rows a point lands in depends on the segments dropped, as above.
 * VB_E_INVALID as vb_fragment_from_device_paths, and also: point_kinds that is not device or managed memory of the renderer's
 * device; checked on the device, naming the first offending row: a kind other than 0 or 1, a ring whose first or last point is
 * off-curve, a third off-curve point in a row. Arcs, TrueType's implied on-curve midpoints (the caller inserts them), dashes and
 * other brushes are not part of it. */
int vb_fragment_from_device_curves(vb_renderer *, const vb_device_paths *, const uint8_t *point_kinds, uint32_t *fragment_out,
                                   uint32_t *n_draw_objects_out);
/* vb_fragment_from_device_dashes: dashed strokes of the paths above (an addition; no vello counterpart): chart grid lines and
 * threshold series, map borders and trails, focus rings and animated "marching ants". d->kind must be 1; point_kinds is as for
 * vb_fragment_from_device_curves (NULL: polylines). The fragment is word for word what vb_fragment_upload receives from a fresh
 * Scene that, for each path i in order, calls
 *     stroke(Stroke{width, join, miter_limit, start_cap, end_cap, pattern, offset_i}, IDENTITY, Color(colors[i]), None, shape_i)
 * offset_i being (double) offsets[i], or `offset` when offsets is NULL, and shape_i the shape of vb_fragment_from_device_curves
 * with one exception: a ring of fewer than two points contributes no element. (The host dasher, kurbo's DashIterator as
 * restated here, turns a closed one-point ring `M p Z` into Z and a segment left over from the rings before it; the undashed
 * calls write nothing for such rings.) So the dashes are the host's bit for bit: each ring is dashed on its own, the phase
 * starting again at each ring; every cut is made in f64 (pieces are sub-segments, their ends rounded to f32 like the host's);
 * the first dash of a ring broken into several comes last, continuing the last dash when a closed ring ends inside one; and a
 * closed ring that stays inside one dash comes out as M p0, its segments but the last, Z, then the last segment, which the
 * encoder draws again from p0 when the path has already kept a segment (visible for a curved closing segment). That last
 * behaviour is the host encoder's, which this call reproduces; it is not checked against kurbo itself. The fragment's
 * allocation is the worst case of vb_fragment_from_device_paths for the dashes' points and sub-rings. The call synchronises
 * vb_stream twice: once to size the dashes, once for the fragment's totals. An animated offset is a new fragment (and a
 * recompose) per frame. Each ring's walk is serial, one warp per ring: a single long ring takes as long as its dashes.
 * VB_E_INVALID as vb_fragment_from_device_curves, and also: dash NULL; kind 0; a pattern NULL, empty, with an entry that is not
 * finite or is below 0, or whose entries sum to 0; a scalar offset that is not finite or lies more than 2^24 pattern entries
 * before the pattern's start; offsets not 4-byte aligned device or managed memory of the renderer's device, or a pitch that is
 * not a multiple of 4, below 4 or 4 GiB or more; dashes of more than 2^31 - 1 points or sub-rings, a ring whose control
 * polygon's length allows 2^31 dash breaks (n_pattern (1.01 length / the pattern's sum + 2), refused before it is walked), or a
 * worst case past 32-bit word offsets. Checked on the device, naming the first offending path: an offset that is not finite or lies more than 2^24
 * pattern entries before the start; a piece's point that is not finite once rounded to f32. */
typedef struct {
    const double *pattern; uint32_t n_pattern; /* host memory: dash, gap, dash, ... lengths */
    double offset;                             /* every path's offset when offsets is NULL */
    const float *offsets; size_t offset_pitch_bytes; /* optional device f32, n_paths rows: path i's offset */
} vb_dash;
int vb_fragment_from_device_dashes(vb_renderer *, const vb_device_paths *, const uint8_t *point_kinds, const vb_dash *dash,
                                   uint32_t *fragment_out, uint32_t *n_draw_objects_out);
int vb_compose(vb_renderer *, const vb_instance *, uint32_t n, vb_layout *layout_out, uint32_t *draw_offsets);
/* vb_recompose: vb_compose, followed by a frame that repaints only what the new instance list changed (an addition; no vello
 * counterpart). It installs exactly the scene vb_compose would (scene, layout, ramps, atlas and draw offsets, byte for byte),
 * with the same errors; on an error the previous scene and the damage state are left as they were. A toolkit recomposes for
 * every edit: a hover colour is a new fragment in the same slot, a popup an inserted instance, a closed dialog a removed one,
 * a raised window a move in z-order. With damage tracking (below) the next frame is then incremental, with the damage between
 * the composition the base frame rendered and the new one, when all of these hold:
 *  - tracking is on and there is a base frame, which rendered the scene being replaced: a composition, with no instance
 *    transforms, draw colours, path points, gradient stops or transforms bound, with no scene installation, binding, view, cell split or tracking switch since, and
 *    hit tests answering from it (no failed frame, vb_run_stages, vb_debug_upload or vb_debug_limit_arena since);
 *  - no other vb_recompose / vb_compose since that frame, and no vb_run_stages before the next one;
 *  - the next frame meets every condition of an incremental frame (size, AA, base colour, destination, one cell, no window).
 * Otherwise it is vb_compose: the next frame is full, and still correct. vb_compose itself always makes the next frame full.
 * The damage: instance k's key is (fragment, has_transform, the six f32 transform words). The old and new instance lists are
 * matched in order between equal keys: common prefix and suffix, then Myers' diff of the middle up to VB_RECOMPOSE_MAX_EDITS
 * insertions and deletions, past that the middle by position. A matched instance counts as changed when one of its images got
 * another atlas slot, pixel source or place, or comes from an override (the compose copies its pixels again); a different
 * ramp row does not count (a ramp's row holds the same bytes wherever it is). The damaged tiles are those of the clipped
 * draw boxes of unmatched and changed instances (old boxes in the base frame, new ones in this frame); both boxes of a matched
 * draw object whose box is not bit for bit the old one (an enclosing open clip came or went); the END_CLIPs after the last
 * instance, paired from the end, when unpaired or when their boxes differ; and vb_add_damage rectangles as usual. The host work
 * is O(instances + patches) like vb_compose's; the frame adds one kernel and the recompose one device copy of the old boxes. */
#define VB_RECOMPOSE_MAX_EDITS 32u
int vb_recompose(vb_renderer *, const vb_instance *, uint32_t n, vb_layout *layout_out, uint32_t *draw_offsets);
/* test-only: vb_recompose's matching on plain keys. match[j] = the old index paired with new key j, or 0xffffffff; returns the
 * middle's edit count, or VB_RECOMPOSE_MAX_EDITS + 1 when it was paired by position */
uint32_t vb_debug_match_instances(const uint32_t *old_keys, uint32_t n_old, const uint32_t *new_keys, uint32_t n_new, uint32_t *match);
/* Bind the instance transforms of the composed scene to device memory (an addition; no vello counterpart). A simulation, an
 * animation or a layout model that writes its instances' transforms on the GPU moves them without a host call per frame:
 *  - Rows. Row k is at device_transforms + k * row_pitch_bytes. It holds six f32 values [a b c d e f] in kurbo Affine order.
 *  - What a frame renders. While the array is bound, every frame renders the scene that vb_compose would have made with the
 *    same fragments in the same order, with instance k as Some(row k). This includes instances that were composed with
 *    has_transform = 0. The scene's products row_k * T are bit-identical to vb_compose given transform = (double)row_k for
 *    every instance: both use the same f32 product (Encoding::append's, without FMA).
 *  - When the array is read. A frame reads the array when it runs on vb_stream, in the frame's first stage (like a view's
 *    coefficients). The caller orders its writes before the frame, on vb_stream or with a synchronisation, and does not write
 *    the array while a frame that reads it is running. A blocking frame that is re-run after an arena overflow reads the same
 *    contents again; an enqueued frame is never re-run (vb_frame_finish). The caller keeps the memory alive while it is bound.
 *    Changing only the contents replays the captured frame graph; nothing crosses PCIe per frame.
 *  - Non-finite rows. If a row has a coefficient that is not finite, that instance keeps the transform it was composed with
 *    (Some(T_k) or None) for that frame.
 *  - Views. A view applies on top: a viewed frame renders V * (row_k * T), the same two f32 products as vb_compose followed by
 *    vb_set_view. Culling to the frame stays tied to the view: on exactly while a view is set (set the identity view to cull
 *    without panning).
 *  - Other state. The binding survives vb_set_cells, vb_set_view and vb_hit_test; hit tests answer from the last frame, bound or
 *    not. Every scene installation unbinds: every upload form, vb_render, vb_render_begin and vb_compose. device_transforms NULL
 *    unbinds; frames then render the scene as composed.
 *  - Fragments. The call copies what it needs from the fragments (their untransformed transforms) and from the compose (each
 *    instance's transform prefix and compose-time transform): freeing fragments afterwards does not affect bound frames.
 *  - Binding, unbinding, or binding another pointer, pitch or n changes the frame's key, so the next frame captures its graph
 *    anew.
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: the current scene was not made by
 * vb_compose; n is 0 or not the last compose's instance count; a pointer that is not device memory of the renderer's device
 * (or managed memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 24, or 4 GiB or more; a fragment of
 * that compose freed before the call; a renderer of a vb_group or with the exchange enabled; a call between vb_render_enqueue
 * and vb_frame_finish; a scene whose bound transforms plus a view's would pass 32-bit word offsets. */
int vb_bind_instance_transforms(vb_renderer *, const float *device_transforms, uint32_t n, size_t row_pitch_bytes);
/* Bind the colours of the installed scene's draw objects to device memory (an addition; no vello counterpart). A hover or
 * selection highlight, a choropleth coloured by a model's output, a particle view coloured by simulation state or a fade changes
 * colours without re-encoding or re-uploading the scene, and without a host call per frame:
 *  - Rows. Row k is at device_rgba + k * row_pitch_bytes. It holds four f32 values r, g, b, a: straight-alpha, sRGB-encoded
 *    components, exactly a vello / peniko Color. Row k belongs to draw object k of the installed scene: the indices vb_hit_test
 *    returns and vb_scene_n_draw_objects / Scene.n_draw_objects counts. In a composed scene they are global (instance i's draws
 *    are draw_offsets[i] ..), and in a batch too (cell c's draws are draw_offsets[c] ..).
 *  - What a frame renders. While rows are bound, every frame renders the scene it would render if draw object k, for every
 *    k < n, had been encoded with Color(row k). This applies to draw objects whose paint is one colour: DRAWTAG_COLOR (solid
 *    fills and strokes) and BLUR_RECT (the colour of draw_blurred_rounded_rect[_in]). Rows of every other draw object
 *    (gradients, images, BEGIN_CLIP, END_CLIP) are ignored; gradients take bound stops instead (vb_bind_gradient_stops).
 *    Draw objects from n on keep the colour they were encoded with.
 *  - Conversion. The colour word is exactly the encoder's premultiply().to_rgba8().to_u32(): p = (r*a, g*a, b*a, a) in f32, and
 *    each channel is clamp(floor(p*255 + 0.5), 0, 255), where p*255 and + 0.5 are rounded separately in f32; r is the low byte.
 *    So a bound frame is byte-identical to uploading the scene re-encoded with those colours.
 *  - Non-finite rows. If any of a row's four values is NaN or +-inf, that draw object keeps its encoded colour for that frame.
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, in the frame's first stage, like bound transforms.
 *    The caller orders its writes before the frame, on vb_stream or with a synchronisation, and does not write the rows while a
 *    frame that reads them is running. A blocking frame that is re-run after an arena overflow reads the same rows again; an
 *    enqueued frame is never re-run. The caller keeps the memory alive while it is bound. Changing only the contents replays the
 *    captured frame graph, with no host call and no PCIe traffic. Binding, unbinding, or binding another pointer, n or pitch
 *    changes the frame's key, so the next frame captures its graph anew. With nothing bound a frame launches, configures and
 *    captures exactly what it would without this call.
 *  - Scope. Every scene installation unbinds: every upload form, vb_render, vb_render_begin, vb_compose and vb_recompose. The
 *    binding survives vb_set_view, vb_set_cells, vb_bind_instance_transforms and hit tests; transforms and colours can be bound
 *    together. device_rgba NULL unbinds; frames then render the scene as encoded.
 *  - Hit tests and hit maps do not change: colour never mattered to them. Damage tracking follows the rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the installed layout's n_draw_objects; a pointer that is not device memory of the renderer's device (or
 * managed memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 16, or 4 GiB or more; a renderer of a
 * vb_group or with the exchange configured; a call between vb_render_enqueue and vb_frame_finish; a scene whose draw data and
 * transform regions past its streams would pass 32-bit word offsets. */
int vb_bind_draw_colors(vb_renderer *, const float *device_rgba, uint32_t n, size_t row_pitch_bytes);
/* Bind the points of the installed scene's paths to device memory (an addition; no vello counterpart). A live chart of a GPU
 * time series, a simulation mesh or cloth outline, polygons a model predicts, a morph between outlines or a graph layout whose
 * edges follow their nodes moves its geometry every frame without re-encoding or re-uploading the scene, and without a host
 * call per frame:
 *  - Rows. Row k is at device_xy + k * row_pitch_bytes and holds two f32 values x, y. Row k is point k of the installed scene's
 *    path-data stream: path-data words 2k and 2k + 1. Points are global in a composed scene or a batch (fragments and cells in
 *    stream order), and they are in the coordinates they were encoded in: the path's transform, bound instance transforms and
 *    a view all still apply on top. vb_scene_n_points / Scene.n_points counts them, read before and after a call to learn the
 *    rows that call produced. The encoders lay points out so:
 *     - a move-to writes 1 point, a line-to, quad-to and cubic-to 1, 2 and 3 (the end point last); a repeated move-to replaces
 *       the one before it, and a segment of zero length writes nothing;
 *     - a closed fill (every fill subpath closes) repeats its start point, as a line-to, when its last point differs from it;
 *     - a stroke ends each subpath with a cap marker: a closed one with a line-to (1 point, the end of its start tangent), an
 *       open one with a quad-to (2 points: its start point, then the end of its start tangent);
 *     - a dash's pieces are separate subpaths; arcs, circles and ellipses are a move-to and cubics, a rounded rectangle a
 *       move-to, then per corner a line-to and its cubics;
 *     - a fill or stroke whose shape encodes nothing writes no point (and no draw object); a push_*_layer whose clip encodes
 *       nothing writes the empty path in its place, 2 points: a line-to from (0, 0) to (0, 0).
 *  - What a frame renders. While rows are bound, every frame renders byte for byte what uploading the scene would render after
 *    overwriting path-data words 2k and 2k + 1, for every k < n, with the f32 bits of row k. The definition is at stream level:
 *    binding never changes tags, so it is not always re-encoding a moved shape, which may drop a repeated move-to or add a
 *    closing point the bound scene does not have. Points from n on keep their encoded values.
 *  - Non-finite rows. If x or y of a row is NaN or +-inf, that point keeps its encoded words for that frame.
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, at the start of flatten's stage, and every
 *    vb_run_stages range that contains flatten reads them again. The caller orders its writes before the frame, on vb_stream
 *    or with a synchronisation, and does not write the rows while a frame that reads them is running. A blocking frame that is
 *    re-run after an arena overflow reads the same rows again; an enqueued frame is never re-run. The caller keeps the memory
 *    alive while it is bound. Changing only the contents replays the captured frame graph, with no host call and no PCIe
 *    traffic. Binding, unbinding, or binding another pointer, n or pitch changes the frame's key, so the next frame captures
 *    its graph anew. With nothing bound a frame launches, configures and captures exactly what it would without this call.
 *  - Scope. Every scene installation unbinds: every upload form, vb_render, vb_render_begin, vb_compose and vb_recompose. The
 *    binding survives vb_set_view, vb_set_cells, vb_bind_instance_transforms, vb_bind_draw_colors, vb_bind_gradient_stops and
 *    hit tests; all four bindings can be active together. device_xy NULL unbinds; frames then render the scene as encoded.
 *  - The call finds each path's first point once, with one kernel over the path tags, and synchronises with vb_stream once to
 *    read back whether the scene has a 16-bit segment. Hit tests and hit maps answer from the bound geometry, and damage
 *    tracking follows the rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the scene's point count (its path-data words / 2); a pointer that is not device memory of the renderer's
 * device (or managed memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 8, or 4 GiB or more; a renderer
 * of a vb_group or with the exchange configured; a call between vb_render_enqueue and vb_frame_finish; a scene with a 16-bit
 * segment (a segment tag without the F32 bit: its points are not f32 pairs; neither encoder emits one); a scene whose path
 * data, draw data and transform regions past its streams would pass 32-bit word offsets. */
int vb_bind_path_points(vb_renderer *, const float *device_xy, uint32_t n, size_t row_pitch_bytes);
/* Bind the stops of the installed scene's gradients to device memory (an addition; no vello counterpart). A heat-map legend or
 * choropleth whose colour scale a model moves, a progress bar or shimmer that slides a stop, gradient-filled chart bars
 * recoloured by live data or the fade of a gradient-filled widget changes its ramps without re-encoding or re-uploading the
 * scene, and without a host call per frame:
 *  - Rows. Row k is at device_stops + k * row_pitch_bytes and holds five f32 values offset, r, g, b, a: a vb_ramp_stop, i.e.
 *    a straight-alpha, sRGB-encoded peniko ColorStop after the brush alpha the encoder applies. Row k is stop k of the
 *    installed scene's ramp patches, concatenated in draw-data order (vello's Resources::color_stops); global in instance order
 *    in a composed scene and in cell order in a batch. vb_scene_n_stops / Scene.n_stops counts them, read before and after a
 *    call to learn the rows that call produced. Only gradients that keep a ramp have stops: a gradient with no stop or one
 *    stop, and a degenerate radial or sweep gradient, is encoded as a colour (vb_bind_draw_colors binds it).
 *  - What a frame renders. While rows are bound, every frame renders byte for byte what vb_scene_upload_streams renders for
 *    the same streams with stop k of the patches replaced by row k, for every k < n. Each gradient keeps its extend mode,
 *    interpolation alpha space and geometry. Offsets may be any finite values (out of order, equal, outside [0, 1]): make_ramp's
 *    walk defines the ramp, on the device exactly as on the host. Stops from n on keep their encoded values.
 *  - Non-finite rows. If any of a row's five values is NaN or +-inf, that stop keeps its encoded values for that frame.
 *  - Scenes. Only a scene whose stops the renderer keeps can be bound: one installed from its streams (vb_scene_upload_streams,
 *    vb_scene_upload_device, vb_render_scene) or by vb_compose / vb_recompose. A scene installed as packed bytes
 *    (vb_scene_upload, vb_render, vb_render_begin) has only its resolved ramps.
 *  - How. Resolves share one ramp row between gradients whose stops are equal, and bound rows may part them, so each bound
 *    gradient (a patch with a stop below n) renders from a row of its own, after the scene's ramps. vb_debug_download("ramps")
 *    returns the rows the last frame read: the scene's, then one per bound gradient in patch order.
 *  - When rows are read, graphs and keys, scope: as vb_bind_draw_colors. Rows are read when the frame runs on vb_stream, in its
 *    first stage (and again by a vb_run_stages range that starts at draw); a blocking re-run after an overflow reads them
 *    again; changing only the contents replays the captured graph; binding, unbinding, or another pointer, n or pitch changes
 *    the frame's key. Every scene installation unbinds; the binding survives views, cells, the three other bindings and hit
 *    tests. device_stops NULL unbinds. With nothing bound a frame launches, configures and captures exactly what it would
 *    without this call.
 *  - The call copies the scene's ramps once on the device and synchronises with vb_stream once. Hit tests and hit maps do not
 *    change, and damage tracking follows the rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed, or one installed as
 * packed bytes; n = 0 with a non-NULL pointer, or n above the scene's stop count; a pointer that is not device memory of the
 * renderer's device (or managed memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 20, or 4 GiB or
 * more; a renderer of a vb_group or with the exchange configured; a call between vb_render_enqueue and vb_frame_finish; a scene
 * whose ramps and one per bound gradient would pass the 30 bits of the (ramp id << 2) | extend word, or whose regions past its
 * streams would pass 32-bit word offsets. */
int vb_bind_gradient_stops(vb_renderer *, const float *device_stops, uint32_t n, size_t row_pitch_bytes);
/* Bind the transform stream of the installed scene to device memory (an addition; no vello counterpart). Sprites, markers,
 * map symbols or widgets a simulation or a layout model places on the GPU move, rotate and scale every frame without
 * re-encoding or re-uploading the scene, and without a host call per frame. Unlike moving their points (vb_bind_path_points),
 * a transform also scales and shears a stroke's width, joins and dashes, and it also places gradients and images (brush
 * transforms, draw_image), clip layers and blurred rectangles:
 *  - Rows. Row k is at device_affines + k * row_pitch_bytes and holds six f32 values [a b c d e f] in kurbo Affine order. Row k
 *    is transform-stream entry k of the installed scene: global in instance order in a composed scene and in cell order in a
 *    batch. vb_scene_n_transforms / Scene.n_transforms counts the entries, read before and after a call to learn the rows that
 *    call produced. The encoders lay the entries out so:
 *     - a call pushes its transform only when it differs from the last entry, so consecutive fills, strokes or layers with
 *       equal transforms share one row, and moving that row moves all of them;
 *     - a brush transform (fill / stroke with brush_transform) is an entry of its own after the shape's, holding the product
 *       transform * brush_transform; the gradient or image is placed by it (it is pushed, like any entry, only when it differs
 *       from the last one). A blurred rectangle likewise pushes transform * translate(centre of its rectangle) after its
 *       shape's. draw_image is a fill with no brush transform: its one entry places both the rectangle and the image;
 *     - a fill whose shape encodes nothing still pushes its transform (and no brush transform), and so does a push_*_layer
 *       with a fill-style clip; a stroke of width 0 pushes nothing.
 *  - What a frame renders. While rows are bound, every frame renders byte for byte what installing the same scene would render
 *    after overwriting transform entry k with the f32 bits of row k, for every finite row k < n. The definition is at stream
 *    level: binding never adds or drops transform tags, so rows that share an entry stay shared. Entries from n on keep their
 *    values. Rows are copied as bits, never multiplied or converted.
 *  - Non-finite rows. If any of a row's six values is NaN or +-inf, that entry keeps, for that frame, the value the frame would
 *    read without this binding (the encoded transform, or the product of bound instance transforms).
 *  - With bound instance transforms (vb_bind_instance_transforms) both bindings apply: a finite row k replaces the product
 *    row_i * T that instance i's binding makes for entry k.
 *  - Views. A view applies on top: a viewed frame renders V * row_k, the same f32 product vb_set_view applies to the scene's
 *    own transforms. Culling to the frame stays tied to the view.
 *  - Singular rows (a zero scale mid-animation) are legal: such a frame renders what the patched upload renders.
 *  - Scenes. Every installation form can be bound, packed bytes included: a packed scene carries its transform stream.
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, at the start of flatten's stage, and a vb_run_stages
 *    range that starts at draw reads them again. The caller orders its writes before the frame, on vb_stream or with a
 *    synchronisation, and does not write the rows while a frame that reads them is running. A blocking frame that is re-run
 *    after an arena overflow reads the same rows again; an enqueued frame is never re-run. The caller keeps the memory alive
 *    while it is bound. Changing only the contents replays the captured frame graph, with no host call and no PCIe traffic.
 *    Binding, unbinding, or binding another pointer, n or pitch changes the frame's key, so the next frame captures its graph
 *    anew. With nothing bound a frame launches, configures and captures exactly what it would without this call.
 *  - Scope. Every scene installation unbinds: every upload form, vb_render, vb_render_begin, vb_compose and vb_recompose. The
 *    binding survives vb_set_view, vb_set_cells, the four other bindings and hit tests; all five can be active together.
 *    device_affines NULL unbinds; frames then render the scene as encoded.
 *  - The call finds each path's transform range once, with one kernel over the path tags, for damage tracking; it does not
 *    synchronise. Hit tests and hit maps answer from the frame's geometry, so they follow the bound transforms, and damage
 *    tracking follows the rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the scene's transform count; a pointer that is not device memory of the renderer's device (or managed
 * memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 24, or 4 GiB or more; a renderer of a vb_group or
 * with the exchange configured; a call between vb_render_enqueue and vb_frame_finish; a scene whose transform, draw-data and
 * path-data regions past its streams would pass 32-bit word offsets. */
int vb_bind_transforms(vb_renderer *, const float *device_affines, uint32_t n, size_t row_pitch_bytes);
/* Bind the visibility of the installed scene's draw objects to device memory (an addition; no vello counterpart). A particle or
 * marker view whose live count changes every frame (compose the maximum, show the live ones), a chart or map whose filter a
 * model changes, and panels, tooltips and selection overlays that appear and disappear change which draw objects are drawn
 * without re-encoding or re-uploading the scene (which would unbind every binding), and without a host call per frame. Unlike
 * a bound colour with alpha 0, hiding works for every paint and for layers, a hidden draw object takes no hit test, and its
 * path costs nothing after flatten:
 *  - Rows. Row k is the byte at device_flags + k * row_pitch_bytes and belongs to draw object k of the installed scene, with
 *    the indices of vb_hit_test and Scene.n_draw_objects: global in a composed scene (instance i owns draw_offsets[i] ..) and
 *    in cell order in a batch. A nonzero byte shows draw object k and 0 hides it. Draw objects from n on are shown.
 *  - What a frame renders. While rows are bound, every frame renders what installing the scene re-encoded without the hidden
 *    draw objects renders: byte for byte in MSAA8 and MSAA16, and in Area up to the last-bit differences the order of a
 *    tile's segments makes in its area sums. Hiding a BEGIN_CLIP (any push_*_layer) hides the whole layer: the push, everything up to its END_CLIP and the
 *    layer's blend or compose effect. The row of an END_CLIP is ignored.
 *  - How. At the start of flatten's stage the frame packs the rows into a bit mask of its own, and flatten emits nothing for the
 *    tags of a hidden path: no line and, under a view, no box point either. Its path box stays empty, so binning, tile_alloc,
 *    coarse and fine never see it, and a hidden BEGIN_CLIP's empty clip empties its layer. Hidden tags still pass the tag scan
 *    and flatten's tag threads, and draw, clip and binning still see every draw object. The draws inside a hidden layer are
 *    flattened unless their own rows hide them too; hide them as well to skip their lines.
 *  - Hit tests and hit maps answer from the frame, so they never return a hidden draw object, nor anything inside a hidden
 *    layer.
 *  - A hidden path is hidden also when its points or transforms are bound (vb_bind_path_points, vb_bind_transforms).
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, at the start of flatten's stage, like bound points,
 *    and a vb_run_stages range that contains flatten reads them again. The caller orders its writes before the frame, on
 *    vb_stream or with a synchronisation. A blocking frame that is re-run after an arena overflow reads the rows again; an
 *    enqueued frame is never re-run. Flatten and damage tracking read only the frame's mask, so rows written while a frame runs
 *    cannot make its kernels disagree. The caller keeps the memory alive while it is bound. Changing only the contents replays
 *    the captured frame graph. Binding, unbinding, or binding another pointer, n or pitch changes the frame's key, so the next
 *    frame captures its graph anew. With nothing bound a frame launches, configures and captures exactly what it would without
 *    this call; bound, it launches one kernel more.
 *  - Scope. Every scene installation unbinds: every upload form, vb_render, vb_render_begin, vb_compose and vb_recompose. The
 *    binding survives vb_set_view, vb_set_cells, the five other bindings and hit tests; all six can be active together.
 *    device_flags NULL unbinds; frames then render every draw object.
 *  - The call makes nothing but the mask's buffer, and does not synchronise unless that grows. Damage tracking follows the rows
 *    (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the scene's draw-object count; a pointer that is not device memory of the renderer's device (or managed
 * memory); a pitch of 0, or of 4 GiB or more; a renderer of a vb_group or with the exchange configured; a call between
 * vb_render_enqueue and vb_frame_finish. */
int vb_bind_draw_visibility(vb_renderer *, const uint8_t *device_flags, uint32_t n, size_t row_pitch_bytes);
/* Bind the line widths of the installed scene's strokes to device memory (an addition; no vello counterpart). Maps, charts and
 * node editors keep road outlines, grid lines and graph edges one width on screen while a view zooms; flow maps and graph
 * layouts draw data-driven widths; hover and selection widen one edge. Each without re-encoding or re-uploading the scene
 * (which would unbind every binding), and without a host call per frame:
 *  - Rows. Row k is the f32 at device_widths + k * row_pitch_bytes and belongs to draw object k of the installed scene, which is
 *    path k: the indices of vb_hit_test and Scene.n_draw_objects, global in a composed scene and in cell order in a batch. Rows
 *    are per draw object, not per style entry: the encoders push a style entry only when it differs from the previous one, so
 *    consecutive strokes of equal width share one entry, and each of them still has a row of its own.
 *  - A row is a line width in the stroke's own coordinates: it plays the part of Stroke::width, and the path's transform,
 *    bound instance transforms, bound transforms and a view all still apply on top. For a constant on-screen width under a
 *    uniform zoom z, write w / z.
 *  - Which rows apply. Row k applies when draw object k is a stroke (it is no layer's BEGIN_CLIP or END_CLIP, and the style
 *    entry in effect at its path's end tag has the STYLE bit), k < n, and the row is finite and > 0. Rows of fills, images, blurred rectangles, layers and END_CLIPs are
 *    ignored. A non-finite, zero or negative row keeps the encoded width for that frame (hiding is vb_bind_draw_visibility's
 *    job). Joins, caps, miter limit and dashes keep their encoded values; dashes are cut on the host along the centreline, so
 *    each dash takes the bound width, and its caps follow.
 *  - What a frame renders. When every bound stroke has a style entry of its own (as when the encoded widths all differ), a
 *    bound frame is byte for byte, in all three AA modes, the frame that installing the scene renders after overwriting the
 *    width word (style_base + 2 s + 1) of that stroke's entry s with the row's bits. In general it is what the scene re-encoded
 *    with those widths renders: byte for byte in MSAA8 and MSAA16, and in Area up to the last-bit differences the order of a
 *    tile's segments makes in its area sums.
 *  - Culling under a view or a window uses the bound width (the reach of a stroke's hull is 0.5 |width| x miter limit), so a
 *    thin stroke just outside the frame that a row widens into it appears.
 *  - Hit tests and hit maps answer from the frame's lines, so they follow the bound widths.
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, at the start of flatten's stage, into a snapshot of
 *    its own (vb_debug_download("stroke_widths"): per draw object the width flatten used, 0 where the encoded width applied),
 *    and a vb_run_stages range that contains flatten reads them again. The caller orders its writes before the frame, on
 *    vb_stream or with a synchronisation. A blocking frame that is re-run after an arena overflow reads the rows again; an
 *    enqueued frame is never re-run. Flatten and damage tracking read only the snapshot, so rows written while a frame runs
 *    cannot make its kernels disagree. The caller keeps the memory alive while it is bound. Changing only the contents replays
 *    the captured frame graph. Binding, unbinding, or binding another pointer, n or pitch changes the frame's key, so the next
 *    frame captures its graph anew. With nothing bound a frame launches, configures and captures exactly what it would without
 *    this call; bound, it launches one kernel more.
 *  - Scope. Any installed scene can be bound, packed bytes included. Every scene installation unbinds: every upload form,
 *    vb_render, vb_render_begin, vb_compose and vb_recompose. The binding survives vb_set_view, vb_set_cells, the six other
 *    bindings and hit tests; all seven can be active together. device_widths NULL unbinds.
 *  - The call makes nothing but the snapshot's buffer, and does not synchronise unless that grows. Damage tracking follows the
 *    rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the scene's draw-object count; a pointer that is not device memory of the renderer's device (or managed
 * memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 4, or 4 GiB or more; a renderer of a vb_group or
 * with the exchange configured; a call between vb_render_enqueue and vb_frame_finish. */
int vb_bind_stroke_widths(vb_renderer *, const float *device_widths, uint32_t n, size_t row_pitch_bytes);
/* Bind the opacity of the installed scene's layers and images to device memory (an addition; no vello counterpart). Panels,
 * map layers, tooltips and Lottie-style groups fade, and images or video frames cross-fade, without re-encoding or re-uploading
 * the scene (which would unbind every binding), and without a host call per frame. A layer's alpha cannot be made from bound
 * colours: a group's alpha is not the product of its children's alphas where they overlap, and gradient and image children
 * have no bound colour.
 *  - Rows. Row k is the f32 at device_alpha + k * row_pitch_bytes and belongs to draw object k of the installed scene: the
 *    indices of vb_hit_test and Scene.n_draw_objects, global in a composed scene and in cell order in a batch. Draw objects
 *    from n on keep their encoded values.
 *  - Which rows apply. A row applies only when it is finite; a NaN or infinite row keeps the encoded words for that frame. A
 *    finite row is first clamped to [0, 1], as vb_scene_push_layer clamps its alpha.
 *     - A layer (the BEGIN_CLIP of any push_*_layer: blend, luminance-mask and clip layers): its alpha becomes the row. The
 *       row of its END_CLIP is ignored.
 *     - A clip layer (blend word CLIP_BLEND_MODE, 0x8003) with a row below 1 is also drawn as a Normal / SrcOver layer (blend
 *       word 3): the frame renders what push_layer(Mix::Normal, Compose::SrcOver, row, ...) renders in place of
 *       push_clip_layer. A clip layer's blend skips the tiles wholly inside its clip, so without the change only its edge tiles
 *       would fade. With a row of 1 the clip layer is drawn exactly as encoded.
 *     - An image (draw_image, or an image brush): the low byte of its sample word becomes int(row * 255 + 0.5), the encoders'
 *       conversion with each step rounded on its own. The row takes the place of the image's alpha times the brush alpha; the
 *       format, alpha type, quality and extends are kept.
 *     - Rows of solid fills, strokes, gradients and blurred rectangles are ignored: bind their colours or stops instead.
 *  - What a frame renders. While rows are bound, every frame renders what installing the scene re-encoded with those alphas
 *    renders (the clip-layer rule included): byte for byte in MSAA8 and MSAA16, and in Area up to the last-bit differences the
 *    order of a tile's segments makes in its area sums. Opacity changes no geometry, so hit tests and hit maps answer as
 *    unbound, even at row 0 (hiding is vb_bind_draw_visibility's job).
 *  - How. The frame reads its draw data from the region past the scene's streams that bound colours and stops write
 *    (vb_debug_download("draw_data")): at the start of flatten's stage one kernel writes the scene's draw data there, with the
 *    bound colour, ramp, alpha, blend and sample words in place of the encoded ones. A vb_run_stages range that starts at draw
 *    writes it again.
 *  - When rows are read. A frame reads the rows when it runs on vb_stream, at the start of flatten's stage. The caller orders its
 *    writes before the frame, on vb_stream or with a synchronisation, and does not write the rows while a frame that reads
 *    them is running. A blocking frame that is re-run after an arena overflow reads the rows again; an enqueued frame is never
 *    re-run. The caller keeps the memory alive while it is bound. Changing only the contents replays the captured frame graph.
 *    Binding, unbinding, or binding another pointer, n or pitch changes the frame's key, so the next frame captures its graph
 *    anew. With nothing bound a frame launches, configures and captures exactly what it would without this call; bound, it
 *    launches one kernel more (the draw-data pass) when neither colours nor stops are bound, and none more when they are.
 *  - Scope. Any installed scene can be bound, packed bytes included. Every scene installation unbinds: every upload form,
 *    vb_render, vb_render_begin, vb_compose and vb_recompose. The binding survives vb_set_view, vb_set_cells, the seven other
 *    bindings and hit tests; all eight can be active together. device_alpha NULL unbinds.
 *  - The call finds the bound words once, with one kernel over the draw tags, and does not synchronise unless its table grows.
 *    Damage tracking follows the rows (see below).
 * VB_E_INVALID (vb_last_error says why), with any previous binding left as it was: no scene installed; n = 0 with a non-NULL
 * pointer, or n above the scene's draw-object count; a pointer that is not device memory of the renderer's device (or managed
 * memory), or not 4-byte aligned; a pitch that is not a multiple of 4, below 4, or 4 GiB or more; a renderer of a vb_group or
 * with the exchange configured; a call between vb_render_enqueue and vb_frame_finish; a scene whose regions past its streams
 * would pass 32-bit word offsets. */
int vb_bind_draw_opacity(vb_renderer *, const float *device_alpha, uint32_t n, size_t row_pitch_bytes);

/* ---- damage tracking: repaint only the tiles that changed since the last frame in the same destination (an addition; vello
 * repaints every frame in full) ----
 * While tracking is on, a frame written into the destination of the renderer's last successful frame re-renders only its
 * damaged 16 x 16 tiles and writes no other pixel; the damaged tiles are byte-identical to a full frame. Off (the default)
 * changes nothing: not the pixels, the launches or the captured graphs.
 *  - Incremental frames. A frame is incremental when tracking is on; the scene installation is the same (no upload form,
 *    vb_compose, vb_render or vb_render_begin since; vb_recompose, and uploads with vb_set_upload_diff on, see there, can keep the frame after them incremental); width, height, AA, base colour and the device destination pointer are
 *    those of the last successful frame (NULL counts as the renderer's own target); the view, the bindings and vb_set_cells are
 *    unchanged; it has one cell and no bin_row / tile_row window; and the renderer is not in a vb_group and has no exchange.
 *    Every other frame is full: it reports every tile as damaged and becomes the base of the next one (a batch or a windowed
 *    frame becomes no base). Host destinations (vb_render_uploaded with a host pointer, vb_render) are always full; use
 *    vb_last_damage to read back only what changed.
 *  - Automatic damage, for composed scenes with bound instance transforms (vb_bind_instance_transforms). Instance k changed if
 *    any transform word the frame reads for it (its bound products, or their viewed ones under a view) differs bit for bit
 *    from the last successful frame's: a non-finite row that falls back to its composed transform is no change. The damage is
 *    the tiles of the clipped boxes of its draw objects (draw_offsets[k] .. draw_offsets[k + 1] of vb_compose) in the last
 *    frame and in this one. A moved open clip or blend layer is covered by its own box. The comparison and the snapshot it
 *    needs are kernels of the frame: moving rows replays the captured graph.
 *  - Automatic damage, for bound draw colours (vb_bind_draw_colors). Draw object d changed if the colour word the frame reads
 *    for it differs bit for bit from the last successful frame's: a row that converts to the same word, or a non-finite row
 *    that falls back to an unchanged encoded word, is no change. The damage is the tiles of its clipped box in the last frame
 *    and in this one, and nothing else; the two boxes are equal unless bound transforms also moved it. A change of opacity can
 *    move fine's occlusion start only inside the draw's own box, so the box covers it. Changing rows replays the captured graph.
 *  - Automatic damage, for bound path points (vb_bind_path_points). Path p changed if the words of one of its bound points that
 *    the frame reads differ bit for bit from the last successful frame's: a non-finite row that falls back to an unchanged
 *    encoded point is no change. The damage is the tiles of the clipped box of draw object p (path p is draw object p) in the
 *    last frame and in this one. A changed clip path changes the boxes of the draws inside it only within its BEGIN_CLIP's own
 *    old and new box, which that draw object contributes.
 *  - Automatic damage, for bound gradient stops (vb_bind_gradient_stops). A bound gradient changed if its 512-texel ramp row
 *    differs byte for byte from the last successful frame's: rows that convert to the same texels are no change. The damage is
 *    the tiles of its draw object's clipped box in the last frame and in this one.
 *  - Automatic damage, for bound transforms (vb_bind_transforms). Transform k changed if the six words the frame reads for it
 *    (the bound region, or the viewed one under a view) differ bit for bit from the last successful frame's: a non-finite row
 *    that falls back to an unchanged word is no change. Path p reads the transforms t_lo(p) .. t_hi(p): t_lo is the one in
 *    effect at its first segment tag (its geometry's), t_hi the one at its end tag (where its brush is placed: a brush
 *    transform, or the same one). When one of them changed, the damage is the tiles of the clipped box of draw object p in the
 *    last frame and in this one. So moving one sprite of two neighbours damages only that sprite's old and new boxes.
 *  - Automatic damage, for bound visibility (vb_bind_draw_visibility). Draw object d changed if its bit of the frame's mask
 *    differs from the last successful frame's: only shown or hidden counts, so a row going from 1 to 2 is no change. The damage
 *    is the tiles of its clipped box in the last frame and in this one; a hidden draw object's box is empty, so that is the box
 *    it has while shown. A shown or hidden layer is covered by its BEGIN_CLIP's box, which holds everything inside the layer.
 *  - Automatic damage, for bound stroke widths (vb_bind_stroke_widths). Draw object d changed if the width its frame used
 *    differs bit for bit from the last successful frame's: a fill's row, or a row that falls back to an unchanged encoded
 *    width, is no change. The damage is the tiles of its clipped box in the last frame and in this one; a widened stroke's box
 *    grows, so the new box covers it.
 *  - Automatic damage, for bound opacity (vb_bind_draw_opacity). Draw object d changed if its opacity word in the frame's draw
 *    data (a layer's alpha word, an image's sample word) differs bit for bit from the last successful frame's: a row that
 *    converts to the same word, a non-finite row that falls back to an unchanged encoded word, and the row of any other draw
 *    object are no change. The damage is the tiles of its clipped box in the last frame and in this one; a layer's is its
 *    BEGIN_CLIP's box, which holds everything inside the layer and the pixels its blend touches.
 *  - vb_set_damage_tracking(on): switching it on, or calling it again with 1, makes the next frame full. VB_E_INVALID on a
 *    renderer of a vb_group or with the exchange configured.
 *  - vb_add_damage: n half-open pixel rectangles rects[4i .. 4i + 3] = x0 y0 x1 y1, clamped to the frame and rounded out to
 *    tiles, added to the next frame's damage in stream order (like vb_set_view's coefficients) on top of the automatic
 *    damage. This is the explicit invalidate: use it for a scene re-uploaded with local edits (which is a full frame anyway,
 *    unless vb_set_upload_diff is on or the edit is written into the resident scene in place), dirty image overrides, or a destination the caller
 *    changed. A frame after vb_mark_override_image_dirty / vb_override_image is full unless rectangles were added since the
 *    last successful frame. No effect while tracking is off or before the first tracked frame. VB_E_INVALID: NULL rects
 *    with n > 0; a frame enqueued and not finished (vb_render_enqueue until vb_frame_finish, vb_render_begin until
 *    vb_readback_wait), since the rectangles are meant for the frame after it.
 *  - vb_last_damage: one byte per tile of the last frame that completed successfully, row-major (height_in_tiles x
 *    width_in_tiles), 1 for a tile that frame rendered, and their count in *n_damaged (either output may be NULL).
 *    Synchronous. VB_E_INVALID: no completed frame, a frame enqueued and not finished, or cap below the tile count; also
 *    when a tracked frame after the last successful one failed for good or was streamed (vb_render_begin), as it rewrote the
 *    mask.
 *  - Unchanged by tracking: flatten, path_count, backdrop and path_tiling run in full, so vb_hit_test answers on an
 *    incremental frame equal those on a full one. vb_debug_fine_traffic counts the damaged tiles only, and after an
 *    incremental frame vb_debug_download("seg_holes") also counts the segment slots of the tiles coarse skipped. */
int vb_set_damage_tracking(vb_renderer *, int on);
/* vb_set_upload_diff: diff re-uploaded scenes against the scene the base frame rendered (an addition; off by default, and off
 * changes nothing). An application that re-encodes its whole scene every frame (vb_render, vb_scene_upload_streams) then gets
 * incremental frames without naming the damage itself. While it and damage tracking are on, a scene installed by
 * vb_scene_upload, vb_scene_upload_streams, vb_scene_upload_device, or the upload inside vb_render / vb_render_scene is compared
 * draw object by draw object, on the device, with the scene the base frame rendered, and the next frame is incremental when
 * all of these hold:
 *  - tracking and the switch are on, and there is a base frame, which rendered the scene being replaced: unbound (no draw
 *    colours, path points, gradient stops, transforms or visibility bound either), one cell, no scene installation, binding, view, cell split or tracking switch since, and hit
 *    tests answering from it (no failed frame, vb_run_stages, vb_debug_upload or vb_debug_limit_arena since);
 *  - the upload is the only scene change since that frame (two uploads without a successful frame between them make the next
 *    frame full), and no vb_run_stages before the next one;
 *  - the next frame meets every condition of an incremental frame (size, AA, base colour, device destination, one cell, no
 *    window).
 * Otherwise the next frame is full, and still correct. vb_compose stays full, vb_recompose keeps its own diff, streamed frames
 * (vb_render_begin) and host destinations stay full; vb_add_damage rectangles and dirty overrides apply as usual.
 * The damage: draw objects are equal when their draw tag and draw data, their path's tag bytes (from the byte after the
 * previous path's end tag through its own) and path data, and the transforms and styles those tags read are the same words,
 * a gradient's ramp row holds the same bytes (a ramp that moved to another row is equal), and an image sits at the same atlas
 * place with the same texels. With m the smaller draw-object count, p the common prefix and s the common suffix (at most
 * m - p), new draw object j pairs with old j below p, with old j + n_old - n_new from n_new - s on, with old j in between when
 * the two are equal, and with nothing otherwise: an order-preserving matching of equal draw objects. The damaged tiles are
 * those of the clipped boxes of unmatched draw objects (old boxes in the base frame, new ones in this frame) and both boxes of
 * a matched pair whose boxes differ. The upload keeps the base's scene, ramps and atlas (a spare set of buffers it writes
 * instead, swapped without a copy; counted in arena_bytes and freed when the switch is turned off), copies the base's draw
 * boxes and records its draw objects on the device; the frame adds three kernels before vb_recompose's damage kernel. Frames
 * without such an upload launch nothing new. VB_E_INVALID (switching on) for a renderer of a vb_group or with the exchange
 * configured. */
int vb_set_upload_diff(vb_renderer *, int on);
int vb_add_damage(vb_renderer *, const uint32_t *rects, uint32_t n);
int vb_last_damage(vb_renderer *, uint8_t *tile_mask, size_t cap, uint32_t *n_damaged);

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
int vb_group_set_view(vb_group *, const double affine[6]); /* vb_set_view on every renderer of the group */

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
