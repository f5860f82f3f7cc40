// vb_stages.h -- the stage launchers of k_*.cu and the records they share with the host code (vb_renderer.h).
//
// Internal to the library. The host files and every k_*.cu that defines a launcher include it, so a definition that disagrees with
// its declaration here does not compile. Stage launchers take the frame's config, its device buffers (VbFrameBufs) and their
// own per-call scalars, derive their grids themselves and return the number of kernels they launched.
#ifndef VB_STAGES_H
#define VB_STAGES_H
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "vb_resolve.h"
#include "vb_types.h"

// k_resolve.cu: records of the device resolve, staged by vb_scene_upload_streams and vb_compose (and RsPatch, vb_resolve.h)
struct RsRamp { uint32_t first_stop, n_stops, premul, pad; };     // one gradient ramp: its stops and interpolation space
struct RsStop { float offset, r, g, b, a; };                      // == vb_ramp_stop

struct FlLit; // flatten's scratch records (k_flatten.cu)
struct FlJob;
struct CmpXform; // an instance's transform (k_compose.cu, below)
struct VbUdiff;  // the upload diff's state (k_upload_diff.cu, below)

// The bindings of a scene to device rows that every frame reads (vb_bind_*): instance transforms, draw colours, path points,
// gradient stops, transforms, visibility, stroke widths and opacity. Binding k's rows are `n` rows `pitch` bytes apart from
// `rows`, null while unbound.
enum { VB_BIND_INSTANCES, VB_BIND_COLORS, VB_BIND_POINTS, VB_BIND_STOPS, VB_BIND_TRANSFORMS, VB_BIND_VISIBILITY, VB_BIND_WIDTHS, VB_BIND_OPACITY,
       VB_N_BINDINGS };
struct VbRows {
    const uint8_t *rows;
    uint32_t n, pitch;
};
// What is bound, as the renderer keeps it and each frame reads it (VbFrameBufs::bound): the rows, and the tables each binding
// made at bind time (vb_compose.cu), null or 0 while it is unbound.
struct VbBound {
    VbRows rows[VB_N_BINDINGS];
    // instances (k_instance_transforms): the exclusive prefix of their transform counts (n + 1), their compose-time transforms
    // (n), the fragments' untransformed transforms, and their draw prefix for damage tracking (n + 1: instance k draws draw
    // objects inst_draw[k] .. inst_draw[k + 1])
    const uint32_t *inst_prefix;
    const CmpXform *inst_xf;
    const uint32_t *inst_src, *inst_draw;
    // colours, stops or opacity (k_draw_data): per draw-data word of the scene, the draw object whose binding replaces it, or
    // VB_COLOR_NONE; null while none of them is bound
    const uint32_t *dd_slots;
    // stops (k_bound_ramps): the bound gradients (rs_grads_n RsRamp records over the scene's stop indices), their encoded
    // stops, and per draw object its bound gradient or VB_COLOR_NONE (k_draw_data, k_damage). Gradient g's ramp row is ramps +
    // (rs_ramp0 + g) * 512.
    const RsRamp *rs_grads;
    const RsStop *rs_stops;
    const uint32_t *rs_draw;
    // points (k_path_points): each path's first point (layout.n_paths + 1; k_damage maps changed points to paths with it)
    const uint32_t *pt_first;
    // transforms: the range of transforms each path reads (layout.n_paths {t_lo, t_hi}; k_damage)
    const uint2 *xf_range;
    uint32_t rs_grads_n, rs_ramp0;
};

// Damage tracking's state of a frame (vb_set_damage_tracking; k_damage.cu), filled by damage_prepare (vb_damage.cu) and all
// zero while tracking is off.
struct VbDamage {
    // the frame's damage (one byte per tile), the caller's rectangles staged for the next frame (vb_add_damage), and while
    // anything is bound the snapshot (vb_dmg_layout)
    uint8_t *mask, *pending;
    uint32_t *snap;
    // set only for the first frame after a diff that tracking follows, null otherwise: a recompose's (vb_recompose;
    // k_recompose.cu) or an upload's (vb_set_upload_diff; k_upload_diff.cu). The base frame's draw boxes and k_recompose_damage's
    // tables (vb_rcmp_tables); for an upload also the diff's buffer (VbUdiff, then vb_udiff_layout), whose tables describe one
    // draw object per "instance".
    const VbBbox4 *old_boxes;
    const uint32_t *tables;
    VbUdiff *udiff;
    // VB_DMG_OFF, VB_DMG_FULL (render everything, record the snapshot) or VB_DMG_INCREMENTAL (coarse and fine only for damaged
    // tiles); the transforms the frame reads (at layout.transform_base)
    uint32_t mode, n_xf;
    // the diff's old and new instances and draw objects (the END_CLIPs after the last instance included)
    uint32_t n_old, n_new, old_draws, new_draws;
};
static_assert(sizeof(VbDamage) == 6 * sizeof(void *) + 6 * sizeof(uint32_t), "VbDamage has no padding (GraphKey is compared bytewise)");

// The device buffers a frame's launches read and write: the current scene slot's inputs, every intermediate and arena, and
// the look-back regions of the control block with their partition counts. prepare() (vb_frame.cu) fills it once every buffer
// has its size. It is part of the key of a captured frame (GraphKey), so it holds launch inputs only, and no padding.
struct VbFrameBufs {
    // scene slot and the renderer's fixed tables
    const uint32_t *scene, *ramps;
    const uint8_t *atlas;
    const uint32_t *mask8, *mask16;
    const float *view; // the view's six f32 coefficients (vb_set_view), written in stream order; read by k_view_transforms
    // what is bound to device rows (VbBound), and the scene's own words the bound regions are made from: its draw data, path
    // data and transforms (the bound transform region's source without bound instance transforms). Null while unbound.
    VbBound bound;
    const uint32_t *dd_src, *pt_src, *xf_src;
    // fixed-size intermediates
    VbTagMonoid *tag_monoids;
    VbPathBbox *path_bboxes;
    uint2 *path_draw; // per path: {style_ix, trans_ix}, written by pathtag for draw (what flatten's path_bboxes fields come from)
    VbDrawMonoid *draw_monoids;
    uint32_t *info_bin_data;
    VbClipInp *clip_inp;
    VbBbox4 *clip_bboxes;
    int32_t *clip_scratch; // vb_clip_scratch_words
    VbBbox4 *draw_bboxes;
    VbBinHeader *bin_headers;
    VbPath *paths;
    uint32_t *tile_start;
    uint2 *cls_list; // fine's cost-ordered tile lists, written by coarse: VB_FINE_LISTS x (width_in_tiles * tile_rows)
    // bump arenas, and flatten's scratch arenas sized from the lines capacity
    VbLineSoup *lines;
    FlLit *line_scratch;
    FlJob *flatten_jobs;
    uint32_t *flatten_parts; // vb_flatten_part_words
    VbTile *tiles;
    VbSegmentCount *seg_counts;
    VbSegment *segments;
    uint32_t *ptcl, *blend_spill;
    VbDamage dmg;
    // control block: [VbBump, header words (vb_types.h)] [look-back states], zeroed at the start of every frame
    uint32_t *ctl;
    size_t ctl_words;
    uint32_t *lb_pathtag, *lb_flatten, *lb_draw, *lb_tile, *lb_clip, *lb_backdrop;
    uint32_t parts_pathtag, parts_flatten, parts_draw, parts_tile, parts_backdrop;
    // the lengths of the regions prepare reserved past the scene's streams (regions_of, vb_renderer.h), 0 for an absent one:
    // the transforms of each transform region (the bound one and the viewed one), the words of the bound draw data and of the
    // bound path data. A launcher that writes a region writes this many and no more.
    uint32_t xf_len, dd_len, pd_len, pad;
    int sm_count; // the grids of the persistent and grid-stride kernels are sized from it

    VbBump *bump() const { return reinterpret_cast<VbBump *>(ctl); }
};

// The words of the visibility mask of a scene: one bit per draw object, and per path (path p is draw object p).
static inline uint32_t vb_vis_words(const VbLayout &L) {
    return ((L.n_draw_objects > L.n_paths ? L.n_draw_objects : L.n_paths) + 31u) / 32u;
}

// k_exchange.cu: flatten sharded by tag range, lines and path boxes exchanged through peer memory
#define XG_MAX 8u // GPUs of one box
struct XPeers {
    unsigned char *base[XG_MAX]; // peer s: its arena (own arena at [rank])
    uint32_t rows[XG_MAX + 1];   // stripe boundaries in tile rows
    uint32_t world, rank, n_paths, lines_cap;
    unsigned long long half_bytes;
};


extern "C" {
// stages, in pipeline order
uint32_t vb_launch_pathtag(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_pathtag_parts(uint32_t n_tag_words);
// partitions [part_base, part_end) of the tag stream (0, parts_flatten: all); clear_bboxes: reset the path boxes first
uint32_t vb_launch_flatten(const VbConfig &cfg, const VbFrameBufs &b, bool clear_bboxes, uint32_t part_base, uint32_t part_end,
                           cudaStream_t st);
uint32_t vb_flatten_parts(uint32_t n_tag_words);
size_t vb_flatten_part_words(uint32_t n_parts);
void vb_flatten_arena_bytes(uint32_t cap_lines, size_t *lit_bytes, size_t *job_bytes);
uint32_t vb_launch_draw(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_draw_parts(uint32_t n_draw);
// clip in two launchers: the depth scan and the links read only draw's clip_inp, the boxes also the path boxes flatten writes
uint32_t vb_launch_clip_links(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_clip_bboxes(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_clip_parts(uint32_t n_clips);
size_t vb_clip_scratch_words(uint32_t n_clips);
uint32_t vb_launch_binning(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_tile_alloc(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_tile_alloc_parts(uint32_t n_draw);
uint32_t vb_launch_path_count(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_backdrop(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_backdrop_parts(uint32_t tiles_size);
uint32_t vb_launch_coarse(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_path_tiling(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
// Where fine stores a frame. Without `dst`: RGBA8 at `out`, cfg.out_pitch_px pixels a row, frame row cfg.out_row0 at out[0].
// With `dst` (a registered destination other than linear RGBA8 with straight alpha; the FI_DST instantiations): texels of
// `texel` bytes (4: 8-bit, 8: RGBA16F, 16: RGBA32F) with straight or, with `premul`, premultiplied alpha, cfg.out_pitch_px
// texels a row. An 8-bit pixel's bytes are permuted by __byte_perm selector `swz`. They are stored as without `dst`, or with
// `array` through `surf`, frame pixel (x, y) at texel (x0 + x, y0 + y).
struct VbFineOut {
    uint32_t *out;
    cudaSurfaceObject_t surf;
    uint32_t dst, swz, array, x0, y0, texel, premul;
};
// What fine's tiles start from with `on` (vb_set_background; the FI_BG instantiations), instead of the base colour: texels of
// `texel` bytes (as VbFineOut's), straight or, with `premul`, premultiplied, r and b swapped with `bgra`. Linear: pixel (x, y) of
// cell c at ptr + (c * target_height + y) * pitch + texel * x. With `array`, through `surf`, pixel (x, y) at texel (x0 + x, y0 + y).
// No padding: it is part of the graph key.
struct VbFineBg {
    const uint8_t *ptr;
    cudaSurfaceObject_t surf;
    unsigned long long pitch; // bytes
    uint32_t on, array, x0, y0, texel, premul, bgra, pad;
};
// tile rows cfg.win_ty0..win_ty1 into `o`, over `bg` when bg.on; `band` picks the launch's tile queue (one of 8 control-block
// words) and cls_order starts the tiles in coarse's cost order
uint32_t vb_launch_fine(const VbConfig &cfg, const VbFrameBufs &b, const VbFineOut &o, const VbFineBg &bg, int aa, uint32_t cull,
                        uint32_t band, bool cls_order, cudaStream_t st);
int vb_fine_init_constants(void);

// multi-GPU exchange: send = everything up to raising my flags, recv = wait for the peers, combine the boxes, pull my lines
size_t vb_exchange_half_bytes(uint32_t n_paths, uint32_t lines_cap);
uint32_t vb_exchange_epoch_word(void);
uint32_t vb_launch_exchange_send(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &peers, cudaStream_t st);
uint32_t vb_launch_exchange_recv(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &peers, cudaStream_t st);

// views (k_view.cu): store the coefficients m[6] at dst in stream order; write V * T of every scene transform to the view region
void vb_launch_view_set(float *dst, const float m[6], cudaStream_t st);
uint32_t vb_launch_view_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// hit testing (k_hit.cu): for n points xy (interleaved f32 pairs, device memory) the last draw object covering each of them
// in the finished frame `cfg` / `b` describe, or -1 (vb_hit_test); reads the frame's buffers and writes only draw_ix
uint32_t vb_launch_hit_test(const VbConfig &cfg, const VbFrameBufs &b, const float *xy, uint32_t n, int32_t *draw_ix, cudaStream_t st);
// hit maps (k_hit.cu): the same answer at every pixel centre of the rectangle [x0, x0 + w) x [y0, y0 + h) of the tall frame,
// pixel (i, j) at (char *)draw_ix + j * pitch + 4 * i (vb_hit_map); the rectangle must lie inside the frame
uint32_t vb_launch_hit_map(const VbConfig &cfg, const VbFrameBufs &b, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, int32_t *draw_ix,
                           size_t pitch, cudaStream_t st);

// device resolve (vb_scene_upload_streams)
void vb_launch_resolve_finish(uint32_t *scene, uint32_t n_tag_bytes, uint32_t n_open_clips, uint32_t padded_tag_bytes, uint32_t end_clip_word0,
                              const RsPatch *patches, uint32_t n_patches, cudaStream_t st);
void vb_launch_make_ramps(const RsRamp *ramps, const RsStop *stops, uint32_t n_ramps, uint32_t *out, cudaStream_t st);
// bound gradient stops (vb_bind_gradient_stops). Per frame, in flatten's stage after the draw data (vb_frame.cu): each bound
// gradient's ramp row from its stops, each read from the caller's row when it is bound and finite, else as encoded; nothing
// while unbound. k_draw_data (k_colors.cu) points each bound gradient's ramp word at its row.
uint32_t vb_launch_bound_ramps(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_compose.cu: the six streams of a composition of resident fragments (vb_compose), staged by vb_compose.cu
struct CmpXform { float m[6]; uint32_t on, pad; }; // an instance's transform (on == 0: appended without one)
struct CmpArgs {
    uint32_t *scene;              // the packed scene being composed
    const uint32_t *prefix;       // 6 x (n + 1): per stream, the exclusive prefix of the instances' lengths (path tags in bytes,
                                  // transforms in transforms, the other streams in words)
    const unsigned long long *src; // n: each instance's fragment allocation, which starts with the word offsets of its streams
    const CmpXform *xf;           // n
    uint32_t n;
    uint32_t dst[6];              // the streams' Layout offsets in words
    uint32_t units[6];            // destination units per stream: tag words, words, transforms (stream 4), words
    uint32_t cta0[6];             // first CTA of each stream (set by the launcher)
};
uint32_t vb_launch_compose(CmpArgs a, cudaStream_t st);
// A fragment's allocation starts with CMP_HEADER_WORDS words: the word offset of each of its six streams, then two zeros.
#define CMP_HEADER_WORDS 8u

// k_device_paths.cu: a fragment built from device arrays (vb_fragment_from_device_paths, vb_fragment_from_device_curves). The
// caller's arrays, the style, the scratch the four launches share and the fragment they write. The scratch: per ring the end
// point of its first kept segment and the last end point kept by the span test (set to all ones and zero), the last end point
// of a dropped segment that may need the encoders' walk (zero), its record {last kept end point, code, start tangent end}; a
// keep byte per end point of a walked ring; a kept flag per path (zero); the error (all ones until a check fails: (kind << 32)
// | first row); the look-back (vb_lookback_words(n_parts, 3), its leading words zero); each partition's exclusive prefix (3
// words); the totals of tag bytes, path-data words and draw objects (zero), which the caller reads back.
// ring_flags (optional, one byte per ring; the dashes' sub-rings, k_device_dashes.cu) replaces the uniform closing: a ring
// closes when it has VB_DP_RING_CLOSED, and a VB_DP_RING_CONDITIONAL ring is kept only after a kept unconditional ring of its
// path: path_min (all ones) gets each path's lowest such ring.
#define VB_DP_ERR_RING_OFFSETS 1u
#define VB_DP_ERR_PATH_OFFSETS 2u
#define VB_DP_ERR_POINTS 3u
#define VB_DP_ERR_COLOR 4u
#define VB_DP_ERR_KINDS 5u // a kind other than 0 or 1; an off-curve point first or last in its ring, or third in a row
#define VB_DP_ERR_DASH_OFFSETS 6u // a dash offset that is not finite, or whose pre-roll into the pattern passes 2^24 steps
#define VB_DP_RING_CLOSED 1u
#define VB_DP_RING_CONDITIONAL 2u
struct DpArgs {
    const float *points;
    const uint8_t *kinds; // null: every point on-curve
    const int32_t *ring_offsets, *path_offsets; // path_offsets null: one ring per path
    const float *colors;
    size_t point_pitch, color_pitch; // bytes
    uint32_t n_points, n_rings, n_paths, n_parts;
    uint32_t kind, closed, style_flags, style_width; // kind 0 fill, 1 stroke; the style entry's two words
    uint32_t *ring_first, *ring_last, *ring_odd;
    uint4 *rings;
    uint8_t *keep_fix;
    uint32_t *path_kept;
    unsigned long long *err;
    uint32_t *lookback, *part_excl, *totals;
    uint32_t *fragment;
    int32_t *draw_index; // optional
    const uint8_t *ring_flags; // optional: VB_DP_RING_* per ring
    uint32_t *path_min;
};
uint32_t vb_device_paths_parts(uint32_t n_points);
uint32_t vb_launch_device_paths(const DpArgs &a, cudaStream_t st);
// the first launch alone: the checks (and the per-ring tables they fill, ring_first, ring_last and ring_odd)
uint32_t vb_launch_device_paths_checks(const DpArgs &a, cudaStream_t st);

// k_device_dashes.cu: the dashes of vb_fragment_from_device_dashes, cut on the device into an intermediate of sub-rings that
// k_device_paths.cu encodes (ring_flags). The input arrays (as DpArgs), the pattern (device f64) and the offsets: per path
// (offsets, f32 rows) or one pre-rolled phase for all (scalar_rem, scalar_ix: the dash index, bit 31 set when not drawn). The
// scratch: per path its pre-rolled phase; the error word DpArgs::err; per ring its record {points, sub-rings, S's points, S's
// sub-rings} and its exclusive prefix {points, sub-rings}, entry n_rings the totals (zero when there is no ring), saturating at
// 2^31; the look-back (vb_lookback_words(n_parts, 2), its leading words zero). The intermediate: f32 points (8 bytes apart),
// a kind per point, ring offsets (totals.y + 1), path offsets over the sub-rings (n_paths + 1) and a VB_DP_RING_* per sub-ring.
struct DdArgs {
    const float *points;
    const uint8_t *kinds;
    const int32_t *ring_offsets, *path_offsets;
    size_t point_pitch;
    uint32_t n_points, n_rings, n_paths, n_parts, closed, n_pattern;
    const double *pattern;
    double pattern_period; // the sum of the pattern's entries (> 0)
    const float *offsets;
    size_t offset_pitch;
    double scalar_rem;
    uint32_t scalar_ix;
    double *phase_rem;
    uint32_t *phase_ix;
    unsigned long long *err;
    uint4 *rec;
    uint2 *excl;
    uint32_t *lookback;
    float *out_points;
    uint8_t *out_kinds, *out_flags;
    int32_t *out_ring_offsets, *out_path_offsets;
};
uint32_t vb_device_dashes_parts(uint32_t n_rings);
uint32_t vb_launch_device_dashes(const DpArgs &checks, const DdArgs &a, cudaStream_t st); // the checks, phases, counts and scan
uint32_t vb_launch_device_dashes_emit(const DdArgs &a, cudaStream_t st);
// bound instance transforms: row_k * T of every transform T of the composed scene into the frame's bound region (prepare,
// vb_frame.cu), in flatten's stage before the view's transforms; nothing while unbound
uint32_t vb_launch_instance_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_colors.cu: the bound draw data of bound colours (vb_bind_draw_colors), gradient stops (vb_bind_gradient_stops) and opacity
// (vb_bind_draw_opacity). The bindings' slot table, once at bind time, from the scene's draw tags at `tags` and its n_words words
// of draw data at `dd`: slots[w] = k for each draw-data word w that b's bindings replace, draw object k's colour, ramp, alpha,
// clip-layer blend or image sample word; and b.rs_draw[k] = g for the gradient draw object k whose ramp word is bound gradient
// g's (grad_dd[g], relative to the draw data). It reads at most n_draw tags, and the caller sets both tables to VB_COLOR_NONE
// first. Per frame, in flatten's stage after the transforms (prepare reserved the region, vb_frame.cu): the scene's draw data
// into the frame's region at layout.draw_data_base, each slot's word replaced by the word its binding makes from its row;
// nothing while none of the three is bound.
#define VB_COLOR_NONE 0xffffffffu
uint32_t vb_launch_draw_data_slots(const VbBound &b, const uint32_t *tags, const uint32_t *dd, uint32_t n_words, uint32_t n_draw,
                                   const uint32_t *grad_dd, uint32_t *slots, cudaStream_t st);
uint32_t vb_launch_draw_data(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_points.cu: bound path points (vb_bind_path_points). The binding's table, once at bind time, from the n_words path tag words
// at `tags`: first[p] = the first point of path p for p <= n_paths (first[n_paths]: the scene's points), and *i16 = 1 when a
// segment tag lacks the F32 bit. Per frame, in flatten's stage after the draw data (prepare reserved the region, vb_frame.cu):
// the scene's path data into the frame's region at layout.path_data_base, the words of each bound point with a finite row
// replaced by the row's bits; nothing while unbound.
// With xf_range (bound transforms; first and i16 may then be null), xf_range[p] = {t_lo, t_hi}: the transforms path p reads are
// t_lo (in effect at its first segment tag) .. t_hi (at its TAG_PATH); the caller sets xf_range to all ones first.
uint32_t vb_launch_path_point_slots(const uint32_t *tags, uint32_t n_words, uint32_t n_paths, uint32_t *first, uint32_t *i16, uint2 *xf_range,
                                    cudaStream_t st);
uint32_t vb_launch_path_points(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_transforms.cu: bound transforms (vb_bind_transforms). Per frame, in flatten's stage after the bound instance transforms and
// before the view's (prepare reserved the region, vb_frame.cu): the bound region's entries below b.xf_n with a finite row get
// the row's bits, the others the scene's own transforms, or keep the bound instance transforms' products; nothing while
// unbound.
uint32_t vb_launch_bound_transforms(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_visibility.cu: bound visibility (vb_bind_draw_visibility). Per frame, at the start of flatten's stage after the path data:
// the caller's rows packed into the mask at cfg.vis (vb_vis_words words; bit k set for a nonzero byte k below b.vis_n and for
// every k from b.vis_n on), which flatten and damage tracking read; nothing while unbound.
uint32_t vb_launch_draw_visibility(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// The entries of the stroke-width snapshot of a scene: one per draw object, and per path (path p is draw object p).
static inline uint32_t vb_width_entries(const VbLayout &L) { return L.n_draw_objects > L.n_paths ? L.n_draw_objects : L.n_paths; }
// k_widths.cu: bound stroke widths (vb_bind_stroke_widths). Per frame, at the start of flatten's stage after the visibility
// mask: entry k of the snapshot at cfg.widths (vb_width_entries floats) is row k when draw object k is a stroke, k < b.rows.n
// and the row is finite and > 0, else 0 (the encoded width); flatten and damage tracking read it; nothing while unbound.
uint32_t vb_launch_stroke_widths(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_damage.cu: damage tracking. vb_launch_damage runs between binning and coarse: the frame's damage mask, and the snapshot
// the next frame compares against; vb_launch_damage_commit, the frame's last kernel, makes that snapshot current when the frame
// succeeded. vb_launch_damage_rects stages caller rectangles (tile ranges x0 y0 x1 y1, clipped) into `pending` in stream order.
#define VB_DMG_OFF 0u
#define VB_DMG_FULL 1u
#define VB_DMG_INCREMENTAL 2u
uint32_t vb_launch_damage(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_damage_commit(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
uint32_t vb_launch_damage_rects(uint8_t *pending, uint32_t width_in_tiles, const uint32_t *tile_rects, uint32_t n, cudaStream_t st);
// The damage snapshot (VbDamage::snap) of a frame with the bindings B, of the scene of layout S, reading n_xf transforms. It
// exists while anything is bound (any_binding): [generation, pad x3] [slot 0] [slot 1] [flags]. A slot holds
//   [the transform words the frame reads (6 n_xf)] [the draw boxes (4 n_draw)] [the colour words of the first n_col draw
//   objects] [the words of the first n_pt points (2 n_pt)] [the ramp rows of the n_grads bound gradients (512 n_grads)] [the
//   n_vis words of the visibility mask] [the stroke widths the first n_wid draw objects were drawn with (their snapshot entry,
//   or for 0 the encoded width word of their path's style)] [the opacity words the first n_op draw objects were drawn with (a
//   layer's alpha word, an image's sample word, 0 for any other draw object)].
// The flags, which k_damage_begin and k_damage_mark rewrite every frame, are one per bound instance, with points or visibility
// bound one per path, and with transforms bound one per transform. Offsets are in words: a section's from the start of its
// slot, a flag array's from the start of the snapshot (0: absent).
#define VB_DMG_HEADER_WORDS 4u
struct VbDmgLayout {
    uint32_t n_xf, n_draw, n_col, n_pt, n_grads, n_vis, n_wid, n_op, n_inst, n_paths;
    size_t box, col, pt, ramp, vis, wid, op, slot_words;
    size_t changed, paths, xf, bytes;
};
static inline VbDmgLayout vb_dmg_layout(const VbBound &B, const VbLayout &S, uint32_t n_xf) {
    const VbRows *k = B.rows;
    VbDmgLayout L;
    L.n_xf = n_xf, L.n_draw = S.n_draw_objects, L.n_inst = k[VB_BIND_INSTANCES].n, L.n_paths = S.n_paths;
    L.n_col = k[VB_BIND_COLORS].n, L.n_pt = k[VB_BIND_POINTS].n, L.n_grads = B.rs_grads_n;
    L.n_vis = k[VB_BIND_VISIBILITY].rows ? vb_vis_words(S) : 0u;
    L.n_wid = k[VB_BIND_WIDTHS].n;
    L.n_op = k[VB_BIND_OPACITY].n;
    L.box = 6u * (size_t)n_xf;
    L.col = L.box + 4u * (size_t)L.n_draw;
    L.pt = L.col + L.n_col;
    L.ramp = L.pt + 2u * (size_t)L.n_pt;
    L.vis = L.ramp + 512u * (size_t)L.n_grads;
    L.wid = L.vis + L.n_vis;
    L.op = L.wid + L.n_wid;
    L.slot_words = L.op + L.n_op;
    size_t end = VB_DMG_HEADER_WORDS + 2u * L.slot_words;
    L.changed = k[VB_BIND_INSTANCES].rows ? end : 0u;
    end += L.changed ? L.n_inst : 0u;
    L.paths = k[VB_BIND_POINTS].rows || k[VB_BIND_VISIBILITY].rows ? end : 0u;
    end += L.paths ? L.n_paths : 0u;
    L.xf = k[VB_BIND_TRANSFORMS].rows ? end : 0u;
    L.bytes = (end + (L.xf ? n_xf : 0u)) * 4u;
    return L;
}
// k_recompose.cu: the damage of the first frame after vb_recompose, ORed into dmg.mask right after vb_launch_damage: the boxes
// of unmatched instances' draw objects, and both boxes of matched draw objects whose boxes differ; nothing while the tables
// are null
#define VB_RCMP_NONE 0xffffffffu
uint32_t vb_launch_recompose_damage(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
// k_recompose_damage's tables at `base` for n_old instances of the base frame's scene and n_new of this frame's: [old draw
// prefix (n_old + 1)] [new draw prefix (n_new + 1)] [new instance -> old instance, or VB_RCMP_NONE (n_new)] [old instance
// unmatched (n_old)], `words` in all. Instance k draws draw objects prefix[k] .. prefix[k + 1]. W is uint32_t or const
// uint32_t, as the caller writes or reads them; sizing passes a null base and reads `words` alone.
extern "C++" {
template <class W> struct VbRcmpTables {
    W *old_pre, *new_pre, *map, *unmatched;
    size_t words;
};
template <class W> __host__ __device__ inline VbRcmpTables<W> vb_rcmp_tables(W *base, uint32_t n_old, uint32_t n_new) {
    const size_t at_new = (size_t)n_old + 1u, at_map = at_new + n_new + 1u, at_unmatched = at_map + n_new;
    return VbRcmpTables<W>{base, base + at_new, base + at_map, base + at_unmatched, at_unmatched + n_old};
}
}

// k_upload_diff.cu: the damage of the first frame after an upload that tracking follows (vb_set_upload_diff). The upload keeps
// the base frame's scene (the renderer's spare buffers), copies its draw boxes and runs vb_launch_upload_records on its
// intermediates; the frame runs vb_launch_upload_diff in coarse's stage, between vb_launch_damage and
// vb_launch_recompose_damage, which then ORs the damage of the tables it built.
// One draw object's inputs, relative to its scene's streams: path tag bytes [tag0, tag1), path data words [pd0, pd1),
// transforms [t0, t1), style words [s0, s1), its draw tag and its draw-data offset in words.
struct VbUdRec { uint32_t tag0, tag1, pd0, pd1, t0, t1, s0, s1, dtag, dd; };
// One side of the diff, as uploaded (layout.transform_base is the scene's own transforms, never a view's).
struct VbUdSide {
    const uint32_t *scene, *ramps;
    const uint8_t *atlas;
    VbLayout layout;
    uint32_t n_ramps, atlas_w, atlas_h, pad;
};
// The head of the diff's buffer: the base frame's scene and the uploaded one, written by the upload; and the common prefix and
// suffix lengths, which the frame finds (atomicMin) before it builds the tables.
struct VbUdiff {
    VbUdSide old_side, new_side;
    uint32_t prefix, suffix, pad[2];
};
// The diff's buffer after the head: the base frame's draw boxes (n_old), the records of both scenes (n_old, n_new), the
// positional equality flags (min(n_old, n_new)) and k_recompose_damage's tables (vb_rcmp_tables: identity draw prefixes,
// new -> old or VB_RCMP_NONE, old unmatched).
struct VbUdLayout { size_t boxes, old_rec, new_rec, eq, tables, bytes; };
static inline VbUdLayout vb_udiff_layout(uint32_t n_old, uint32_t n_new) {
    const size_t m = n_old < n_new ? n_old : n_new;
    VbUdLayout u;
    u.boxes = (sizeof(VbUdiff) + 15u) & ~(size_t)15u;
    u.old_rec = u.boxes + (size_t)n_old * sizeof(VbBbox4);
    u.new_rec = u.old_rec + (size_t)n_old * sizeof(VbUdRec);
    u.eq = u.new_rec + (size_t)n_new * sizeof(VbUdRec);
    u.tables = u.eq + m * 4u;
    u.bytes = u.tables + vb_rcmp_tables((uint32_t *)nullptr, n_old, n_new).words * 4u;
    return u;
}
// the records of a scene's n_draw draw objects from its tag and draw monoids; `init` (nullable) gets [m, m], the starting
// prefix and suffix of the frame's matching
uint32_t vb_launch_upload_records(const uint32_t *scene, uint32_t path_tag_base, uint32_t draw_tag_base, uint32_t n_tag_words, uint32_t n_draw,
                                  const VbTagMonoid *tag_monoids, const VbDrawMonoid *draw_monoids, VbUdRec *out, uint32_t *init, uint32_t m,
                                  cudaStream_t st);
// the new scene's records, the equality of the draw objects paired by position and from the end, and the tables; nothing while
// b.dmg.udiff is null
uint32_t vb_launch_upload_diff(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);

// k_atlas.cu: images in device memory copied into the atlas, all rectangles in one launch (also called through ctypes by
// tools/atlas_blit_probe.py: keep the symbol and its C signature)
uint32_t vb_atlas_blit_units_per_row(uint32_t w);
uint32_t vb_launch_atlas_blit(const VbBlitRect *rects, uint32_t n, uint64_t total_units, uint8_t *atlas, uint32_t atlas_w, cudaStream_t st);

// k_debug_lookback.cu (test-only, vb_debug_lookback): the words per partition of look-back `op` (VB_LOOKBACK_*), 0 for an
// unknown op; one launch of n_parts partitions over the zeroed look-back state lb_mem (vb_lookback_words(n_parts, K) words)
uint32_t vb_debug_lookback_words(int op);
uint32_t vb_launch_debug_lookback(int op, uint32_t n_parts, uint32_t *lb_mem, const uint32_t *agg, const uint32_t *delay_ns,
                                  uint32_t *excl, cudaStream_t st);
}

#endif
