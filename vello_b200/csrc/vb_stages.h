// vb_stages.h -- the stage launchers of k_*.cu and the records they share with the host code (vb_api.cu).
//
// Internal to the library. vb_api.cu and every k_*.cu that defines a launcher include it, so a definition that disagrees with
// its declaration here does not compile. Stage launchers take the frame's config, its device buffers (VbFrameBufs) and their
// own per-call scalars, derive their grids themselves and return the number of kernels they launched.
#ifndef VB_STAGES_H
#define VB_STAGES_H
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "vb_types.h"

struct FlLit; // flatten's scratch records (k_flatten.cu)
struct FlJob;

// The device buffers a frame's launches read and write: the current scene slot's inputs, every intermediate and arena, and
// the look-back regions of the control block with their partition counts. prepare() (vb_api.cu) fills it once every buffer
// has its size. It is part of the key of a captured frame (GraphKey), so it holds launch inputs only, and no padding.
struct VbFrameBufs {
    // scene slot and the renderer's fixed tables
    const uint32_t *scene, *ramps;
    const uint8_t *atlas;
    const uint32_t *mask8, *mask16;
    // fixed-size intermediates
    VbTagMonoid *tag_monoids;
    VbPathBbox *path_bboxes;
    VbDrawMonoid *draw_monoids;
    uint32_t *info_bin_data;
    VbClipInp *clip_inp;
    VbBbox4 *clip_bboxes;
    int32_t *clip_scratch; // vb_clip_scratch_words
    VbBbox4 *draw_bboxes;
    VbBinHeader *bin_headers;
    VbPath *paths;
    uint32_t *tile_start;
    uint2 *cls_list; // fine's cost-ordered tile lists, written by coarse: VB_FINE_CLASSES x (width_in_tiles * tile_rows)
    // bump arenas, and flatten's scratch arenas sized from the lines capacity
    VbLineSoup *lines;
    FlLit *line_scratch;
    FlJob *flatten_jobs;
    uint32_t *flatten_parts; // vb_flatten_part_words
    VbTile *tiles;
    VbSegmentCount *seg_counts;
    VbSegment *segments;
    uint32_t *ptcl, *blend_spill;
    // control block: [VbBump, header words (vb_types.h)] [look-back states], zeroed at the start of every frame
    uint32_t *ctl;
    size_t ctl_words;
    uint32_t *lb_pathtag, *lb_flatten, *lb_draw, *lb_tile, *lb_clip, *lb_backdrop;
    uint32_t parts_pathtag, parts_flatten, parts_draw, parts_tile, parts_backdrop;
    int sm_count; // the grids of the persistent and grid-stride kernels are sized from it

    VbBump *bump() const { return reinterpret_cast<VbBump *>(ctl); }
};

// k_exchange.cu: flatten sharded by tag range, lines and path boxes exchanged through peer memory
#define XG_MAX 8u // GPUs of one box
struct XPeers {
    unsigned char *base[XG_MAX]; // peer s: its arena (own arena at [rank])
    uint32_t rows[XG_MAX + 1];   // stripe boundaries in tile rows
    uint32_t world, rank, n_paths, lines_cap;
    unsigned long long half_bytes;
};

// k_resolve.cu: records of the device resolve, staged by vb_scene_upload_streams
struct RsPatch { uint32_t word, value; };                        // scene[word] = value
struct RsRamp { uint32_t first_stop, n_stops, premul, pad; };     // one gradient ramp: its stops and interpolation space
struct RsStop { float offset, r, g, b, a; };                      // == vb_ramp_stop

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
uint32_t vb_launch_clip(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st);
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
// tile rows cfg.win_ty0..win_ty1 into `out`; `band` picks the launch's tile queue (one of 8 control-block words) and
// cls_order starts the tiles in coarse's cost order
uint32_t vb_launch_fine(const VbConfig &cfg, const VbFrameBufs &b, uint32_t *out, int aa, uint32_t cull, uint32_t band, bool cls_order,
                        cudaStream_t st);
int vb_fine_init_constants(void);

// multi-GPU exchange: send = everything up to raising my flags, recv = wait for the peers, combine the boxes, pull my lines
size_t vb_exchange_half_bytes(uint32_t n_paths, uint32_t lines_cap);
uint32_t vb_exchange_epoch_word(void);
uint32_t vb_launch_exchange_send(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &peers, cudaStream_t st);
uint32_t vb_launch_exchange_recv(const VbConfig &cfg, const VbFrameBufs &b, const XPeers &peers, cudaStream_t st);

// device resolve (vb_scene_upload_streams)
void vb_launch_resolve_finish(uint32_t *scene, uint32_t n_tag_bytes, uint32_t n_open_clips, uint32_t padded_tag_bytes, uint32_t end_clip_word0,
                              const RsPatch *patches, uint32_t n_patches, cudaStream_t st);
void vb_launch_make_ramps(const RsRamp *ramps, const RsStop *stops, uint32_t n_ramps, uint32_t *out, cudaStream_t st);

// k_atlas.cu: images in device memory copied into the atlas, all rectangles in one launch (also called through ctypes by
// tools/atlas_blit_probe.py: keep the symbol and its C signature)
uint32_t vb_atlas_blit_units_per_row(uint32_t w);
uint32_t vb_launch_atlas_blit(const VbBlitRect *rects, uint32_t n, uint64_t total_units, uint8_t *atlas, uint32_t atlas_w, cudaStream_t st);
}

#endif
