/* vb_types.h -- record layouts of every buffer in the pipeline (host + device).
 *
 * These are the reference's #[repr(C)] layouts, byte for byte, so that each stage's output can be
 * compared with the reference's CPU shaders / our oracle:
 *   vello_encoding/src/path.rs:192-222 (LineSoup, SegmentCount, PathSegment), :319-332 (PathMonoid),
 *   :380-423 (PathBbox, Path, Tile); draw.rs:61-65,239-250; clip.rs:13-55; binning.rs:8-11;
 *   config.rs:24-37 (BumpAllocators), :120-154 (ConfigUniform); the shader/shared/ wgsl headers.
 */
#ifndef VB_TYPES_H
#define VB_TYPES_H
#include <stdint.h>

typedef struct { uint32_t trans_ix, pathseg_ix, pathseg_offset, style_ix, path_ix; } VbTagMonoid;
typedef struct { int32_t x0, y0, x1, y1; uint32_t draw_flags, trans_ix; } VbPathBbox;
typedef struct { uint32_t path_ix, _pad; float p0[2], p1[2]; } VbLineSoup;
typedef struct { uint32_t path_ix, clip_ix, scene_offset, info_offset; } VbDrawMonoid;
typedef struct { uint32_t ix; int32_t path_ix; } VbClipInp;
typedef struct { float x0, y0, x1, y1; } VbBbox4;
typedef struct { uint32_t element_count, chunk_offset; } VbBinHeader;
typedef struct { uint32_t bbox[4]; uint32_t tiles; uint32_t _pad[3]; } VbPath;
typedef struct { int32_t backdrop; uint32_t segment_count_or_ix; } VbTile;
typedef struct { uint32_t line_ix, counts; } VbSegmentCount;
typedef struct { float p0[2], p1[2]; float y_edge; uint32_t _pad; } VbSegment;
typedef struct { uint32_t failed, binning, ptcl, tile, seg_counts, segments, blend, lines; } VbBump;
/* The control block starts with VbBump (8 words) padded to 16; word 8 counts segment slots that backdrop assigned but no
 * CMD_FILL of coarse uses (fills skipped inside a zero-coverage clip, ...): bump.segments - holes = the reference's
 * bump.segments. */
#define VB_CTL_SEG_HOLES 8
/* words 16..23: fine's tile queues, one per launch of a frame (up to 8 read-back bands); the header is 32 words */
#define VB_CTL_FINE_QUEUE 16
/* words 24..31: fill counts of fine's cost-class tile lists (written by coarse) */
#define VB_CTL_FINE_CLASS 24
#define VB_FINE_CLASSES 8
/* words 32..47: per-destination counts and cursors of the multi-GPU line routing (k_exchange.cu) */
#define VB_CTL_XCHG_SCRATCH 32
#define VB_CTL_HEADER_WORDS 64

typedef struct {
    uint32_t n_draw_objects, n_paths, n_clips, bin_data_start;
    uint32_t path_tag_base, path_data_base, draw_tag_base, draw_data_base;
    uint32_t transform_base, style_base;
} VbLayout;

/* ConfigUniform (config.rs:120-154) followed by vello_b200 extensions (stripe window etc.). */
typedef struct {
    uint32_t width_in_tiles, height_in_tiles, target_width, target_height, base_color;
    VbLayout layout;
    uint32_t lines_size, binning_size, tiles_size, seg_counts_size, segments_size, blend_size, ptcl_size;
    /* --- extensions, not part of the reference uniform --- */
    uint32_t win_ty0, win_ty1; /* tile-row window [ty0, ty1) this GPU renders (bin-row stripes) */
    uint32_t win_by0, win_by1; /* same in bin rows */
    uint32_t n_tag_words;      /* padded tag stream length in u32 words */
    uint32_t scene_words;
    uint32_t n_ramps, atlas_w, atlas_h;
    uint32_t out_pitch_px;     /* output row pitch in pixels */
    uint32_t out_row0;         /* first pixel row stored at out[0] (stripe outputs) */
    uint32_t win_cull;         /* 1: a stripe window is set -- flatten skips segments that cannot reach its rows */
    /* Batch (vb_set_cells): the draw objects are split into n_cells ranges cell_draw[c] .. cell_draw[c + 1], each rendered
     * into its own width x height frame. The tile grid is a tall frame of tile_rows = n_cells * height_in_tiles rows; cell c
     * owns tile rows [c * height_in_tiles, (c + 1) * height_in_tiles) and bin rows [c * hB, (c + 1) * hB). width_in_tiles,
     * height_in_tiles and the windows above stay the CELL's. n_cells = 1: no batch (cell_draw unused). */
    uint32_t n_cells, tile_rows;
    const uint32_t *cell_draw; /* device: n_cells + 1 draw-object offsets */
} VbConfig;

/* One rectangle of k_atlas_blit (k_atlas.cu): w x h RGBA8 texels from device memory (rows src_pitch bytes apart, 4-byte
 * aligned) to atlas texel (dst_x, dst_y). unit0 = exclusive prefix of h * spr over the rectangles before it. */
typedef struct {
    const uint8_t *src;
    uint64_t src_pitch;
    uint64_t unit0;
    uint32_t w, h, dst_x, dst_y;
    uint32_t spr, _pad; /* units (16-byte destination windows) per row: vb_atlas_blit_units_per_row(w) */
} VbBlitRect;

#define VB_STAGE_BINNING 0x1u
#define VB_STAGE_TILE_ALLOC 0x2u
#define VB_STAGE_FLATTEN 0x4u
#define VB_STAGE_PATH_COUNT 0x8u
#define VB_STAGE_COARSE 0x10u
#define VB_STAGE_FINE_SEGMENTS 0x20u /* extension: segments arena too small (assigned in k_backdrop, checked in k_path_tiling) */
#define VB_STAGE_EXCHANGE 0x40u      /* extension: multi-GPU line exchange (outbox too small, or a peer never signalled) */
/* the bits coarse and path_tiling skip on: every stage before them. Not each other's: the two run side by side. */
#define VB_STAGES_BEFORE_COARSE (VB_STAGE_BINNING | VB_STAGE_TILE_ALLOC | VB_STAGE_FLATTEN | VB_STAGE_PATH_COUNT | VB_STAGE_EXCHANGE)

#define VB_TILE_WIDTH 16u
#define VB_TILE_HEIGHT 16u
#define VB_N_TILE_X 16u
#define VB_N_TILE_Y 16u
#define VB_N_TILE 256u
#define VB_PTCL_INITIAL_ALLOC 64u
#define VB_PTCL_INCREMENT 256u
#define VB_PTCL_HEADROOM 2u
#define VB_BLEND_STACK_SPLIT 4u

#define VB_DRAWTAG_NOP 0u
#define VB_DRAWTAG_FILL_COLOR 0x44u
#define VB_DRAWTAG_FILL_LIN_GRADIENT 0x114u
#define VB_DRAWTAG_FILL_RAD_GRADIENT 0x29cu
#define VB_DRAWTAG_FILL_SWEEP_GRADIENT 0x254u
#define VB_DRAWTAG_FILL_IMAGE 0x28Cu
#define VB_DRAWTAG_BLURRED_ROUNDED_RECT 0x2d4u
#define VB_DRAWTAG_BEGIN_CLIP 0x49u
#define VB_DRAWTAG_END_CLIP 0x21u

#define VB_CMD_END 0u
#define VB_CMD_FILL 1u
#define VB_CMD_SOLID 3u
#define VB_CMD_COLOR 5u
#define VB_CMD_LIN_GRAD 6u
#define VB_CMD_RAD_GRAD 7u
#define VB_CMD_SWEEP_GRAD 8u
#define VB_CMD_IMAGE 9u
#define VB_CMD_BEGIN_CLIP 10u
#define VB_CMD_END_CLIP 11u
#define VB_CMD_JUMP 12u
#define VB_CMD_BLUR_RECT 13u

#endif
