/* vbo.h -- CPU ORACLE for the vello GPU compute pipeline.  TEST INFRASTRUCTURE ONLY.
 *
 * This directory is the parity checker for vello_b200's CUDA path. Nothing in the product
 * (vello_b200/, include/, libvello_b200.so) links, imports or calls it; only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.
 *
 * It is a plain-C restatement (not a copy: the reference is Rust + WGSL) of
 *   vello_shaders/src/cpu/{pathtag_reduce,pathtag_scan,bbox_clear,flatten,euler,draw_reduce,
 *                          draw_leaf,clip_leaf,binning,tile_alloc,path_count,backdrop,coarse,
 *                          path_tiling,util}.rs
 * plus `fine` restated from vello_shaders/shader/fine.wgsl + shared/blend.wgsl (the reference
 * has no usable CPU fine: cpu/fine.rs:111 is a dead draft). Every function cites the lines it
 * follows. Where the Rust CPU twin and the WGSL differ, WGSL wins (the reference's tests use the
 * GPU as source of truth, vello_tests/README.md); the divergences are listed in oracle/README.md.
 *
 * Parity pin: the reference cannot be built here (no Rust toolchain, SURVEY.md section 8c), so the
 * oracle is pinned against the reference's own golden vectors instead: the in-repo smoke PNGs
 * and the exact-pixel property tests (tests/test_oracle_golden.py).
 */
#ifndef VBO_H
#define VBO_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vbo_ctx vbo_ctx;

typedef struct {
    uint32_t n_draw_objects, n_paths, n_clips, bin_data_start;
    uint32_t path_tag_base, path_data_base, draw_tag_base, draw_data_base;
    uint32_t transform_base, style_base;
} vbo_layout; /* == vello_encoding::Layout, resolve.rs:16-39 */

typedef struct {
    uint32_t width, height;
    uint32_t base_color; /* premultiplied RGBA8, r in the low byte (config.rs:183) */
    uint32_t aa;         /* 0 area, 1 msaa8, 2 msaa16 */
    /* bin-row window [bin_row0, bin_row1) for stripe rendering; 0,0 = whole image */
    uint32_t bin_row0, bin_row1;
} vbo_params;

enum {
    VBO_STAGE_PATHTAG = 0,
    VBO_STAGE_FLATTEN,
    VBO_STAGE_DRAW,
    VBO_STAGE_CLIP,
    VBO_STAGE_BINNING,
    VBO_STAGE_TILE_ALLOC,
    VBO_STAGE_PATH_COUNT,
    VBO_STAGE_BACKDROP,
    VBO_STAGE_COARSE,
    VBO_STAGE_PATH_TILING,
    VBO_STAGE_FINE,
    VBO_N_STAGES
};

vbo_ctx *vbo_create(void);
void vbo_destroy(vbo_ctx *);

/* Bind inputs (pointers must stay valid until the next vbo_bind / vbo_destroy). */
int vbo_bind(vbo_ctx *, const uint32_t *scene, size_t scene_words, const vbo_layout *,
             const uint32_t *ramps, uint32_t n_ramps, const uint8_t *atlas_rgba8, uint32_t atlas_w,
             uint32_t atlas_h, const vbo_params *);

/* Run stages first..last inclusive (stage enum above). Fine writes `out_rgba8`
 * (width*height*4 bytes, un-premultiplied, row pitch 4*width); may be NULL for earlier stages.
 * Returns 0; -1 fine without `out_rgba8`; -3 fine met a command, segment slice, draw-info read or
 * blend spill outside its buffer (possible only with buffers installed by vbo_set_buffer). */
int vbo_run(vbo_ctx *, int first_stage, int last_stage, uint8_t *out_rgba8);

/* Intermediate buffers by name: "tag_monoids","path_bboxes","lines","draw_monoids","info_bin_data",
 * "clip_inp","clip_bboxes","draw_bboxes","bin_headers","paths","tiles","seg_counts","segments",
 * "ptcl","bump","config", and "tile_counts": one u32 per tile, its crossing count as path_count left it in
 * `segment_count_or_ix` (coarse then overwrites that word; empty until path_count has run for the bound scene).
 * Returns pointer + size in bytes (valid until the next vbo_run). */
const void *vbo_buffer(vbo_ctx *, const char *name, size_t *bytes);

/* Replace an intermediate buffer after vbo_bind (e.g. feed the CUDA path's line soup to the
 * oracle's tile stages). Supported: "lines" and "path_bboxes" (inputs of the tile stages), and
 * "ptcl", "segments", "info_bin_data" and "blend_spill" (the inputs of fine, so that running
 * only fine replays another implementation's command lists). "blend_spill" also sets the spill
 * size (bump.blend): pass as many words as the blend offsets in the installed ptcl were
 * allocated against. Returns -1 for any other name. */
int vbo_set_buffer(vbo_ctx *, const char *name, const void *data, size_t bytes);

/* Number of worker threads for `fine` (per-tile independent). 1 = serial. */
void vbo_set_threads(vbo_ctx *, int n);

/* elementary-function hooks so tests can measure vb_detmath.h against libm */
float vbo_math(int fn, float a, float b);
/* 1 if built with -DVBO_LIBM (transcendentals from libm like the Rust CPU shaders), else 0 */
int vbo_uses_libm(void);

#ifdef __cplusplus
}
#endif
#endif
