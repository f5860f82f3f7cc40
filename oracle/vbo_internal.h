/* vbo_internal.h -- record layouts and helpers shared by the oracle's translation units.
 * TEST INFRASTRUCTURE ONLY (see vbo.h). Layouts are the reference's #[repr(C)] structs:
 * vello_encoding/src/{path.rs:192-222,319-423, draw.rs:61-65,239-250, clip.rs:13-55,
 * binning.rs:8-11, config.rs:24-37,120-154}. */
#ifndef VBO_INTERNAL_H
#define VBO_INTERNAL_H
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vbo.h"

#ifdef VBO_LIBM
/* transcendentals exactly as the Rust CPU shaders get them: the platform libm */
#define M_SINF sinf
#define M_COSF cosf
#define M_ATAN2F atan2f
#define M_ASINF asinf
#define M_ACOSF acosf
#define M_EXPF expf
static inline float M_POW23(float ax) { return powf(ax, 2.0f / 3.0f); }
static inline float M_POWF(float x, float y) { return powf(x, y); }
#else
#include "../vello_b200/csrc/vb_detmath.h"
#define M_SINF vb_sinf
#define M_COSF vb_cosf
#define M_ATAN2F vb_atan2f
#define M_ASINF vb_asinf
#define M_ACOSF vb_acosf
#define M_EXPF vb_expf
#define M_POW23 vb_pow_2_3
#define M_POWF vb_powf_pos
#endif

typedef struct { float x, y; } v2;
static inline v2 V2(float x, float y) { v2 r = {x, y}; return r; }
static inline v2 v2add(v2 a, v2 b) { return V2(a.x + b.x, a.y + b.y); }
static inline v2 v2sub(v2 a, v2 b) { return V2(a.x - b.x, a.y - b.y); }
static inline v2 v2scale(v2 a, float s) { return V2(a.x * s, a.y * s); }
static inline float v2dot(v2 a, v2 b) { return a.x * b.x + a.y * b.y; }
static inline float v2len(v2 a) { return sqrtf(a.x * a.x + a.y * a.y); } /* WGSL length() */
static inline v2 v2normalize(v2 a) { float l = v2len(a); return V2(a.x / l, a.y / l); }
static inline int v2eq(v2 a, v2 b) { return a.x == b.x && a.y == b.y; }

/* WGSL u32(f32)/i32(f32) saturate; C casts are undefined out of range. */
static inline uint32_t f2u_sat(float f) {
    if (!(f > 0.0f)) return 0u;
    if (f >= 4294967296.0f) return 0xffffffffu;
    return (uint32_t)f;
}
static inline int32_t f2i_sat(float f) {
    if (f != f) return 0;
    if (f >= 2147483648.0f) return 2147483647;
    if (f <= -2147483648.0f) return (int32_t)0x80000000;
    return (int32_t)f;
}
static inline float u2f_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f2u_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float signf(float x) { return (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f); }
static inline float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
static inline int32_t clampi(int32_t x, int32_t lo, int32_t hi) { return x < lo ? lo : (x > hi ? hi : x); }
static inline uint32_t span_u(float a, float b) { /* cpu/util.rs:196-198 */
    return f2u_sat(fmaxf(ceilf(fmaxf(a, b)) - floorf(fminf(a, b)), 1.0f));
}

typedef struct { uint32_t trans_ix, pathseg_ix, pathseg_offset, style_ix, path_ix; } TagMonoid;
typedef struct { int32_t x0, y0, x1, y1; uint32_t draw_flags, trans_ix; } PathBbox;
typedef struct { uint32_t path_ix, _pad; float p0[2], p1[2]; } LineSoup;
typedef struct { uint32_t path_ix, clip_ix, scene_offset, info_offset; } DrawMonoid;
typedef struct { uint32_t ix; int32_t path_ix; } ClipInp;
typedef struct { float b[4]; } Bbox4;
typedef struct { uint32_t element_count, chunk_offset; } BinHeader;
typedef struct { uint32_t bbox[4]; uint32_t tiles; uint32_t _pad[3]; } PathRec;
typedef struct { int32_t backdrop; uint32_t segment_count_or_ix; } Tile;
typedef struct { uint32_t line_ix, counts; } SegmentCount;
typedef struct { float p0[2], p1[2]; float y_edge; uint32_t _pad; } Segment;
typedef struct { uint32_t failed, binning, ptcl, tile, seg_counts, segments, blend, lines; } Bump;
typedef struct {
    uint32_t width_in_tiles, height_in_tiles, target_width, target_height, base_color;
    vbo_layout layout;
    uint32_t lines_size, binning_size, tiles_size, seg_counts_size, segments_size, blend_size, ptcl_size;
} Config;

typedef struct { void *p; size_t n, cap, elem; } Vec; /* growable array */
static inline void vec_init(Vec *v, size_t elem) { v->p = NULL; v->n = v->cap = 0; v->elem = elem; }
static inline void vec_free(Vec *v) { free(v->p); v->p = NULL; v->n = v->cap = 0; }
static inline void *vec_reserve(Vec *v, size_t n) { /* ensure capacity for n elements, zero-filling new space */
    if (n > v->cap) {
        size_t nc = v->cap ? v->cap : 64;
        while (nc < n) nc *= 2;
        v->p = realloc(v->p, nc * v->elem);
        memset((char *)v->p + v->cap * v->elem, 0, (nc - v->cap) * v->elem);
        v->cap = nc;
    }
    return v->p;
}
static inline void *vec_resize(Vec *v, size_t n) { vec_reserve(v, n); v->n = n; return v->p; }

struct vbo_ctx {
    const uint32_t *scene; size_t scene_words;
    const uint32_t *ramps; uint32_t n_ramps;
    const uint8_t *atlas; uint32_t atlas_w, atlas_h;
    vbo_params params;
    Config cfg;
    uint32_t win_ty0, win_ty1, win_by0, win_by1; /* tile-row / bin-row window */
    Bump bump;
    Vec tag_monoids, path_bboxes, lines, draw_monoids, info_bin_data, clip_inp, clip_bboxes, draw_bboxes,
        bin_headers, paths, tiles, seg_counts, segments, ptcl, blend_spill;
    Vec tile_counts; /* each tile's crossing count as path_count left it (coarse later overwrites the tile's word) */
    int lines_overridden;
    int threads;
};

/* 0, or -3 when a command, segment slice, draw-info read or blend spill lies outside its buffer */
int vbo_fine(vbo_ctx *c, uint8_t *out);

#endif
