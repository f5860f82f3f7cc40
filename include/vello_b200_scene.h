/* vello_b200_scene.h -- C ABI of the scene-building front end (SURVEY.md section 8 row (f), items 2 and 4).
 *
 * Above the drop-in boundary the reference has `vello::Scene` (vello/src/scene.rs:52-470), the stream encoder
 * `vello_encoding::Encoding` / `PathEncoder` (vello_encoding/src/encoding.rs:26-530, path.rs:425-838) and
 * `Resolver::resolve` (vello_encoding/src/resolve.rs:107-399, gradient ramps ramp_cache.rs:119-155). A Rust caller keeps
 * using those and hands the packed bytes to vb_render (include/vello_b200.h). This header is the same thing for callers
 * WITHOUT a Rust toolchain: a native (C++) implementation producing byte-identical packed scenes, so a C / C++ / Python
 * program can go from shapes to pixels through libvello_b200.so alone. Glyph runs are not covered (they need a font
 * stack); everything else `Scene` offers is.
 *
 * Conventions: transforms are kurbo `Affine` coefficient order [a, b, c, d, e, f] (x' = a x + c y + e), doubles like kurbo;
 * paths are kurbo `PathEl` sequences; colours are straight-alpha sRGB floats like peniko `Color`.
 * All functions return VB_OK (0) or a negative vb_status; none of them touches the GPU.
 */
#ifndef VELLO_B200_SCENE_H
#define VELLO_B200_SCENE_H

#include <stddef.h>
#include <stdint.h>

#include "vello_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vb_scene vb_scene;

/* kurbo::PathEl stream: verbs[i] in {'M','L','Q','C','Z'} consuming 2,2,4,6,0 doubles of `coords` (kurbo/bezpath.rs). */
typedef struct {
    const uint8_t *verbs;
    uint32_t n_verbs;
    const double *coords;
} vb_path;

/* A growable path: kurbo::BezPath plus the `Shape::path_elements(tolerance)` conversions of the kurbo shapes vello's callers
 * use most (kurbo 0.13: rect.rs, line.rs, circle.rs, rounded_rect.rs / arc.rs). vb_pathbuf_view() stays valid until the
 * buffer is changed or freed. vello uses tolerance 0.1 for fills, clips AND
 * non-dashed strokes (Encoding::encode_shape -> PathEncoder::shape, vello_encoding/src/path.rs:655-657); only the CPU dash
 * expansion flattens shapes at 0.01 (scene.rs:404,426). */
typedef struct vb_pathbuf vb_pathbuf;
vb_pathbuf *vb_pathbuf_new(void);
void vb_pathbuf_free(vb_pathbuf *);
void vb_pathbuf_clear(vb_pathbuf *);
int vb_pathbuf_move_to(vb_pathbuf *, double x, double y);
int vb_pathbuf_line_to(vb_pathbuf *, double x, double y);
int vb_pathbuf_quad_to(vb_pathbuf *, double x1, double y1, double x, double y);
int vb_pathbuf_curve_to(vb_pathbuf *, double x1, double y1, double x2, double y2, double x, double y);
int vb_pathbuf_close(vb_pathbuf *);
int vb_pathbuf_rect(vb_pathbuf *, double x0, double y0, double x1, double y1);
int vb_pathbuf_line(vb_pathbuf *, double x0, double y0, double x1, double y1);
int vb_pathbuf_circle(vb_pathbuf *, double cx, double cy, double r, double tolerance);
int vb_pathbuf_rounded_rect(vb_pathbuf *, double x0, double y0, double x1, double y1, double radius, double tolerance);
/* kurbo Ellipse::new(center, radii, x_rotation) (ellipse.rs) and Arc { center, radii, start_angle, sweep_angle, x_rotation }
 * (arc.rs): the closed ellipse, and the open arc starting with a MoveTo; angles in radians. */
int vb_pathbuf_ellipse(vb_pathbuf *, double cx, double cy, double rx, double ry, double x_rotation, double tolerance);
int vb_pathbuf_arc(vb_pathbuf *, double cx, double cy, double rx, double ry, double start_angle, double sweep_angle, double x_rotation,
                   double tolerance);
/* kurbo::BezPath::from_svg (kurbo svg.rs): SVG path data with the commands MmLlHhVvCcSsQqTtAaZz, appended to the buffer;
 * elliptical arcs become cubics. VB_E_INVALID on a syntax error (elements parsed before it stay in the buffer). */
int vb_pathbuf_svg(vb_pathbuf *, const char *path_data);
vb_path vb_pathbuf_view(const vb_pathbuf *);

typedef struct { float r, g, b, a; } vb_color; /* peniko::Color, straight alpha */
typedef struct { float offset; vb_color color; } vb_color_stop; /* peniko::ColorStop */

/* peniko::ImageBrush (image data + sampler). format: 0 RGBA8, 1 BGRA8; alpha_type: 0 straight, 1 premultiplied;
 * quality: 0 low, 1 medium, 2 high; extend: 0 pad, 1 repeat, 2 reflect.
 * `pixels` is referenced, not copied: it must stay valid until the scene is resolved for the last time. Images are placed
 * in the atlas once per distinct pixel buffer (the reference keys its image cache by blob id, image_cache.rs:113). */
typedef struct {
    const uint8_t *pixels; /* height x width x 4 */
    uint32_t width, height;
    uint32_t format, alpha_type, quality, x_extend, y_extend;
    float alpha;
} vb_image;

enum { VB_BRUSH_SOLID = 0, VB_BRUSH_LINEAR = 1, VB_BRUSH_RADIAL = 2, VB_BRUSH_SWEEP = 3, VB_BRUSH_IMAGE = 4 };

/* peniko::Brush. geom: linear {x0,y0,x1,y1}; radial {cx0,cy0,cx1,cy1,r0,r1}; sweep {cx,cy,start_angle,end_angle}. */
typedef struct {
    uint32_t kind;
    vb_color color;             /* VB_BRUSH_SOLID */
    double geom[6];             /* gradients */
    const vb_color_stop *stops; /* gradients */
    uint32_t n_stops;
    uint32_t extend;            /* gradients: 0 pad, 1 repeat, 2 reflect */
    uint32_t premul_interp;     /* gradients: interpolate in premultiplied space (peniko default: 1) */
    const vb_image *image;      /* VB_BRUSH_IMAGE */
} vb_brush;

/* kurbo::Stroke (path.rs:70-120 for the encoded part). A dash pattern is expanded on the CPU exactly where vello does it
 * (Scene::stroke -> kurbo::dash, vello/src/scene.rs:404-438): the path passed with a dashed stroke should have been flattened at
 * tolerance 0.01 (SHAPE_TOLERANCE there), an undashed one at 0.1. */
enum { VB_JOIN_BEVEL = 0, VB_JOIN_MITER = 0x10000000, VB_JOIN_ROUND = 0x20000000 };
enum { VB_CAP_BUTT = 0, VB_CAP_SQUARE = 0x01000000, VB_CAP_ROUND = 0x02000000 };
typedef struct {
    double width;
    uint32_t join, start_cap, end_cap;
    double miter_limit;
    const double *dash_pattern; /* NULL / n_dashes == 0: solid */
    uint32_t n_dashes;
    double dash_offset;
} vb_stroke;

/* kurbo::dash(path, dash_offset, dashes) appended to `out` (kurbo 0.13.1 stroke.rs DashIterator; closed forms for lines, composite
 * Gauss-Legendre arc length + bisection for curves -- same arithmetic as vello_b200/shapes.py `dash`). */
int vb_path_dash(const vb_path *path, double dash_offset, const double *dashes, uint32_t n_dashes, vb_pathbuf *out);

enum { VB_FILL_NON_ZERO = 0, VB_FILL_EVEN_ODD = 1 };

vb_scene *vb_scene_new(void);        /* Scene::new, scene.rs:54 */
void vb_scene_free(vb_scene *);
void vb_scene_reset(vb_scene *);     /* Scene::reset, scene.rs:59 */

/* Scene::fill, scene.rs:316-345. brush_transform may be NULL. */
int vb_scene_fill(vb_scene *, uint32_t fill_rule, const double transform[6], const vb_brush *, const double *brush_transform,
                  const vb_path *);
/* Scene::stroke, scene.rs:347-441 (solid strokes; a zero width draws nothing). */
int vb_scene_stroke(vb_scene *, const vb_stroke *, const double transform[6], const vb_brush *, const double *brush_transform,
                    const vb_path *);
/* Scene::push_layer / push_luminance_mask_layer / push_clip_layer, scene.rs:105-249. The clip is filled with
 * `clip_fill_rule`, or stroked when clip_stroke is not NULL. mix / compose: peniko numeric values (0..15, 128 = clip;
 * 0..13). */
int vb_scene_push_layer(vb_scene *, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, uint32_t mix, uint32_t compose, float alpha,
                        const double transform[6], const vb_path *clip);
int vb_scene_push_luminance_mask_layer(vb_scene *, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, float alpha,
                                       const double transform[6], const vb_path *clip);
int vb_scene_push_clip_layer(vb_scene *, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, const double transform[6],
                             const vb_path *clip);
int vb_scene_pop_layer(vb_scene *);  /* scene.rs:251-254 */
/* Scene::draw_image, scene.rs:443-452. */
int vb_scene_draw_image(vb_scene *, const vb_image *, const double transform[6]);
/* Scene::draw_blurred_rounded_rect, scene.rs:256-314. rect = {x0, y0, x1, y1}. */
int vb_scene_draw_blurred_rounded_rect(vb_scene *, const double transform[6], const double rect[4], vb_color color, double radius,
                                       double std_dev);

/* Scene::draw_blurred_rounded_rect_in, scene.rs:282-314: the same, clipped to `shape` instead of the inflated rectangle. */
int vb_scene_draw_blurred_rounded_rect_in(vb_scene *, const vb_path *shape, const double transform[6], const double rect[4],
                                          vb_color color, double radius, double std_dev);

/* Scene::append, scene.rs:464-469: add everything `src` holds to `dst`, with `transform` (may be NULL) applied in front of
 * src's transforms. Images referenced by src must stay alive like dst's own. */
int vb_scene_append(vb_scene *dst, const vb_scene *src, const double *transform);

/* A batch of n scenes for vb_set_cells: dst is reset, then every scene is appended with the identity transform and its open
 * layers are closed right behind it (the END_CLIP draw tag and PATH tag of vb_scene_pop_layer, which resolve would add at the
 * end of a single scene). draw_offsets (n + 1 entries) receives the draw-object range of each scene. Upload dst as any scene
 * (vb_scene_upload_device, or vb_scene_resolve + vb_scene_upload), then vb_set_cells(r, draw_offsets, n). */
int vb_scene_batch(vb_scene *dst, const vb_scene *const *scenes, uint32_t n, uint32_t *draw_offsets);

/* Resolver::resolve (resolve.rs:183-399) without glyph runs: late-bound gradient ramps (512 premultiplied RGBA8 samples
 * each) and the image atlas are built, their indices patched into the draw data, and the six streams packed. The
 * pointers stay owned by the scene and valid until it is changed, resolved again or freed. */
typedef struct {
    const uint8_t *scene;
    size_t scene_len;
    vb_layout layout;
    const uint32_t *ramps;
    uint32_t ramp_w, ramp_h;
    const uint8_t *atlas;
    uint32_t atlas_w, atlas_h;
} vb_packed;
int vb_scene_resolve(vb_scene *, vb_packed *out);

/* Renderer::render_to_texture (vello/src/lib.rs:474-515) for a vb_scene: resolve + vb_render. */
int vb_render_scene(vb_renderer *, vb_scene *, const vb_params *, void *out, uint32_t out_is_device, vb_frame_stats *);
/* The first half of vb_render_scene: resolve the scene's streams on the device (vb_scene_upload_streams) and leave them uploaded. */
int vb_scene_upload_device(vb_renderer *, vb_scene *, vb_layout *layout_out);

/* Renderer::register_texture / unregister_texture (vello/src/lib.rs:578-603): draw pixels that live in device memory.
 * vb_register_texture fills *out with a fresh key as `pixels` -- an address that no host buffer can have, kept in one
 * process-wide registry -- and the size, and sets an override of that key to device_pixels on this renderer (vb_override_image,
 * same checks). The pixels are RGBA8 with straight alpha (vello's assumption: format 0, alpha_type 0); quality (medium),
 * extends (pad) and alpha (1) are defaults the caller may change. The host resolve (vb_scene_resolve) never reads through such a
 * key and leaves its atlas region zero; a device resolve on a renderer without an override of the key returns VB_E_INVALID
 * (vello panics), so a texture registered on one renderer is not drawn by another. vb_unregister_texture (on the registering
 * renderer) removes the key and its override; its atlas region keeps the pixels copied last until the next device resolve. */
int vb_register_texture(vb_renderer *, const void *device_pixels, uint32_t width, uint32_t height, size_t row_pitch_bytes, vb_image *out);
int vb_unregister_texture(vb_renderer *, const vb_image *);

#ifdef __cplusplus
}
#endif
#endif
