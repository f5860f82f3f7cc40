// vb_scene.cpp -- native scene front end: Scene builder, stream encoder, path encoder, resolve / pack.
//
// What it stands in for (for callers without a Rust toolchain; see include/vello_b200_scene.h):
//   vello::Scene                       vello/src/scene.rs:52-470
//   vello_encoding::Encoding           vello_encoding/src/encoding.rs:26-530
//   vello_encoding::PathEncoder        vello_encoding/src/path.rs:425-838   (state machine, stroke cap markers)
//   Style bit layout                   vello_encoding/src/path.rs:11-120
//   draw tags / draw data              vello_encoding/src/draw.rs:17-236
//   f32 -> f16                         vello_encoding/src/math.rs:93-127
//   Resolver::resolve, Layout          vello_encoding/src/resolve.rs:16-39,107-399
//   gradient ramps                     vello_encoding/src/ramp_cache.rs:119-155
// Written from the behaviour of those (and kept byte-identical to vello_b200/encoding.py, the Python statement of the
// same behaviour that the reference's golden images pin): tests/test_scene_native.py compares the packed bytes, layout,
// ramps and atlas of both on every test scene. Plain C++17, no CUDA; all arithmetic that reaches the output is done in
// float exactly where the reference uses f32 (no contraction: this file is compiled with -ffp-contract=off).
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <new>
#include <vector>

#include "../../include/vello_b200_scene.h"
#include "vb_textures.h"

namespace {

constexpr uint8_t TAG_LINE_TO_F32 = 0x9, TAG_QUAD_TO_F32 = 0xA, TAG_CUBIC_TO_F32 = 0xB;
constexpr uint8_t TAG_TRANSFORM = 0x20, TAG_PATH = 0x10, TAG_STYLE = 0x40, TAG_SUBPATH_END_BIT = 0x4;
constexpr uint32_t DRAWTAG_COLOR = 0x44, DRAWTAG_LINEAR_GRADIENT = 0x114, DRAWTAG_RADIAL_GRADIENT = 0x29C, DRAWTAG_SWEEP_GRADIENT = 0x254,
                   DRAWTAG_IMAGE = 0x28C, DRAWTAG_BLUR_RECT = 0x2D4, DRAWTAG_BEGIN_CLIP = 0x49, DRAWTAG_END_CLIP = 0x21;
constexpr uint32_t STYLE_FLAGS_STYLE_BIT = 0x80000000u, STYLE_FLAGS_FILL_BIT = 0x40000000u;
constexpr uint32_t CLIP_BLEND_MODE = 0x8003u, LUMINANCE_MASK_BLEND_MODE = 0x10000u; // draw.rs:215-216
constexpr uint32_t PATH_REDUCE_WG = 256;                                            // config.rs
constexpr uint32_t N_RAMP_SAMPLES = 512;
constexpr float EPS = 1e-12f; // path.rs:841

inline uint32_t f32_bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float bits_f32(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

uint32_t f32_to_f16(float val) { // math.rs:93-127 (float_to_half_fast3)
    const uint32_t INF_32 = 255u << 23, INF_16 = 31u << 23, MAGIC = 15u << 23, ROUND_MASK = ~0xFFFu;
    uint32_t u = f32_bits(val);
    const uint32_t sign = u & 0x80000000u;
    u ^= sign;
    uint32_t out;
    if (u >= INF_32) {
        out = u > INF_32 ? 0x7E00u : 0x7C00u;
    } else {
        u &= ROUND_MASK;
        u = f32_bits(bits_f32(u) * bits_f32(MAGIC));
        u -= ROUND_MASK;
        if (u > INF_16) u = INF_16;
        out = (u >> 13) & 0xFFFFu;
    }
    return out | (sign >> 16);
}

struct Color { float r, g, b, a; };
inline bool operator==(const Color &x, const Color &y) { return x.r == y.r && x.g == y.g && x.b == y.b && x.a == y.a; }
inline Color multiply_alpha(Color c, float m) { return Color{c.r, c.g, c.b, c.a * m}; }
uint32_t premul_rgba8(Color c) { // premultiply().to_rgba8().to_u32(), draw.rs:76-84; r is the low byte
    const float comps[4] = {c.r * c.a, c.g * c.a, c.b * c.a, c.a};
    uint32_t out = 0;
    for (int i = 0; i < 4; i++) {
        double v = std::floor((double)(comps[i] * 255.0f + 0.5f));
        if (!(v > 0.0)) v = 0.0; // also NaN
        if (v > 255.0) v = 255.0;
        out |= (uint32_t)v << (8 * i);
    }
    return out;
}
const Color TRANSPARENT{0.f, 0.f, 0.f, 0.f};

struct Affine {
    double c[6];
};
inline Affine mul(const Affine &a, const Affine &b) { // kurbo Affine * Affine
    Affine r;
    r.c[0] = a.c[0] * b.c[0] + a.c[2] * b.c[1];
    r.c[1] = a.c[1] * b.c[0] + a.c[3] * b.c[1];
    r.c[2] = a.c[0] * b.c[2] + a.c[2] * b.c[3];
    r.c[3] = a.c[1] * b.c[2] + a.c[3] * b.c[3];
    r.c[4] = a.c[0] * b.c[4] + a.c[2] * b.c[5] + a.c[4];
    r.c[5] = a.c[1] * b.c[4] + a.c[3] * b.c[5] + a.c[5];
    return r;
}

struct Stop { float offset; Color color; };
struct RampPatch { uint32_t draw_data_offset; std::vector<Stop> stops; uint32_t extend; bool premul; };
struct ImagePatch { uint32_t draw_data_offset; vb_image image; };
struct Style { uint32_t flags; float width; };
struct Xform { float c[6]; };

struct Encoding {
    std::vector<uint8_t> path_tags;
    std::vector<float> path_data;
    std::vector<uint32_t> draw_tags, draw_data;
    std::vector<Xform> transforms;
    std::vector<Style> styles;
    uint32_t n_paths = 0, n_path_segments = 0, n_clips = 0, n_open_clips = 0;
    std::vector<RampPatch> ramp_patches;
    std::vector<ImagePatch> image_patches;

    void encode_style(Style s) { // encoding.rs: only emitted when it changes
        if (styles.empty() || styles.back().flags != s.flags || !(styles.back().width == s.width)) {
            path_tags.push_back(TAG_STYLE);
            styles.push_back(s);
        }
    }
    void encode_fill_style(uint32_t fill) { encode_style(Style{fill == VB_FILL_EVEN_ODD ? STYLE_FLAGS_FILL_BIT : 0u, 0.0f}); }
    bool encode_stroke_style(const vb_stroke &s) { // path.rs:70-120
        if (s.width == 0.0) return false;
        const uint32_t flags = STYLE_FLAGS_STYLE_BIT | s.join | (s.start_cap << 2) | s.end_cap | f32_to_f16((float)s.miter_limit);
        encode_style(Style{flags, (float)s.width});
        return true;
    }
    bool encode_transform(const Affine &t) {
        Xform x;
        for (int i = 0; i < 6; i++) x.c[i] = (float)t.c[i];
        bool same = !transforms.empty();
        if (same)
            for (int i = 0; i < 6; i++) same = same && transforms.back().c[i] == x.c[i];
        if (!same) {
            path_tags.push_back(TAG_TRANSFORM);
            transforms.push_back(x);
            return true;
        }
        return false;
    }
    void swap_last_path_tags() {
        const size_t n = path_tags.size();
        const uint8_t t = path_tags[n - 1];
        path_tags[n - 1] = path_tags[n - 2];
        path_tags[n - 2] = t;
    }
    void encode_color(Color c) {
        draw_tags.push_back(DRAWTAG_COLOR);
        draw_data.push_back(premul_rgba8(c));
    }
    void encode_begin_clip(uint32_t blend_mode, float alpha) {
        draw_tags.push_back(DRAWTAG_BEGIN_CLIP);
        draw_data.push_back(blend_mode);
        draw_data.push_back(f32_bits(alpha));
        n_clips += 1;
        n_open_clips += 1;
    }
    void encode_end_clip() {
        if (n_open_clips > 0) {
            draw_tags.push_back(DRAWTAG_END_CLIP);
            path_tags.push_back(TAG_PATH);
            n_paths += 1;
            n_clips += 1;
            n_open_clips -= 1;
        }
    }
};

// path.rs:425-838. Coordinates are rounded to f32 on entry.
class PathEncoder {
public:
    PathEncoder(Encoding &e, bool fill) : enc(e), tags(e.path_tags), data(e.path_data), is_fill(fill) {}
    void move_to(float x, float y) {
        if (is_fill) close();
        if (state == MOVETO) {
            data.resize(data.size() - 2);
        } else if (state == NONEMPTY) {
            if (!is_fill) insert_stroke_cap_marker(false);
            if (!tags.empty()) tags.back() |= TAG_SUBPATH_END_BIT;
        }
        first_x = x; first_y = y;
        data.push_back(x); data.push_back(y);
        state = MOVETO;
    }
    void line_to(float x, float y) {
        if (state == START) {
            if (n_encoded_segments == 0) { move_to(x, y); return; }
            move_to(first_x, first_y);
        }
        if (state == MOVETO) {
            if (!neq(x, y, first_x, first_y)) return;
            const float third = 1.0f / 3.0f;
            tan_x = first_x + third * (x - first_x);
            tan_y = first_y + third * (y - first_y);
        }
        if (zero_len(x, y, x, y, x, y)) return;
        data.push_back(x); data.push_back(y);
        tags.push_back(TAG_LINE_TO_F32);
        state = NONEMPTY;
        n_encoded_segments += 1;
    }
    void quad_to(float x1, float y1, float x2, float y2) {
        if (state == START) {
            if (n_encoded_segments == 0) { move_to(x2, y2); return; }
            move_to(first_x, first_y);
        }
        if (state == MOVETO) {
            const float third = 1.0f / 3.0f;
            if (neq(x1, y1, first_x, first_y)) {
                tan_x = x1 + third * (first_x - x1);
                tan_y = y1 + third * (first_y - y1);
            } else if (neq(x2, y2, first_x, first_y)) {
                tan_x = x1 + third * (x2 - x1);
                tan_y = y1 + third * (y2 - y1);
            } else {
                return;
            }
        }
        if (zero_len(x1, y1, x2, y2, x2, y2)) return; // (p3 defaults to p1 in the Python statement; see zero_len)
        data.push_back(x1); data.push_back(y1); data.push_back(x2); data.push_back(y2);
        tags.push_back(TAG_QUAD_TO_F32);
        state = NONEMPTY;
        n_encoded_segments += 1;
    }
    void cubic_to(float x1, float y1, float x2, float y2, float x3, float y3) {
        if (state == START) {
            if (n_encoded_segments == 0) { move_to(x3, y3); return; }
            move_to(first_x, first_y);
        }
        if (state == MOVETO) {
            if (neq(x1, y1, first_x, first_y)) { tan_x = x1; tan_y = y1; }
            else if (neq(x2, y2, first_x, first_y)) { tan_x = x2; tan_y = y2; }
            else if (neq(x3, y3, first_x, first_y)) { tan_x = x3; tan_y = y3; }
            else return;
        }
        if (zero_len(x1, y1, x2, y2, x3, y3)) return;
        data.push_back(x1); data.push_back(y1); data.push_back(x2); data.push_back(y2); data.push_back(x3); data.push_back(y3);
        tags.push_back(TAG_CUBIC_TO_F32);
        state = NONEMPTY;
        n_encoded_segments += 1;
    }
    void empty_path() {
        for (int i = 0; i < 4; i++) data.push_back(0.0f);
        tags.push_back(TAG_LINE_TO_F32);
        n_encoded_segments += 1;
    }
    void close() {
        if (state == START) return;
        if (state == MOVETO) {
            data.resize(data.size() - 2);
            state = START;
            return;
        }
        if (data.size() < 2) return;
        const float lx = data[data.size() - 2], ly = data[data.size() - 1];
        if (f32_bits(lx) != f32_bits(first_x) || f32_bits(ly) != f32_bits(first_y)) { // bitwise, path.rs:661-662
            data.push_back(first_x); data.push_back(first_y);
            tags.push_back(TAG_LINE_TO_F32);
            n_encoded_segments += 1;
        }
        if (!is_fill) insert_stroke_cap_marker(true);
        if (!tags.empty()) tags.back() |= TAG_SUBPATH_END_BIT;
        state = START;
    }
    uint32_t finish(bool insert_path_marker) {
        if (is_fill) close();
        if (state == MOVETO) data.resize(data.size() - 2);
        if (n_encoded_segments != 0) {
            if (!is_fill && state == NONEMPTY) insert_stroke_cap_marker(false);
            if (!tags.empty()) tags.back() |= TAG_SUBPATH_END_BIT;
            enc.n_path_segments += n_encoded_segments;
            if (insert_path_marker) {
                tags.push_back(TAG_PATH);
                enc.n_paths += 1;
            }
        }
        return n_encoded_segments;
    }
    int path_elements(const vb_path &p) {
        const double *c = p.coords;
        for (uint32_t i = 0; i < p.n_verbs; i++) {
            switch (p.verbs[i]) {
            case 'M': move_to((float)c[0], (float)c[1]); c += 2; break;
            case 'L': line_to((float)c[0], (float)c[1]); c += 2; break;
            case 'Q': quad_to((float)c[0], (float)c[1], (float)c[2], (float)c[3]); c += 4; break;
            case 'C': cubic_to((float)c[0], (float)c[1], (float)c[2], (float)c[3], (float)c[4], (float)c[5]); c += 6; break;
            case 'Z': close(); break;
            default: return VB_E_INVALID;
            }
        }
        return VB_OK;
    }

private:
    enum State { START, MOVETO, NONEMPTY };
    Encoding &enc;
    std::vector<uint8_t> &tags;
    std::vector<float> &data;
    float first_x = 0.f, first_y = 0.f, tan_x = 0.f, tan_y = 0.f;
    State state = START;
    uint32_t n_encoded_segments = 0;
    bool is_fill;

    static bool neq(float ax, float ay, float bx, float by) { return std::fabs(ax - bx) > EPS || std::fabs(ay - by) > EPS; }
    // all of (last point, p1, p2, p3) within EPS of each other in both axes
    bool zero_len(float x1, float y1, float x2, float y2, float x3, float y3) const {
        const float x0 = data[data.size() - 2], y0 = data[data.size() - 1];
        const float xmax = std::fmax(std::fmax(x0, x1), std::fmax(x2, x3)), xmin = std::fmin(std::fmin(x0, x1), std::fmin(x2, x3));
        const float ymax = std::fmax(std::fmax(y0, y1), std::fmax(y2, y3)), ymin = std::fmin(std::fmin(y0, y1), std::fmin(y2, y3));
        return !((xmax - xmin) > EPS || (ymax - ymin) > EPS);
    }
    void insert_stroke_cap_marker(bool is_closed) { // path.rs:711-730: carries the start tangent
        if (is_closed) line_to(tan_x, tan_y);
        else quad_to(first_x, first_y, tan_x, tan_y);
    }
};

// ramp_cache.rs:119-155: 512 premultiplied RGBA8 samples
void make_ramp(const std::vector<Stop> &stops, bool premul, uint32_t *out) {
    float last_u = 0.0f, this_u = 0.0f;
    Color last_c = stops[0].color, this_c = last_c;
    size_t j = 0;
    for (uint32_t i = 0; i < N_RAMP_SAMPLES; i++) {
        const float u = (float)i / (float)(N_RAMP_SAMPLES - 1);
        while (u > this_u) {
            last_u = this_u;
            last_c = this_c;
            if (j + 1 < stops.size()) {
                this_u = stops[j + 1].offset;
                this_c = stops[j + 1].color;
                j += 1;
            } else {
                break;
            }
        }
        const float du = this_u - last_u;
        Color c;
        if (du < 1e-9f) {
            c = this_c;
        } else {
            const float t = (u - last_u) / du;
            const Color a = last_c, b = this_c;
            if (premul) { // AlphaColor::lerp: premultiply, lerp_rect, un-premultiply (color crate)
                const float pa[4] = {a.r * a.a, a.g * a.a, a.b * a.a, a.a};
                const float pb[4] = {b.r * b.a, b.g * b.a, b.b * b.a, b.a};
                float pc[4];
                for (int k = 0; k < 4; k++) pc[k] = pa[k] + (pb[k] - pa[k]) * t;
                if (pc[3] == 0.0f || pc[3] == 1.0f) {
                    c = Color{pc[0], pc[1], pc[2], pc[3]};
                } else {
                    const float inv = 1.0f / pc[3];
                    c = Color{pc[0] * inv, pc[1] * inv, pc[2] * inv, pc[3]};
                }
            } else {
                c = Color{a.r + (b.r - a.r) * t, a.g + (b.g - a.g) * t, a.b + (b.b - a.b) * t, a.a + (b.a - a.a) * t};
            }
        }
        out[i] = premul_rgba8(c);
    }
}

} // namespace

struct vb_scene {
    Encoding e;
    // outputs of the last resolve
    std::vector<uint32_t> packed;
    std::vector<uint32_t> ramps;
    std::vector<uint8_t> atlas;
};

namespace {

inline Affine to_affine(const double t[6]) {
    Affine a;
    for (int i = 0; i < 6; i++) a.c[i] = t[i];
    return a;
}
inline Color to_color(vb_color c) { return Color{c.r, c.g, c.b, c.a}; }

bool encode_path(Encoding &e, const vb_path &p, bool is_fill, int *rc) {
    PathEncoder pe(e, is_fill);
    *rc = pe.path_elements(p);
    return pe.finish(true) != 0;
}
void encode_empty_shape(Encoding &e) {
    PathEncoder pe(e, true);
    pe.empty_path();
    pe.finish(true);
}
bool encode_rect(Encoding &e, double x0, double y0, double x1, double y1) { // kurbo Rect::path_elements
    PathEncoder pe(e, true);
    pe.move_to((float)x0, (float)y0);
    pe.line_to((float)x1, (float)y0);
    pe.line_to((float)x1, (float)y1);
    pe.line_to((float)x0, (float)y1);
    pe.close();
    return pe.finish(true) != 0;
}

// encoding.rs:300-470 (encode_brush and the gradient special cases)
int encode_brush(Encoding &e, const vb_brush &b, float alpha) {
    switch (b.kind) {
    case VB_BRUSH_SOLID: {
        const Color c = to_color(b.color);
        e.encode_color(alpha == 1.0f ? c : multiply_alpha(c, alpha));
        return VB_OK;
    }
    case VB_BRUSH_LINEAR:
    case VB_BRUSH_RADIAL:
    case VB_BRUSH_SWEEP: {
        float p[6];
        for (int i = 0; i < 6; i++) p[i] = (float)b.geom[i];
        float t0 = 0.f, t1 = 0.f;
        if (b.kind == VB_BRUSH_RADIAL) {
            if (p[0] == p[2] && p[1] == p[3] && std::fabs((double)p[4] - (double)p[5]) < 1.0 / (1 << 12)) {
                e.encode_color(TRANSPARENT);
                return VB_OK;
            }
        }
        if (b.kind == VB_BRUSH_SWEEP) {
            const float tau = (float)(2.0 * 3.141592653589793);
            t0 = p[2] / tau;
            t1 = p[3] / tau;
            if (std::fabs((double)t0 - (double)t1) < 1.0 / (1 << 15)) {
                e.encode_color(TRANSPARENT);
                return VB_OK;
            }
        }
        if (b.n_stops && !b.stops) return VB_E_INVALID;
        std::vector<Stop> stops(b.n_stops);
        for (uint32_t i = 0; i < b.n_stops; i++) {
            stops[i].offset = b.stops[i].offset;
            stops[i].color = to_color(b.stops[i].color);
            if (alpha != 1.0f) stops[i].color = multiply_alpha(stops[i].color, alpha);
        }
        if (stops.empty()) {
            e.encode_color(TRANSPARENT);
            return VB_OK;
        }
        if (stops.size() == 1) {
            e.encode_color(stops[0].color);
            return VB_OK;
        }
        RampPatch rp;
        rp.draw_data_offset = (uint32_t)e.draw_data.size();
        rp.stops = std::move(stops);
        rp.extend = b.extend;
        rp.premul = b.premul_interp != 0;
        e.ramp_patches.push_back(std::move(rp));
        if (b.kind == VB_BRUSH_LINEAR) {
            e.draw_tags.push_back(DRAWTAG_LINEAR_GRADIENT);
            e.draw_data.push_back(0);
            for (int i = 0; i < 4; i++) e.draw_data.push_back(f32_bits(p[i]));
        } else if (b.kind == VB_BRUSH_RADIAL) {
            e.draw_tags.push_back(DRAWTAG_RADIAL_GRADIENT);
            e.draw_data.push_back(0);
            for (int i = 0; i < 6; i++) e.draw_data.push_back(f32_bits(p[i]));
        } else {
            e.draw_tags.push_back(DRAWTAG_SWEEP_GRADIENT);
            e.draw_data.push_back(0);
            e.draw_data.push_back(f32_bits(p[0]));
            e.draw_data.push_back(f32_bits(p[1]));
            e.draw_data.push_back(f32_bits(t0));
            e.draw_data.push_back(f32_bits(t1));
        }
        return VB_OK;
    }
    case VB_BRUSH_IMAGE: {
        if (!b.image) return VB_E_INVALID;
        const vb_image &im = *b.image;
        const uint32_t a8 = (uint32_t)(int)(im.alpha * alpha * 255.0f + 0.5f) & 0xFFu;
        ImagePatch ip;
        ip.draw_data_offset = (uint32_t)e.draw_data.size();
        ip.image = im;
        e.image_patches.push_back(ip);
        e.draw_tags.push_back(DRAWTAG_IMAGE);
        e.draw_data.push_back(0);
        e.draw_data.push_back((im.width << 16) | (im.height & 0xFFFFu));
        e.draw_data.push_back((im.format << 15) | (im.alpha_type << 14) | (im.quality << 12) | (im.x_extend << 10) | (im.y_extend << 8) | a8);
        return VB_OK;
    }
    default: return VB_E_INVALID;
    }
}

bool stroke_inner(Encoding &e, const vb_stroke &st, const Affine &t, const vb_path &p, int *rc) {
    e.encode_transform(t);
    e.encode_stroke_style(st);
    if (st.n_dashes == 0u || !st.dash_pattern) return encode_path(e, p, false, rc);
    // dashes are cut on the CPU and encoded as the path (vello/src/scene.rs:422-437)
    vb_pathbuf *tmp = vb_pathbuf_new();
    if (!tmp) { *rc = VB_E_INVALID; return false; }
    bool ok = false;
    const int drc = vb_path_dash(&p, st.dash_offset, st.dash_pattern, st.n_dashes, tmp);
    if (drc != VB_OK) {
        *rc = drc;
    } else {
        const vb_path dashed = vb_pathbuf_view(tmp);
        ok = encode_path(e, dashed, false, rc);
    }
    vb_pathbuf_free(tmp);
    return ok;
}

int push_layer_inner(vb_scene *s, uint32_t blend_mode, float alpha, uint32_t fill_rule, const vb_stroke *stroke, const double transform[6],
                     const vb_path *clip) {
    if (!s || !transform || !clip) return VB_E_INVALID;
    Encoding &e = s->e;
    const Affine t = to_affine(transform);
    int rc = VB_OK;
    bool ok;
    if (stroke) {
        if (stroke->width == 0.0) {
            e.encode_fill_style(VB_FILL_NON_ZERO);
            ok = false;
        } else {
            ok = stroke_inner(e, *stroke, t, *clip, &rc);
        }
    } else {
        e.encode_transform(t);
        e.encode_fill_style(fill_rule);
        ok = encode_path(e, *clip, true, &rc);
    }
    if (!ok) encode_empty_shape(e);
    e.encode_begin_clip(blend_mode, alpha);
    return rc;
}

inline float clamp01(float a) { return a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a); }
inline uint32_t align_up(uint32_t n, uint32_t a) { return (n + a - 1) / a * a; }

} // namespace

struct vb_pathbuf {
    std::vector<uint8_t> verbs;
    std::vector<double> coords;
    void el(uint8_t v, std::initializer_list<double> c) {
        verbs.push_back(v);
        coords.insert(coords.end(), c.begin(), c.end());
    }
};

namespace {
// ---- kurbo::dash (kurbo 0.13.1 stroke.rs DashIterator); identical arithmetic to vello_b200/shapes.py `dash` ----------------
struct DSeg { // a path segment in absolute coordinates: k in {'L','Q','C'}, control points p[0..k's degree]
    char k;
    double p[4][2];
};
const double GL8_X[4] = {0.1834346424956498, 0.5255324099163290, 0.7966664774136267, 0.9602898564975363};
const double GL8_W[4] = {0.3626837833783620, 0.3137066458778873, 0.2223810344533745, 0.1012285362903763};
inline void d_lerp(const double a[2], const double b[2], double t, double o[2]) {
    o[0] = a[0] + t * (b[0] - a[0]);
    o[1] = a[1] + t * (b[1] - a[1]);
}
void dseg_eval(const DSeg &s, double t, double o[2]) {
    if (s.k == 'L') { d_lerp(s.p[0], s.p[1], t, o); return; }
    const double mt = 1.0 - t;
    if (s.k == 'Q') {
        for (int c = 0; c < 2; c++) o[c] = mt * mt * s.p[0][c] + 2.0 * mt * t * s.p[1][c] + t * t * s.p[2][c];
        return;
    }
    const double a = mt * mt * mt, b = 3.0 * mt * mt * t, cc = 3.0 * mt * t * t, d = t * t * t;
    for (int c = 0; c < 2; c++) o[c] = a * s.p[0][c] + b * s.p[1][c] + cc * s.p[2][c] + d * s.p[3][c];
}
void dseg_deriv(const DSeg &s, double t, double o[2]) {
    const double mt = 1.0 - t;
    if (s.k == 'Q') {
        for (int c = 0; c < 2; c++) o[c] = 2.0 * (mt * (s.p[1][c] - s.p[0][c]) + t * (s.p[2][c] - s.p[1][c]));
        return;
    }
    const double a = 3.0 * mt * mt, b = 6.0 * mt * t, cc = 3.0 * t * t;
    for (int c = 0; c < 2; c++) o[c] = a * (s.p[1][c] - s.p[0][c]) + b * (s.p[2][c] - s.p[1][c]) + cc * (s.p[3][c] - s.p[2][c]);
}
double dseg_curve_arclen(const DSeg &s, double t0, double t1) { // composite 8-point Gauss-Legendre, 16 pieces
    const int pieces = 16;
    double total = 0.0;
    const double h = (t1 - t0) / pieces;
    for (int i = 0; i < pieces; i++) {
        const double a = t0 + h * i;
        const double mid = a + 0.5 * h, half = 0.5 * h;
        double acc = 0.0;
        for (int q = 0; q < 4; q++) {
            double d0[2], d1[2];
            dseg_deriv(s, mid - half * GL8_X[q], d0);
            dseg_deriv(s, mid + half * GL8_X[q], d1);
            acc += GL8_W[q] * (std::sqrt(d0[0] * d0[0] + d0[1] * d0[1]) + std::sqrt(d1[0] * d1[0] + d1[1] * d1[1]));
        }
        total += acc * half;
    }
    return total;
}
double dseg_arclen(const DSeg &s) {
    if (s.k == 'L') {
        const double dx = s.p[1][0] - s.p[0][0], dy = s.p[1][1] - s.p[0][1];
        return std::sqrt(dx * dx + dy * dy);
    }
    return dseg_curve_arclen(s, 0.0, 1.0);
}
double dseg_inv_arclen(const DSeg &s, double len) {
    if (s.k == 'L') return len / dseg_arclen(s);
    double lo = 0.0, hi = 1.0;
    for (int it = 0; it < 48; it++) {
        const double mid = 0.5 * (lo + hi);
        if (dseg_curve_arclen(s, 0.0, mid) < len) lo = mid;
        else hi = mid;
    }
    return 0.5 * (lo + hi);
}
DSeg dseg_sub(const DSeg &s, double t0, double t1) {
    DSeg r;
    r.k = s.k;
    for (auto &q : r.p) q[0] = q[1] = 0.0;
    if (s.k == 'L') {
        dseg_eval(s, t0, r.p[0]);
        dseg_eval(s, t1, r.p[1]);
    } else if (s.k == 'Q') {
        dseg_eval(s, t0, r.p[0]);
        dseg_eval(s, t1, r.p[2]);
        const double a[2] = {s.p[1][0] - s.p[0][0], s.p[1][1] - s.p[0][1]}, b[2] = {s.p[2][0] - s.p[1][0], s.p[2][1] - s.p[1][1]};
        double d[2];
        d_lerp(a, b, t0, d);
        r.p[1][0] = r.p[0][0] + d[0] * (t1 - t0);
        r.p[1][1] = r.p[0][1] + d[1] * (t1 - t0);
    } else {
        dseg_eval(s, t0, r.p[0]);
        dseg_eval(s, t1, r.p[3]);
        const double scale = (t1 - t0) * (1.0 / 3.0);
        double d0[2], d1[2];
        dseg_deriv(s, t0, d0);
        dseg_deriv(s, t1, d1);
        r.p[1][0] = r.p[0][0] + scale * d0[0];
        r.p[1][1] = r.p[0][1] + scale * d0[1];
        r.p[2][0] = r.p[3][0] - scale * d1[0];
        r.p[2][1] = r.p[3][1] - scale * d1[1];
    }
    return r;
}
struct DEl { char v; double c[6]; };
DEl dseg_to_el(const DSeg &s) {
    DEl e{};
    e.v = s.k;
    if (s.k == 'L') { e.c[0] = s.p[1][0]; e.c[1] = s.p[1][1]; }
    else if (s.k == 'Q') { e.c[0] = s.p[1][0]; e.c[1] = s.p[1][1]; e.c[2] = s.p[2][0]; e.c[3] = s.p[2][1]; }
    else { for (int i = 0; i < 3; i++) { e.c[2 * i] = s.p[i + 1][0]; e.c[2 * i + 1] = s.p[i + 1][1]; } }
    return e;
}
void pb_push(vb_pathbuf &pb, const DEl &e) {
    switch (e.v) {
    case 'M': case 'L': pb.el((uint8_t)e.v, {e.c[0], e.c[1]}); break;
    case 'Q': pb.el('Q', {e.c[0], e.c[1], e.c[2], e.c[3]}); break;
    case 'C': pb.el('C', {e.c[0], e.c[1], e.c[2], e.c[3], e.c[4], e.c[5]}); break;
    default: pb.el('Z', {}); break;
    }
}

int dash_path(const vb_path &in, double dash_offset, const double *dashes, uint32_t n_dashes, vb_pathbuf &out) {
    if (!n_dashes) return VB_E_INVALID;
    enum { NEED_INPUT, TO_STASH, WORKING, FROM_STASH };
    uint32_t dash_ix = 0;
    double dash_remaining = dashes[0] - dash_offset;
    bool is_active = true;
    for (uint32_t guard = 0; dash_remaining < 0.0; guard++) {
        if (guard > (1u << 24)) return VB_E_INVALID; // all-zero / negative pattern
        dash_ix = (dash_ix + 1u) % n_dashes;
        dash_remaining += dashes[dash_ix];
        is_active = !is_active;
    }
    const uint32_t init_dash_ix = dash_ix;
    const double init_dash_remaining = dash_remaining;
    const bool init_is_active = is_active;
    bool input_done = false, closepath_pending = false;
    int state = NEED_INPUT;
    DSeg seg{};
    seg.k = 'L';
    double t = 0.0, seg_remaining = 0.0, start_pt[2] = {0, 0}, last_pt[2] = {0, 0};
    std::vector<DEl> stash;
    size_t stash_ix = 0;
    uint32_t vi = 0;
    size_t ci = 0;
    auto reset_phase = [&]() { dash_ix = init_dash_ix; dash_remaining = init_dash_remaining; is_active = init_is_active; };
    auto handle_closepath = [&]() {
        if (state == TO_STASH) { DEl z{}; z.v = 'Z'; stash.push_back(z); }
        else if (is_active) stash_ix = 1;
        state = FROM_STASH;
        reset_phase();
    };
    auto get_input = [&]() -> int {
        for (;;) {
            if (closepath_pending) { handle_closepath(); break; }
            if (vi >= in.n_verbs) { input_done = true; state = FROM_STASH; return VB_OK; }
            const uint8_t v = in.verbs[vi++];
            const double *c = in.coords + ci;
            const double p0[2] = {last_pt[0], last_pt[1]};
            if (v == 'M') {
                ci += 2;
                if (!stash.empty()) state = FROM_STASH;
                start_pt[0] = last_pt[0] = c[0];
                start_pt[1] = last_pt[1] = c[1];
                reset_phase();
                continue;
            } else if (v == 'L') {
                ci += 2;
                seg.k = 'L';
                seg.p[0][0] = p0[0]; seg.p[0][1] = p0[1]; seg.p[1][0] = c[0]; seg.p[1][1] = c[1];
                last_pt[0] = c[0]; last_pt[1] = c[1];
            } else if (v == 'Q') {
                ci += 4;
                seg.k = 'Q';
                seg.p[0][0] = p0[0]; seg.p[0][1] = p0[1];
                for (int i = 0; i < 2; i++) { seg.p[i + 1][0] = c[2 * i]; seg.p[i + 1][1] = c[2 * i + 1]; }
                last_pt[0] = c[2]; last_pt[1] = c[3];
            } else if (v == 'C') {
                ci += 6;
                seg.k = 'C';
                seg.p[0][0] = p0[0]; seg.p[0][1] = p0[1];
                for (int i = 0; i < 3; i++) { seg.p[i + 1][0] = c[2 * i]; seg.p[i + 1][1] = c[2 * i + 1]; }
                last_pt[0] = c[4]; last_pt[1] = c[5];
            } else if (v == 'Z') {
                closepath_pending = true;
                if (p0[0] != start_pt[0] || p0[1] != start_pt[1]) {
                    seg.k = 'L';
                    seg.p[0][0] = p0[0]; seg.p[0][1] = p0[1]; seg.p[1][0] = start_pt[0]; seg.p[1][1] = start_pt[1];
                    last_pt[0] = start_pt[0]; last_pt[1] = start_pt[1];
                } else {
                    continue;
                }
            } else {
                return VB_E_INVALID;
            }
            seg_remaining = dseg_arclen(seg);
            break;
        }
        t = 0.0;
        return VB_OK;
    };
    int rc = VB_OK;
    auto step = [&](DEl &result) -> bool {
        bool have = false;
        if (state == TO_STASH && stash.empty()) {
            if (is_active) { result = DEl{}; result.v = 'M'; result.c[0] = seg.p[0][0]; result.c[1] = seg.p[0][1]; have = true; }
            else state = WORKING;
        } else if (dash_remaining < seg_remaining) {
            const DSeg rest = dseg_sub(seg, t, 1.0);
            const double t1 = dseg_inv_arclen(rest, dash_remaining);
            if (is_active) {
                result = dseg_to_el(dseg_sub(rest, 0.0, t1));
                state = WORKING;
            } else {
                double pt[2];
                dseg_eval(rest, t1, pt);
                result = DEl{};
                result.v = 'M'; result.c[0] = pt[0]; result.c[1] = pt[1];
            }
            have = true;
            is_active = !is_active;
            t += t1 * (1.0 - t);
            seg_remaining -= dash_remaining;
            dash_ix += 1;
            if (dash_ix == n_dashes) dash_ix = 0;
            dash_remaining = dashes[dash_ix];
        } else {
            if (is_active) { result = dseg_to_el(dseg_sub(seg, t, 1.0)); have = true; }
            dash_remaining -= seg_remaining;
            const int r2 = get_input();
            if (r2) rc = r2;
        }
        return have;
    };
    for (uint64_t guard = 0;; guard++) {
        if (guard > (1ull << 33) || rc) return rc ? rc : VB_E_INVALID;
        if (state == NEED_INPUT) {
            if (input_done) break;
            const int r2 = get_input();
            if (r2) return r2;
            if (input_done) {
                if (stash.empty()) break;
                continue;
            }
            state = TO_STASH;
        } else if (state == TO_STASH) {
            DEl e;
            if (step(e)) stash.push_back(e);
        } else if (state == WORKING) {
            DEl e;
            if (step(e)) pb_push(out, e);
        } else {
            if (stash_ix < stash.size()) {
                pb_push(out, stash[stash_ix++]);
            } else {
                stash.clear();
                stash_ix = 0;
                if (input_done) break;
                if (closepath_pending) { closepath_pending = false; state = NEED_INPUT; }
                else state = TO_STASH;
            }
        }
    }
    return rc;
}
} // namespace

extern "C" int vb_path_dash(const vb_path *path, double dash_offset, const double *dashes, uint32_t n_dashes, vb_pathbuf *out) {
    if (!path || !dashes || !n_dashes || !out || (path->n_verbs && (!path->verbs || !path->coords))) return VB_E_INVALID;
    return dash_path(*path, dash_offset, dashes, n_dashes, *out);
}

namespace {
const double PI = 3.141592653589793;
// kurbo Arc::append_iter: n cubic pieces (n from the tolerance), arm = 4/3 tan(sweep / 4n)
void arc_elements(vb_pathbuf &pb, double cx, double cy, double rx, double ry, double start, double sweep, double x_rot, double tolerance) {
    const double sign = sweep >= 0 ? 1.0 : -1.0;
    const double scaled_err = std::fmax(rx, ry) / tolerance;
    const double n_err = std::fmax(std::pow(1.1163 * scaled_err, 1.0 / 6.0), 3.999999);
    long n = (long)std::ceil(n_err * std::fabs(sweep) * (1.0 / (2.0 * PI)));
    if (n < 1) n = 1;
    const double angle_step = sweep / (double)n;
    const double arm_len = (4.0 / 3.0) * std::fabs(std::tan(0.25 * angle_step)) * sign;
    const double cr = std::cos(x_rot), sr = std::sin(x_rot);
    auto sample = [&](double a, double &ox, double &oy) {
        const double x = rx * std::cos(a), y = ry * std::sin(a);
        ox = cr * x - sr * y;
        oy = sr * x + cr * y;
    };
    auto rot_d = [&](double a, double &ox, double &oy) { // rotated (rx sin a, -ry cos a)
        const double x = rx * std::sin(a), y = -ry * std::cos(a);
        ox = cr * x - sr * y;
        oy = sr * x + cr * y;
    };
    double angle0 = start, p0x, p0y;
    sample(angle0, p0x, p0y);
    for (long i = 0; i < n; i++) {
        const double angle1 = angle0 + angle_step;
        double d0x, d0y, d1x, d1y, p3x, p3y;
        rot_d(angle0, d0x, d0y);
        const double p1x = p0x - arm_len * d0x, p1y = p0y - arm_len * d0y;
        sample(angle1, p3x, p3y);
        rot_d(angle1, d1x, d1y);
        const double p2x = p3x + arm_len * d1x, p2y = p3y + arm_len * d1y;
        pb.el('C', {cx + p1x, cy + p1y, cx + p2x, cy + p2y, cx + p3x, cy + p3y});
        angle0 = angle1;
        p0x = p3x;
        p0y = p3y;
    }
}
} // namespace

extern "C" {

vb_pathbuf *vb_pathbuf_new(void) { return new (std::nothrow) vb_pathbuf(); }
void vb_pathbuf_free(vb_pathbuf *p) { delete p; }
void vb_pathbuf_clear(vb_pathbuf *p) {
    if (p) {
        p->verbs.clear();
        p->coords.clear();
    }
}
int vb_pathbuf_move_to(vb_pathbuf *p, double x, double y) { if (!p) return VB_E_INVALID; p->el('M', {x, y}); return VB_OK; }
int vb_pathbuf_line_to(vb_pathbuf *p, double x, double y) { if (!p) return VB_E_INVALID; p->el('L', {x, y}); return VB_OK; }
int vb_pathbuf_quad_to(vb_pathbuf *p, double x1, double y1, double x, double y) { if (!p) return VB_E_INVALID; p->el('Q', {x1, y1, x, y}); return VB_OK; }
int vb_pathbuf_curve_to(vb_pathbuf *p, double x1, double y1, double x2, double y2, double x, double y) {
    if (!p) return VB_E_INVALID;
    p->el('C', {x1, y1, x2, y2, x, y});
    return VB_OK;
}
int vb_pathbuf_close(vb_pathbuf *p) { if (!p) return VB_E_INVALID; p->el('Z', {}); return VB_OK; }
int vb_pathbuf_rect(vb_pathbuf *p, double x0, double y0, double x1, double y1) { // kurbo Rect::path_elements
    if (!p) return VB_E_INVALID;
    p->el('M', {x0, y0});
    p->el('L', {x1, y0});
    p->el('L', {x1, y1});
    p->el('L', {x0, y1});
    p->el('Z', {});
    return VB_OK;
}
int vb_pathbuf_line(vb_pathbuf *p, double x0, double y0, double x1, double y1) {
    if (!p) return VB_E_INVALID;
    p->el('M', {x0, y0});
    p->el('L', {x1, y1});
    return VB_OK;
}
int vb_pathbuf_circle(vb_pathbuf *p, double cx, double cy, double radius, double tolerance) { // kurbo Circle::path_elements
    if (!p || !(tolerance > 0.0)) return VB_E_INVALID;
    const double r = std::fabs(radius);
    const double scaled_err = r / tolerance;
    long n;
    double arm;
    if (scaled_err < 1.0 / 1.9608e-4) {
        n = 4;
        arm = 0.551915024494;
    } else {
        n = (long)std::ceil(std::pow(1.1163 * scaled_err, 1.0 / 6.0));
        arm = (4.0 / 3.0) * std::tan(PI / (2.0 * (double)n));
    }
    p->el('M', {cx + r, cy});
    const double dth = 2.0 * PI / (double)n;
    for (long ix = 1; ix <= n; ix++) {
        const double th1 = dth * (double)ix, th0 = th1 - dth;
        const double s0 = std::sin(th0), c0 = std::cos(th0);
        double s1 = 0.0, c1 = 1.0;
        if (ix != n) {
            s1 = std::sin(th1);
            c1 = std::cos(th1);
        }
        const double a = arm * r;
        p->el('C', {cx + r * c0 - a * s0, cy + r * s0 + a * c0, cx + r * c1 + a * s1, cy + r * s1 - a * c1, cx + r * c1, cy + r * s1});
    }
    p->el('Z', {});
    return VB_OK;
}
// kurbo Ellipse::new(center, radii, x_rotation).path_elements(tolerance): the radii and the rotation are recovered from the
// ellipse's affine map (rotate(x_rotation) * scale(rx, ry)) by Affine::svd, then Arc { start 0, sweep 2 pi } + ClosePath.
int vb_pathbuf_ellipse(vb_pathbuf *p, double cx, double cy, double rx, double ry, double x_rotation, double tolerance) {
    if (!p || !(tolerance > 0.0)) return VB_E_INVALID;
    const double a = rx * std::cos(x_rotation), b = rx * std::sin(x_rotation);
    const double c = -ry * std::sin(x_rotation), d = ry * std::cos(x_rotation);
    const double a2 = a * a, b2 = b * b, c2 = c * c, d2 = d * d;
    const double rot = 0.5 * std::atan2(2.0 * (a * b + c * d), a2 - b2 + c2 - d2);
    const double s1 = a2 + b2 + c2 + d2;
    const double s2 = std::sqrt((a2 - b2 + c2 - d2) * (a2 - b2 + c2 - d2) + 4.0 * (a * b + c * d) * (a * b + c * d));
    const double r0 = std::sqrt(0.5 * (s1 + s2)), r1 = std::sqrt(std::fmax(0.5 * (s1 - s2), 0.0));
    p->el('M', {cx + std::cos(rot) * r0, cy + std::sin(rot) * r0});
    arc_elements(*p, cx, cy, r0, r1, 0.0, 2.0 * PI, rot, tolerance);
    p->el('Z', {});
    return VB_OK;
}
// kurbo Arc { center, radii, start_angle, sweep_angle, x_rotation }.path_elements(tolerance): MoveTo(start) + the cubics (open)
int vb_pathbuf_arc(vb_pathbuf *p, double cx, double cy, double rx, double ry, double start_angle, double sweep_angle, double x_rotation,
                   double tolerance) {
    if (!p || !(tolerance > 0.0)) return VB_E_INVALID;
    const double cr = std::cos(x_rotation), sr = std::sin(x_rotation);
    const double x = rx * std::cos(start_angle), y = ry * std::sin(start_angle);
    p->el('M', {cx + cr * x - sr * y, cy + sr * x + cr * y});
    arc_elements(*p, cx, cy, rx, ry, start_angle, sweep_angle, x_rotation, tolerance);
    return VB_OK;
}
int vb_pathbuf_rounded_rect(vb_pathbuf *p, double x0, double y0, double x1, double y1, double radius, double tolerance) {
    if (!p || !(tolerance > 0.0)) return VB_E_INVALID;
    const double rad = std::fmin(std::fabs(radius), std::fmin(0.5 * std::fabs(x1 - x0), 0.5 * std::fabs(y1 - y0)));
    if (rad <= 0.0) return vb_pathbuf_rect(p, x0, y0, x1, y1);
    const double hp = 0.5 * PI;
    p->el('M', {x0 + rad, y0}); // start on the top edge after the top-left corner, clockwise (y down)
    const double corners[4][3] = {{x1 - rad, y0 + rad, -hp}, {x1 - rad, y1 - rad, 0.0}, {x0 + rad, y1 - rad, hp}, {x0 + rad, y0 + rad, 2 * hp}};
    for (const auto &c : corners) {
        p->el('L', {c[0] + rad * std::cos(c[2]), c[1] + rad * std::sin(c[2])});
        arc_elements(*p, c[0], c[1], rad, rad, c[2], hp, 0.0, tolerance);
    }
    p->el('Z', {});
    return VB_OK;
}
// SVG path data, the subset kurbo's BezPath::from_svg accepts (MmLlHhVvCcSsQqTtAaZz; kurbo svg.rs), arcs converted to
// cubics per the SVG implementation notes F.6.5 (endpoint -> centre parametrisation) + Arc::append_iter.
namespace {
struct SvgLexer {
    const char *s;
    size_t i = 0, n;
    explicit SvgLexer(const char *d) : s(d), n(std::strlen(d)) {}
    static bool is_alpha(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
    static bool is_digit(char c) { return c >= '0' && c <= '9'; }
    void skip() {
        while (i < n && (s[i] == ' ' || s[i] == '\t' || s[i] == '\r' || s[i] == '\n' || s[i] == ',')) i++;
    }
    char peek_cmd() {
        skip();
        return (i < n && is_alpha(s[i])) ? s[i] : 0;
    }
    bool more_numbers() {
        skip();
        return i < n && (s[i] == '+' || s[i] == '-' || s[i] == '.' || is_digit(s[i]));
    }
    bool num(double *out) { // [+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?
        skip();
        size_t j = i;
        if (j < n && (s[j] == '+' || s[j] == '-')) j++;
        size_t d0 = j;
        while (j < n && is_digit(s[j])) j++;
        if (j > d0) {
            if (j < n && s[j] == '.') {
                j++;
                while (j < n && is_digit(s[j])) j++;
            }
        } else {
            if (!(j < n && s[j] == '.')) return false;
            j++;
            size_t f0 = j;
            while (j < n && is_digit(s[j])) j++;
            if (j == f0) return false;
        }
        if (j < n && (s[j] == 'e' || s[j] == 'E')) {
            size_t k = j + 1;
            if (k < n && (s[k] == '+' || s[k] == '-')) k++;
            size_t e0 = k;
            while (k < n && is_digit(s[k])) k++;
            if (k > e0) j = k;
        }
        char buf[400];
        const size_t len = j - i;
        if (len == 0 || len >= sizeof buf) return false;
        std::memcpy(buf, s + i, len);
        buf[len] = 0;
        *out = std::strtod(buf, nullptr);
        i = j;
        return true;
    }
    bool flag(bool *out) {
        skip();
        if (i >= n || (s[i] != '0' && s[i] != '1')) return false;
        *out = s[i] == '1';
        i++;
        return true;
    }
};

void svg_arc(vb_pathbuf &pb, double x0, double y0, double rx, double ry, double x_rot_deg, bool large, bool sweep, double x, double y) {
    const double tolerance = 0.1;
    if (rx == 0.0 || ry == 0.0 || (x0 == x && y0 == y)) {
        if (!(x0 == x && y0 == y)) pb.el('L', {x, y});
        return;
    }
    rx = std::fabs(rx);
    ry = std::fabs(ry);
    const double phi = x_rot_deg * (PI / 180.0);
    const double cp = std::cos(phi), sp = std::sin(phi);
    const double dx2 = 0.5 * (x0 - x), dy2 = 0.5 * (y0 - y);
    const double x1p = cp * dx2 + sp * dy2, y1p = -sp * dx2 + cp * dy2;
    const double lam = (x1p * x1p) / (rx * rx) + (y1p * y1p) / (ry * ry);
    if (lam > 1.0) {
        const double sc = std::sqrt(lam);
        rx *= sc;
        ry *= sc;
    }
    const double num = rx * rx * ry * ry - rx * rx * y1p * y1p - ry * ry * x1p * x1p;
    const double den = rx * rx * y1p * y1p + ry * ry * x1p * x1p;
    double coef = den != 0.0 ? std::sqrt(std::fmax(num / den, 0.0)) : 0.0;
    if (large == sweep) coef = -coef;
    const double cxp = coef * rx * y1p / ry, cyp = -coef * ry * x1p / rx;
    const double cx = cp * cxp - sp * cyp + 0.5 * (x0 + x), cy = sp * cxp + cp * cyp + 0.5 * (y0 + y);
    const double a0 = std::atan2((y1p - cyp) / ry, (x1p - cxp) / rx), a1 = std::atan2((-y1p - cyp) / ry, (-x1p - cxp) / rx);
    double d = a1 - a0;
    if (sweep && d < 0) d += 2 * PI;
    else if (!sweep && d > 0) d -= 2 * PI;
    const size_t before = pb.verbs.size();
    arc_elements(pb, cx, cy, rx, ry, a0, d, phi, tolerance);
    if (pb.verbs.size() > before) { // land exactly on the end point
        pb.coords[pb.coords.size() - 2] = x;
        pb.coords[pb.coords.size() - 1] = y;
    }
}
} // namespace

int vb_pathbuf_svg(vb_pathbuf *p, const char *d) {
    if (!p || !d) return VB_E_INVALID;
    SvgLexer lx(d);
    double cx = 0.0, cy = 0.0, sx = 0.0, sy = 0.0, lcx = 0.0, lcy = 0.0;
    bool have_ctrl = false;
    char last_cmd = 0, cmd = 0;
    for (;;) {
        const char c = lx.peek_cmd();
        if (c) {
            cmd = c;
            lx.i++;
        } else if (!lx.more_numbers()) {
            break;
        } else if (!cmd) {
            return VB_E_INVALID; // path data must start with a command
        } else if (cmd == 'M') {
            cmd = 'L'; // implicit line-to after move-to
        } else if (cmd == 'm') {
            cmd = 'l';
        }
        const bool rel = cmd >= 'a' && cmd <= 'z';
        const char u = rel ? (char)(cmd - 32) : cmd;
        double v[7];
        auto nums = [&](int k) {
            for (int q = 0; q < k; q++)
                if (!lx.num(&v[q])) return false;
            return true;
        };
        switch (u) {
        case 'Z':
            p->el('Z', {});
            cx = sx; cy = sy;
            have_ctrl = false;
            last_cmd = u;
            if (lx.more_numbers()) return VB_E_INVALID;
            continue;
        case 'M':
            if (!nums(2)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; }
            p->el('M', {v[0], v[1]});
            cx = sx = v[0]; cy = sy = v[1];
            have_ctrl = false;
            break;
        case 'L':
            if (!nums(2)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; }
            p->el('L', {v[0], v[1]});
            cx = v[0]; cy = v[1];
            have_ctrl = false;
            break;
        case 'H':
            if (!nums(1)) return VB_E_INVALID;
            if (rel) v[0] += cx;
            p->el('L', {v[0], cy});
            cx = v[0];
            have_ctrl = false;
            break;
        case 'V':
            if (!nums(1)) return VB_E_INVALID;
            if (rel) v[0] += cy;
            p->el('L', {cx, v[0]});
            cy = v[0];
            have_ctrl = false;
            break;
        case 'C':
            if (!nums(6)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; v[2] += cx; v[3] += cy; v[4] += cx; v[5] += cy; }
            p->el('C', {v[0], v[1], v[2], v[3], v[4], v[5]});
            lcx = v[2]; lcy = v[3]; have_ctrl = true;
            cx = v[4]; cy = v[5];
            break;
        case 'S': {
            if (!nums(4)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; v[2] += cx; v[3] += cy; }
            double x1 = cx, y1 = cy;
            if ((last_cmd == 'C' || last_cmd == 'S') && have_ctrl) { x1 = 2 * cx - lcx; y1 = 2 * cy - lcy; }
            p->el('C', {x1, y1, v[0], v[1], v[2], v[3]});
            lcx = v[0]; lcy = v[1]; have_ctrl = true;
            cx = v[2]; cy = v[3];
            break;
        }
        case 'Q':
            if (!nums(4)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; v[2] += cx; v[3] += cy; }
            p->el('Q', {v[0], v[1], v[2], v[3]});
            lcx = v[0]; lcy = v[1]; have_ctrl = true;
            cx = v[2]; cy = v[3];
            break;
        case 'T': {
            if (!nums(2)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; }
            double x1 = cx, y1 = cy;
            if ((last_cmd == 'Q' || last_cmd == 'T') && have_ctrl) { x1 = 2 * cx - lcx; y1 = 2 * cy - lcy; }
            p->el('Q', {x1, y1, v[0], v[1]});
            lcx = x1; lcy = y1; have_ctrl = true;
            cx = v[0]; cy = v[1];
            break;
        }
        case 'A': {
            bool large, sweep;
            if (!nums(3) || !lx.flag(&large) || !lx.flag(&sweep)) return VB_E_INVALID;
            const double rx = v[0], ry = v[1], rot = v[2];
            if (!nums(2)) return VB_E_INVALID;
            if (rel) { v[0] += cx; v[1] += cy; }
            svg_arc(*p, cx, cy, rx, ry, rot, large, sweep, v[0], v[1]);
            cx = v[0]; cy = v[1];
            have_ctrl = false;
            break;
        }
        default: return VB_E_INVALID;
        }
        last_cmd = u;
    }
    return VB_OK;
}

vb_path vb_pathbuf_view(const vb_pathbuf *p) {
    vb_path v = {nullptr, 0, nullptr};
    if (p) {
        v.verbs = p->verbs.data();
        v.n_verbs = (uint32_t)p->verbs.size();
        v.coords = p->coords.data();
    }
    return v;
}

vb_scene *vb_scene_new(void) { return new (std::nothrow) vb_scene(); }
void vb_scene_free(vb_scene *s) { delete s; }
void vb_scene_reset(vb_scene *s) {
    if (s) *s = vb_scene();
}

int vb_scene_fill(vb_scene *s, uint32_t fill_rule, const double transform[6], const vb_brush *brush, const double *brush_transform,
                  const vb_path *path) {
    if (!s || !transform || !brush || !path) return VB_E_INVALID;
    Encoding &e = s->e;
    const Affine t = to_affine(transform);
    e.encode_transform(t);
    e.encode_fill_style(fill_rule);
    int rc = VB_OK;
    if (encode_path(e, *path, true, &rc)) {
        if (brush_transform && e.encode_transform(mul(t, to_affine(brush_transform)))) e.swap_last_path_tags();
        const int rb = encode_brush(e, *brush, 1.0f);
        if (rb) return rb;
    }
    return rc;
}

int vb_scene_stroke(vb_scene *s, const vb_stroke *stroke, const double transform[6], const vb_brush *brush, const double *brush_transform,
                    const vb_path *path) {
    if (!s || !stroke || !transform || !brush || !path) return VB_E_INVALID;
    if (stroke->width == 0.0) return VB_OK;
    Encoding &e = s->e;
    const Affine t = to_affine(transform);
    int rc = VB_OK;
    if (stroke_inner(e, *stroke, t, *path, &rc)) {
        if (brush_transform && e.encode_transform(mul(t, to_affine(brush_transform)))) e.swap_last_path_tags();
        const int rb = encode_brush(e, *brush, 1.0f);
        if (rb) return rb;
    }
    return rc;
}

int vb_scene_push_layer(vb_scene *s, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, uint32_t mix, uint32_t compose, float alpha,
                        const double transform[6], const vb_path *clip) {
    return push_layer_inner(s, (mix << 8) | compose, clamp01(alpha), clip_fill_rule, clip_stroke, transform, clip);
}
int vb_scene_push_luminance_mask_layer(vb_scene *s, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, float alpha,
                                       const double transform[6], const vb_path *clip) {
    return push_layer_inner(s, LUMINANCE_MASK_BLEND_MODE, clamp01(alpha), clip_fill_rule, clip_stroke, transform, clip);
}
int vb_scene_push_clip_layer(vb_scene *s, uint32_t clip_fill_rule, const vb_stroke *clip_stroke, const double transform[6],
                             const vb_path *clip) {
    return push_layer_inner(s, CLIP_BLEND_MODE, 1.0f, clip_fill_rule, clip_stroke, transform, clip);
}
int vb_scene_pop_layer(vb_scene *s) {
    if (!s) return VB_E_INVALID;
    s->e.encode_end_clip();
    return VB_OK;
}

int vb_scene_draw_image(vb_scene *s, const vb_image *image, const double transform[6]) {
    if (!s || !image || !transform) return VB_E_INVALID;
    Encoding &e = s->e;
    e.encode_transform(to_affine(transform));
    e.encode_fill_style(VB_FILL_NON_ZERO);
    if (encode_rect(e, 0.0, 0.0, (double)image->width, (double)image->height)) {
        vb_brush b;
        std::memset(&b, 0, sizeof b);
        b.kind = VB_BRUSH_IMAGE;
        b.image = image;
        return encode_brush(e, b, 1.0f);
    }
    return VB_OK;
}

static int blurred_rect_tail(Encoding &e, const Affine &t, const double rect[4], vb_color color, double radius, double std_dev) {
    const double cx = 0.5 * (rect[0] + rect[2]), cy = 0.5 * (rect[1] + rect[3]);
    Affine tr{{1.0, 0.0, 0.0, 1.0, cx, cy}};
    if (e.encode_transform(mul(t, tr))) e.swap_last_path_tags();
    e.draw_tags.push_back(DRAWTAG_BLUR_RECT);
    e.draw_data.push_back(premul_rgba8(to_color(color)));
    e.draw_data.push_back(f32_bits((float)(rect[2] - rect[0])));
    e.draw_data.push_back(f32_bits((float)(rect[3] - rect[1])));
    e.draw_data.push_back(f32_bits((float)radius));
    e.draw_data.push_back(f32_bits((float)std_dev));
    return VB_OK;
}

int vb_scene_draw_blurred_rounded_rect(vb_scene *s, const double transform[6], const double rect[4], vb_color color, double radius,
                                       double std_dev) {
    if (!s || !transform || !rect) return VB_E_INVALID;
    Encoding &e = s->e;
    const Affine t = to_affine(transform);
    const double k = 2.5 * std_dev; // the shape drawn is the rectangle inflated by 2.5 sigma (scene.rs:266-269)
    e.encode_transform(t);
    e.encode_fill_style(VB_FILL_NON_ZERO);
    if (encode_rect(e, rect[0] - k, rect[1] - k, rect[2] + k, rect[3] + k)) return blurred_rect_tail(e, t, rect, color, radius, std_dev);
    return VB_OK;
}

int vb_scene_draw_blurred_rounded_rect_in(vb_scene *s, const vb_path *shape, const double transform[6], const double rect[4],
                                          vb_color color, double radius, double std_dev) {
    if (!s || !shape || !transform || !rect) return VB_E_INVALID;
    Encoding &e = s->e;
    const Affine t = to_affine(transform);
    e.encode_transform(t);
    e.encode_fill_style(VB_FILL_NON_ZERO);
    int rc = VB_OK;
    if (encode_path(e, *shape, true, &rc)) return blurred_rect_tail(e, t, rect, color, radius, std_dev);
    return rc;
}

// Scene::append (scene.rs:464-469) = Encoding::append (encoding.rs:94-174) without glyph runs
int vb_scene_append(vb_scene *dst, const vb_scene *src, const double *transform) {
    if (!dst || !src || dst == src) return VB_E_INVALID;
    Encoding &e = dst->e;
    const Encoding &o = src->e;
    const uint32_t dd = (uint32_t)e.draw_data.size();
    for (RampPatch p : o.ramp_patches) {
        p.draw_data_offset += dd;
        e.ramp_patches.push_back(std::move(p));
    }
    for (ImagePatch p : o.image_patches) {
        p.draw_data_offset += dd;
        e.image_patches.push_back(p);
    }
    e.path_tags.insert(e.path_tags.end(), o.path_tags.begin(), o.path_tags.end());
    e.path_data.insert(e.path_data.end(), o.path_data.begin(), o.path_data.end());
    e.draw_tags.insert(e.draw_tags.end(), o.draw_tags.begin(), o.draw_tags.end());
    e.draw_data.insert(e.draw_data.end(), o.draw_data.begin(), o.draw_data.end());
    e.n_paths += o.n_paths;
    e.n_path_segments += o.n_path_segments;
    e.n_clips += o.n_clips;
    e.n_open_clips += o.n_open_clips;
    if (transform) { // Transform * Transform in f32 (math.rs:51-73)
        float a[6];
        for (int i = 0; i < 6; i++) a[i] = (float)transform[i];
        for (const Xform &x : o.transforms) {
            const float *b = x.c;
            Xform r;
            r.c[0] = a[0] * b[0] + a[2] * b[1];
            r.c[1] = a[1] * b[0] + a[3] * b[1];
            r.c[2] = a[0] * b[2] + a[2] * b[3];
            r.c[3] = a[1] * b[2] + a[3] * b[3];
            r.c[4] = a[0] * b[4] + a[2] * b[5] + a[4];
            r.c[5] = a[1] * b[4] + a[3] * b[5] + a[5];
            e.transforms.push_back(r);
        }
    } else {
        e.transforms.insert(e.transforms.end(), o.transforms.begin(), o.transforms.end());
    }
    e.styles.insert(e.styles.end(), o.styles.begin(), o.styles.end());
    return VB_OK;
}

int vb_scene_batch(vb_scene *dst, const vb_scene *const *scenes, uint32_t n, uint32_t *draw_offsets) {
    if (!dst || (n && (!scenes || !draw_offsets))) return VB_E_INVALID;
    for (uint32_t i = 0; i < n; i++)
        if (!scenes[i] || scenes[i] == dst) return VB_E_INVALID;
    vb_scene_reset(dst);
    Encoding &e = dst->e;
    if (draw_offsets) draw_offsets[0] = 0;
    for (uint32_t i = 0; i < n; i++) {
        vb_scene_append(dst, scenes[i], nullptr);
        while (e.n_open_clips > 0) e.encode_end_clip();
        draw_offsets[i + 1] = e.n_paths; // after resolve every draw object is a path
    }
    return VB_OK;
}

int vb_scene_resolve(vb_scene *s, vb_packed *out) {
    if (!s || !out) return VB_E_INVALID;
    const Encoding &e = s->e;
    std::vector<uint32_t> draw_data = e.draw_data;
    // late-bound gradient ramps, de-duplicated by (stops, interpolation space) -- ramp_cache.rs
    std::vector<const RampPatch *> ramp_of;
    s->ramps.clear();
    for (const RampPatch &p : e.ramp_patches) {
        uint32_t rid = (uint32_t)ramp_of.size();
        for (uint32_t k = 0; k < ramp_of.size(); k++) {
            const RampPatch &q = *ramp_of[k];
            bool same = q.premul == p.premul && q.stops.size() == p.stops.size();
            for (size_t i = 0; same && i < p.stops.size(); i++) same = q.stops[i].offset == p.stops[i].offset && q.stops[i].color == p.stops[i].color;
            if (same) { rid = k; break; }
        }
        if (rid == ramp_of.size()) {
            ramp_of.push_back(&p);
            s->ramps.resize(s->ramps.size() + N_RAMP_SAMPLES);
            make_ramp(p.stops, p.premul, s->ramps.data() + (size_t)rid * N_RAMP_SAMPLES);
        }
        draw_data[p.draw_data_offset] = (rid << 2) | p.extend;
    }
    // late-bound images: shelf-packed atlas (placement is ours; only the (x, y) written into the draw data matters)
    struct Placed { const uint8_t *key; uint32_t w, h, x, y; };
    std::vector<Placed> placed;
    uint32_t atlas_w = 1, x = 0, y = 0, shelf_h = 0;
    const uint32_t MAXW = 2048;
    for (const ImagePatch &p : e.image_patches) {
        const vb_image &im = p.image;
        const Placed *hit = nullptr;
        for (const Placed &q : placed)
            if (q.key == im.pixels && q.w == im.width && q.h == im.height) { hit = &q; break; }
        uint32_t px, py;
        if (!hit) {
            if (x + im.width > MAXW) {
                y += shelf_h;
                x = 0;
                shelf_h = 0;
            }
            placed.push_back(Placed{im.pixels, im.width, im.height, x, y});
            px = x; py = y;
            x += im.width;
            if (im.height > shelf_h) shelf_h = im.height;
            if (x > atlas_w) atlas_w = x;
        } else {
            px = hit->x; py = hit->y;
        }
        draw_data[p.draw_data_offset] = (px << 16) | py;
    }
    const uint32_t atlas_h = (y + shelf_h) > 1u ? (y + shelf_h) : 1u;
    s->atlas.assign((size_t)atlas_w * atlas_h * 4, 0);
    // a registered texture's key points at nothing (its pixels exist only in device memory): its region stays zero, as for NULL
    for (const Placed &q : placed)
        for (uint32_t row = 0; row < q.h && q.key && !vb_texture_key(q.key); row++)
            std::memcpy(&s->atlas[((size_t)(q.y + row) * atlas_w + q.x) * 4], q.key + (size_t)row * q.w * 4, (size_t)q.w * 4);

    // pack the six streams (resolve.rs:107-154); unclosed clips get a trailing PATH tag and END_CLIP draw tag each
    vb_layout L;
    std::memset(&L, 0, sizeof L);
    L.n_paths = e.n_paths;
    L.n_clips = e.n_clips;
    const uint32_t n_tags = (uint32_t)e.path_tags.size() + e.n_open_clips;
    const uint32_t padded = align_up(n_tags, 4 * PATH_REDUCE_WG);
    const size_t total = (size_t)padded / 4 + e.path_data.size() + e.draw_tags.size() + e.n_open_clips + draw_data.size() + e.transforms.size() * 6 +
                         e.styles.size() * 2;
    s->packed.assign(total, 0u);
    uint8_t *tag_bytes = reinterpret_cast<uint8_t *>(s->packed.data());
    if (!e.path_tags.empty()) std::memcpy(tag_bytes, e.path_tags.data(), e.path_tags.size());
    for (uint32_t i = 0; i < e.n_open_clips; i++) tag_bytes[e.path_tags.size() + i] = TAG_PATH;
    uint32_t off = padded / 4;
    L.path_tag_base = 0;
    L.path_data_base = off;
    if (!e.path_data.empty()) std::memcpy(&s->packed[off], e.path_data.data(), e.path_data.size() * 4);
    off += (uint32_t)e.path_data.size();
    L.draw_tag_base = off;
    uint32_t info = 0;
    for (uint32_t t : e.draw_tags) {
        s->packed[off++] = t;
        info += (t >> 6) & 0xFu;
    }
    for (uint32_t i = 0; i < e.n_open_clips; i++) s->packed[off++] = DRAWTAG_END_CLIP;
    L.bin_data_start = info;
    L.draw_data_base = off;
    if (!draw_data.empty()) std::memcpy(&s->packed[off], draw_data.data(), draw_data.size() * 4);
    off += (uint32_t)draw_data.size();
    L.transform_base = off;
    for (const Xform &t : e.transforms)
        for (int i = 0; i < 6; i++) s->packed[off++] = f32_bits(t.c[i]);
    L.style_base = off;
    for (const Style &st : e.styles) {
        s->packed[off++] = st.flags;
        s->packed[off++] = f32_bits(st.width);
    }
    L.n_draw_objects = L.n_paths;
    out->scene = reinterpret_cast<const uint8_t *>(s->packed.data());
    out->scene_len = s->packed.size() * 4;
    out->layout = L;
    out->ramps = s->ramps.empty() ? nullptr : s->ramps.data();
    out->ramp_w = N_RAMP_SAMPLES;
    out->ramp_h = (uint32_t)(s->ramps.size() / N_RAMP_SAMPLES);
    out->atlas = s->atlas.data();
    out->atlas_w = atlas_w;
    out->atlas_h = atlas_h;
    return VB_OK;
}

// Shapes to pixels: the scene's streams are resolved ON THE DEVICE (vb_scene_upload_streams: stream copies to their Layout offsets,
// patch / padding / ramp kernels), then rendered.
int vb_scene_upload_device(vb_renderer *r, vb_scene *s, vb_layout *layout_out) {
    if (!r || !s) return VB_E_INVALID;
    const Encoding &e = s->e;
    static_assert(sizeof(Stop) == sizeof(vb_ramp_stop) && sizeof(Xform) == 24 && sizeof(Style) == 8, "stream record layouts");
    std::vector<vb_ramp_patch> rps;
    for (const RampPatch &p : e.ramp_patches)
        rps.push_back(vb_ramp_patch{p.draw_data_offset, p.extend, p.premul ? 1u : 0u, (uint32_t)p.stops.size(),
                                    reinterpret_cast<const vb_ramp_stop *>(p.stops.data())});
    std::vector<vb_image_patch> ips;
    for (const ImagePatch &p : e.image_patches) ips.push_back(vb_image_patch{p.draw_data_offset, p.image.width, p.image.height, p.image.pixels});
    vb_encoding_streams st;
    std::memset(&st, 0, sizeof st);
    st.path_tags = e.path_tags.data(); st.n_path_tags = (uint32_t)e.path_tags.size();
    st.path_data = reinterpret_cast<const uint32_t *>(e.path_data.data()); st.n_path_data = (uint32_t)e.path_data.size();
    st.draw_tags = e.draw_tags.data(); st.n_draw_tags = (uint32_t)e.draw_tags.size();
    st.draw_data = e.draw_data.data(); st.n_draw_data = (uint32_t)e.draw_data.size();
    st.transforms = reinterpret_cast<const float *>(e.transforms.data()); st.n_transforms = (uint32_t)e.transforms.size();
    st.styles = reinterpret_cast<const uint32_t *>(e.styles.data()); st.n_styles = (uint32_t)e.styles.size();
    st.n_paths = e.n_paths; st.n_clips = e.n_clips; st.n_open_clips = e.n_open_clips;
    st.ramp_patches = rps.data(); st.n_ramp_patches = (uint32_t)rps.size();
    st.image_patches = ips.data(); st.n_image_patches = (uint32_t)ips.size();
    return vb_scene_upload_streams(r, &st, layout_out);
}

int vb_register_texture(vb_renderer *r, const void *device_pixels, uint32_t width, uint32_t height, size_t row_pitch_bytes, vb_image *out) {
    if (!out) return VB_E_INVALID;
    const void *key = nullptr;
    const int rc = vb_texture_register(r, device_pixels, width, height, row_pitch_bytes, &key);
    if (rc) return rc;
    std::memset(out, 0, sizeof *out);
    out->pixels = static_cast<const uint8_t *>(key);
    out->width = width;
    out->height = height;
    out->quality = 1; // peniko's default ImageQuality::Medium; RGBA8, straight alpha, pad: zeros
    out->alpha = 1.0f;
    return VB_OK;
}

int vb_unregister_texture(vb_renderer *r, const vb_image *image) {
    if (!r || !image) return VB_E_INVALID;
    return vb_texture_unregister(r, image->pixels);
}

int vb_render_scene(vb_renderer *r, vb_scene *s, const vb_params *p, void *out, uint32_t out_is_device, vb_frame_stats *stats) {
    const int rc = vb_scene_upload_device(r, s, nullptr);
    if (rc) return rc;
    return vb_render_uploaded(r, p, out, out_is_device, stats);
}

} // extern "C"
