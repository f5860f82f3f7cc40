// vb_resolve.h -- what the library's three Resolver::resolve share, so that their output stays byte-identical. The host resolve
// (vb_scene_resolve, vb_scene.cpp) and the device resolve (vb_scene_upload_streams) apply one plan (vb_resolve_plan). Composition
// (vb_compose.cu) de-duplicates by its fragments' keys, so it shares only the decisions: layout, ramp equality, shelf placement.
// Internal to the library, and plain C++: vb_scene.cpp is built without the CUDA headers.
#ifndef VB_RESOLVE_H
#define VB_RESOLVE_H
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <unordered_map>
#include <vector>

#include "../../include/vello_b200.h"

// The info words of a scene's draw tags (layout.bin_data_start).
static inline uint64_t vb_draw_info_sum(const uint32_t *draw_tags, size_t n) {
    uint64_t info = 0;
    for (size_t i = 0; i < n; i++) info += (draw_tags[i] >> 6) & 0xFu;
    return info;
}

// f32 -> f16 (math.rs:93-127, float_to_half_fast3): the miter limit in a stroke's style word. The native scene front end
// (vb_scene.cpp) and fragments from device arrays (vb_compose.cu) encode it.
static inline uint32_t vb_f32_to_f16(float val) {
    const uint32_t INF_32 = 255u << 23, INF_16 = 31u << 23, MAGIC = 15u << 23, ROUND_MASK = ~0xFFFu;
    uint32_t u;
    memcpy(&u, &val, 4);
    const uint32_t sign = u & 0x80000000u;
    u ^= sign;
    uint32_t out;
    if (u >= INF_32) {
        out = u > INF_32 ? 0x7E00u : 0x7C00u;
    } else {
        u &= ROUND_MASK;
        float f, magic;
        memcpy(&f, &u, 4);
        memcpy(&magic, &MAGIC, 4);
        f = f * magic;
        memcpy(&u, &f, 4);
        u -= ROUND_MASK;
        if (u > INF_16) u = INF_16;
        out = (u >> 13) & 0xFFFFu;
    }
    return out | (sign >> 16);
}

// The packed scene's layout from the sizes of its streams (resolve.rs:107-154): the tag bytes and one PATH tag per open clip,
// padded to 4 * PATH_REDUCE_WG bytes (resolve.rs:625, config.rs:237); path data; draw tags and one END_CLIP per open clip; draw
// data; 6 words per transform; 2 per style. Sets *padded_tags (bytes) and *words (the whole scene). False when the scene, with
// room behind it for a view's transforms, passes 32-bit word offsets. Layout: vb_layout, or the host files' VbLayout (the same record).
template <class Layout>
static inline bool vb_resolve_layout(uint64_t path_tags, uint64_t path_data, uint64_t draw_tags, uint64_t draw_data, uint64_t transforms,
                                     uint64_t styles, uint64_t open_clips, uint64_t paths, uint64_t clips, uint64_t info, Layout *L,
                                     uint32_t *padded_tags, size_t *words) {
    const uint64_t padded = (path_tags + open_clips + 1023u) & ~1023ull;
    const uint64_t total = padded / 4u + path_data + draw_tags + open_clips + draw_data + 6u * transforms + 2u * styles;
    if (padded > 0xffffffffull || total + 6u * transforms > 0xfffffff0ull || paths > 0xffffffffull || info > 0xffffffffull) return false;
    memset(L, 0, sizeof *L);
    L->n_paths = L->n_draw_objects = (uint32_t)paths;
    L->n_clips = (uint32_t)clips;
    L->bin_data_start = (uint32_t)info;
    L->path_tag_base = 0;
    L->path_data_base = (uint32_t)(padded / 4u);
    L->draw_tag_base = L->path_data_base + (uint32_t)path_data;
    L->draw_data_base = L->draw_tag_base + (uint32_t)(draw_tags + open_clips);
    L->transform_base = L->draw_data_base + (uint32_t)draw_data;
    L->style_base = L->transform_base + 6u * (uint32_t)transforms;
    *padded_tags = (uint32_t)padded;
    *words = (size_t)total;
    return true;
}

// Two gradient ramps are one when their interpolation spaces match and their stops compare float by float with ==: -0 equals 0,
// and a stop holding a NaN equals nothing, itself included. vb_ramp_hash agrees (equal ramps hash alike).
static inline bool vb_same_ramp(const vb_ramp_stop *a, uint32_t na, bool premul_a, const vb_ramp_stop *b, uint32_t nb, bool premul_b) {
    if (premul_a != premul_b || na != nb) return false;
    for (uint32_t i = 0; i < na; i++)
        if (!(a[i].offset == b[i].offset && a[i].r == b[i].r && a[i].g == b[i].g && a[i].b == b[i].b && a[i].a == b[i].a)) return false;
    return true;
}
static inline uint64_t vb_ramp_hash(const vb_ramp_stop *s, uint32_t n, bool premul) {
    uint64_t h = 1469598103934665603ull;
    auto mix = [&](uint32_t v) { h = (h ^ v) * 1099511628211ull; };
    mix(premul ? 1u : 0u);
    mix(n);
    for (uint32_t i = 0; i < n; i++) {
        const float v[5] = {s[i].offset, s[i].r, s[i].g, s[i].b, s[i].a};
        for (float x : v) {
            uint32_t bits = 0u; // -0 and 0 alike
            if (x != 0.0f) memcpy(&bits, &x, 4);
            mix(bits);
        }
    }
    return h;
}

// The draw data holds an image's atlas place as (x << 16) | y and its size as (w << 16) | h: each is a 16-bit field, so no
// side may pass VB_ATLAS_MAX_COORD and no place may start below row VB_ATLAS_MAX_COORD. The atlas itself may reach past that
// row (an image placed at y = 65535 extends below it).
#define VB_ATLAS_MAX_COORD 65535u
static inline bool vb_atlas_side_fits(uint32_t w, uint32_t h) { return w <= VB_ATLAS_MAX_COORD && h <= VB_ATLAS_MAX_COORD; }

// Shelf placement in the atlas (ours: only the (x, y) written into the draw data matters to the pipeline). Images go left to
// right in rows up to 2048 wide; one that does not fit starts a new row below the tallest image of the last. The caller places
// each distinct image once, in first-seen order. place() is false, and the packer unchanged, for an image with a side over
// VB_ATLAS_MAX_COORD or one whose place would start below row VB_ATLAS_MAX_COORD; the caller refuses the scene.
struct VbShelfPacker {
    uint32_t width = 1, x = 0, y = 0, shelf_h = 0;
    bool place(uint32_t w, uint32_t h, uint32_t *px, uint32_t *py) {
        if (!vb_atlas_side_fits(w, h)) return false;
        const bool new_shelf = x + w > 2048u;
        if (new_shelf && y + shelf_h > VB_ATLAS_MAX_COORD) return false;
        if (new_shelf) {
            y += shelf_h;
            x = 0;
            shelf_h = 0;
        }
        *px = x;
        *py = y;
        x += w;
        if (h > shelf_h) shelf_h = h;
        if (x > width) width = x;
        return true;
    }
    uint32_t height() const { return y + shelf_h > 1u ? y + shelf_h : 1u; }
};

struct RsPatch { uint32_t word, value; }; // one late-bound word of the packed scene, scene[word] = value (k_resolve_finish's input)

// How a scene's streams resolve (resolve.rs:183-399). Two ramp patches share a ramp when vb_same_ramp holds (ramp_cache.rs), two
// image patches an atlas place when their pixels pointer, width and height match.
struct VbResolvePlan {
    struct Image { const uint8_t *pixels; uint32_t w, h, x, y; }; // a distinct image and its atlas place
    vb_layout layout;
    uint32_t padded_tags = 0; // bytes
    size_t words = 0;         // the whole scene
    std::vector<RsPatch> patches; // every ramp patch's (ramp id << 2) | extend, then every image patch's (x << 16) | y, in stream order
    std::vector<const vb_ramp_patch *> ramps; // the distinct ramps in ramp-id order, each as its first patch
    std::vector<Image> images;                // the distinct images in placement order
    uint32_t atlas_w = 0, atlas_h = 0;
};

// VB_PLAN_LAYOUT: the scene passes 32-bit word offsets (vb_resolve_layout); nothing else is planned. VB_PLAN_ATLAS: the shelf
// packer refused an image; the images placed before it stay in the plan, the rest of it is incomplete.
enum { VB_PLAN_OK, VB_PLAN_LAYOUT, VB_PLAN_ATLAS };
static inline int vb_resolve_plan(const vb_encoding_streams &e, VbResolvePlan *p) {
    if (!vb_resolve_layout(e.n_path_tags, e.n_path_data, e.n_draw_tags, e.n_draw_data, e.n_transforms, e.n_styles, e.n_open_clips, e.n_paths,
                           e.n_clips, vb_draw_info_sum(e.draw_tags, e.n_draw_tags), &p->layout, &p->padded_tags, &p->words))
        return VB_PLAN_LAYOUT;
    const uint32_t dd = p->layout.draw_data_base;
    std::unordered_map<uint64_t, std::vector<uint32_t>> ramp_ids; // by vb_ramp_hash
    for (uint32_t i = 0; i < e.n_ramp_patches; i++) {
        const vb_ramp_patch &rp = e.ramp_patches[i];
        std::vector<uint32_t> &same_hash = ramp_ids[vb_ramp_hash(rp.stops, rp.n_stops, rp.premul_interp != 0u)];
        uint32_t rid = (uint32_t)p->ramps.size();
        for (uint32_t k : same_hash) {
            const vb_ramp_patch &q = *p->ramps[k];
            if (vb_same_ramp(q.stops, q.n_stops, q.premul_interp != 0u, rp.stops, rp.n_stops, rp.premul_interp != 0u)) { rid = k; break; }
        }
        if (rid == p->ramps.size()) {
            same_hash.push_back(rid);
            p->ramps.push_back(&rp);
        }
        p->patches.push_back(RsPatch{dd + rp.draw_data_offset, (rid << 2) | rp.extend});
    }
    VbShelfPacker shelf;
    for (uint32_t i = 0; i < e.n_image_patches; i++) {
        const vb_image_patch &im = e.image_patches[i];
        size_t k = 0;
        while (k < p->images.size() && !(p->images[k].pixels == im.pixels && p->images[k].w == im.width && p->images[k].h == im.height)) k++;
        if (k == p->images.size()) {
            VbResolvePlan::Image q{im.pixels, im.width, im.height, 0, 0};
            if (!shelf.place(q.w, q.h, &q.x, &q.y)) return VB_PLAN_ATLAS;
            p->images.push_back(q);
        }
        p->patches.push_back(RsPatch{dd + im.draw_data_offset, (p->images[k].x << 16) | p->images[k].y});
    }
    p->atlas_w = shelf.width, p->atlas_h = shelf.height();
    return VB_PLAN_OK;
}

#endif
