// vb_upload.cu -- scenes into a renderer: uploads of packed scenes, the device resolve (vb_scene_upload_streams), images from
// device memory (overrides and registered textures, copied into the atlas by k_atlas_blit) and batches of cells.
#include <cuda_runtime.h>
#include <string.h>
#include <sys/mman.h>

#include <algorithm>
#include <mutex>

#include "vb_renderer.h"
#include "vb_resolve.h"
#include "vb_textures.h"

// Keys of registered textures (vb_register_texture) and destinations (vb_register_destination). Each is a fresh address inside
// one reserved, inaccessible (PROT_NONE) range of the process's address space, so no host or device buffer can have it, even
// after it is unregistered: the host resolve recognises such a key by its address alone and never reads through it
// (vb_texture_key), and the entry points that take a plain host or device pointer refuse it. The range is never unmapped and a
// key is never handed out twice. `g_key_owner` holds the renderer that registered each key and what kind of key it is.
enum { KEY_TEXTURE, KEY_DESTINATION };
struct KeyOwner {
    vb_renderer *r;
    int kind;
};
static std::mutex g_tex_mutex;
static std::unordered_map<const void *, KeyOwner> g_key_owner;
static uint8_t *g_tex_base = nullptr;
static size_t g_tex_next = 0;
static const size_t TEX_KEY_STRIDE = 16, TEX_RANGE_BYTES = (size_t)1 << 30;

extern "C" int vb_texture_key(const void *key) { // for vb_scene.cpp's host resolve
    const uint8_t *p = (const uint8_t *)key, *base = __atomic_load_n(&g_tex_base, __ATOMIC_ACQUIRE);
    return base != nullptr && p >= base && p < base + TEX_RANGE_BYTES;
}
static const void *new_key(vb_renderer *owner, int kind) {
    std::lock_guard<std::mutex> lock(g_tex_mutex);
    if (!g_tex_base) {
        void *m = mmap(nullptr, TEX_RANGE_BYTES, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (m == MAP_FAILED) return nullptr;
        __atomic_store_n(&g_tex_base, (uint8_t *)m, __ATOMIC_RELEASE);
    }
    if (g_tex_next + TEX_KEY_STRIDE > TEX_RANGE_BYTES) return nullptr;
    const void *key = g_tex_base + g_tex_next;
    g_tex_next += TEX_KEY_STRIDE;
    g_key_owner[key] = KeyOwner{owner, kind};
    return key;
}
// Forget `key` if it is a key of `kind` that r registered.
static bool drop_key(vb_renderer *r, const void *key, int kind) {
    std::lock_guard<std::mutex> lock(g_tex_mutex);
    auto it = vb_texture_key(key) ? g_key_owner.find(key) : g_key_owner.end();
    if (it == g_key_owner.end() || it->second.r != r || it->second.kind != kind) return false;
    g_key_owner.erase(it);
    return true;
}
void vb_host::drop_registrations(vb_renderer *r) {
    for (auto &d : r->dests)
        if (d.second.surf) cudaDestroySurfaceObject(d.second.surf);
    r->dests.clear();
    std::lock_guard<std::mutex> lock(g_tex_mutex);
    for (auto it = g_key_owner.begin(); it != g_key_owner.end();) it = it->second.r == r ? g_key_owner.erase(it) : std::next(it);
}

// Install the scene the current slot's buffers now hold, and drop what depended on the one before: a new scene is one cell
// until vb_set_cells says otherwise, hit testing has no frame of it yet, and nothing is bound to it (VbBound). Its stops are
// unknown until the installer that has them keeps them (keep_stops).
void vb_host::set_scene(vb_renderer *r, const VbLayout &L, size_t scene_words, uint32_t n_ramps, uint32_t atlas_w, uint32_t atlas_h,
                      std::vector<vb_renderer::SceneSlot::OverridePlace> overridden, bool composed) {
    vb_renderer::SceneSlot &s = *r->cur;
    s.layout = L;
    s.scene_words = scene_words;
    s.n_ramps = n_ramps;
    s.atlas_w = atlas_w;
    s.atlas_h = atlas_h;
    s.overridden = std::move(overridden);
    s.composed = composed;
    s.inst_frag.clear(); // vb_compose fills them afterwards
    s.inst_xf.clear();
    s.inst_draw.clear();
    s.inst_img.clear();
    s.img_place.clear();
    s.have_stops = false;
    s.stop_patches.clear();
    s.stops.clear();
    s.have_scene = true;
    r->cells.clear();
    r->bound = VbBound{};
    r->dmg.epoch++;
    // a diff begun for this installation (diff_begin) makes the next frame of this epoch incremental; any other ends it
    vb_renderer::Damage::Diff &X = r->dmg.diff;
    X.armed = X.pending;
    X.pending = false;
    X.epoch = r->dmg.epoch;
    hit_forget(r);
}

// ---- upload diff: vb_set_upload_diff (k_upload_diff.cu) ----------------------------------------------------------------------
static void swap_spare(vb_renderer *r) {
    std::swap(r->cur->scene, r->spare_scene);
    std::swap(r->cur->ramps, r->spare_ramps);
    std::swap(r->cur->atlas, r->spare_atlas);
}

// An upload that tracking follows swaps the spare set in; if it fails before it installs its scene, this swaps the base's back,
// so the renderer keeps the scene it had.
struct DiffedUpload {
    vb_renderer *r = nullptr;
    ~DiffedUpload() {
        if (r && r->dmg.diff.pending) {
            swap_spare(r);
            r->dmg.diff.pending = false;
        }
    }
};

// Before an upload of layout L writes the current slot: when the next frame can diff it against the scene the base frame
// rendered (the switch is on, base_diffable, and the base read this slot's scene buffer), begin the diff (diff_begin) and keep
// that scene. The slot's scene, ramps and atlas are swapped with the spare set, sized here for the upload, which the upload then
// writes; the base's buffers become the spare set, without a copy. On the upload's stream, before anything overwrites the base
// frame's intermediates, its records (from its tag and draw monoids and its scene, read through the uploaded layout, not the
// view's); and the diff's head, which names both sides.
static int upload_diff_begin(vb_renderer *r, cudaStream_t st, const VbLayout &L, size_t scene_words, uint32_t n_ramps, uint32_t atlas_w,
                             uint32_t atlas_h, DiffedUpload &guard) {
    vb_renderer::SceneSlot &s = *r->cur;
    if (!r->upload_diff || r->hit.bufs.scene != (const uint32_t *)s.scene.p || !base_diffable(r)) return VB_OK;
    const uint32_t n_old = s.layout.n_draw_objects, n_new = L.n_draw_objects;
    int rc;
    if ((rc = ensure(r, r->spare_scene, regions_of(L, scene_words, false, r->view.on, false, false).bytes))) return rc;
    if ((rc = ensure(r, r->spare_ramps, (size_t)n_ramps * 512 * 4))) return rc;
    if ((rc = ensure(r, r->spare_atlas, (size_t)atlas_w * atlas_h * 4))) return rc;
    if ((rc = diff_begin(r, st, true, n_old, n_new, n_new))) return rc;
    swap_spare(r); // s keeps the base's layout and sizes until set_scene
    guard.r = r;
    VbUdiff &h = r->ud_head;
    memset(&h, 0, sizeof h);
    h.old_side = VbUdSide{(const uint32_t *)r->spare_scene.p, (const uint32_t *)r->spare_ramps.p, (const uint8_t *)r->spare_atlas.p, s.layout,
                          s.n_ramps, s.atlas_w, s.atlas_h, 0u};
    h.new_side = VbUdSide{(const uint32_t *)s.scene.p, (const uint32_t *)s.ramps.p, (const uint8_t *)s.atlas.p, L, n_ramps, atlas_w, atlas_h, 0u};
    char *ud = (char *)r->dmg_diff.p;
    vb_launch_upload_records(h.old_side.scene, s.layout.path_tag_base, s.layout.draw_tag_base, r->hit.cfg.n_tag_words, n_old,
                             r->hit.bufs.tag_monoids, r->hit.bufs.draw_monoids, (VbUdRec *)(ud + vb_udiff_layout(n_old, n_new).old_rec), nullptr,
                             0u, st);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ud, &h, sizeof h, cudaMemcpyHostToDevice, st));
    return VB_OK;
}

extern "C" int vb_set_upload_diff(vb_renderer *r, int on) {
    if (!r) return VB_E_INVALID;
    if (on && (r->grouped || r->xc.configured)) {
        r->err = "vb_set_upload_diff: not available for a renderer of a vb_group or with the exchange configured";
        return VB_E_INVALID;
    }
    r->upload_diff = on != 0;
    if (on) return VB_OK;
    // off: the spare set goes, and with it the old side of an upload's diff, whose frame is then full
    if (r->dmg.diff.upload) r->dmg.diff.armed = false;
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream)); // an enqueued frame may still read them
    for (DevBuf *b : {&r->spare_scene, &r->spare_ramps, &r->spare_atlas}) {
        if (b->p) CK(cudaFree(b->p));
        *b = DevBuf{};
    }
    return VB_OK;
}

int vb_host::upload_on(vb_renderer *r, cudaStream_t st, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                     uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h, bool diff) {
    if (!r || !layout || (scene_len && !scene) || (scene_len & 3)) return VB_E_INVALID;
    if (ramp_h && ramp_w != 512) return VB_E_INVALID;
    CK(cudaSetDevice(r->device));
    VbLayout L;
    memcpy(&L, layout, sizeof L);
    if (!atlas) atlas_w = atlas_h = 0;
    int rc;
    DiffedUpload guard;
    if (diff && (rc = upload_diff_begin(r, st, L, scene_len / 4, ramp_h, atlas_w, atlas_h, guard))) return rc;
    if ((rc = ensure(r, r->cur->scene, regions_of(L, scene_len / 4, false, r->view.on, false, false).bytes))) return rc;
    if (scene_len) CK(cudaMemcpyAsync(r->cur->scene.p, scene, scene_len, cudaMemcpyHostToDevice, st));
    if ((rc = ensure(r, r->cur->ramps, (size_t)ramp_h * 512 * 4))) return rc;
    if (ramp_h) CK(cudaMemcpyAsync(r->cur->ramps.p, ramps, (size_t)ramp_h * 512 * 4, cudaMemcpyHostToDevice, st));
    if ((rc = ensure(r, r->cur->atlas, (size_t)atlas_w * atlas_h * 4))) return rc;
    if (atlas_w && atlas_h) CK(cudaMemcpyAsync(r->cur->atlas.p, atlas, (size_t)atlas_w * atlas_h * 4, cudaMemcpyHostToDevice, st));
    set_scene(r, L, scene_len / 4, ramp_h, atlas_w, atlas_h, {}, false); // a caller-packed atlas: overrides do not apply
    return VB_OK;
}

extern "C" int vb_scene_upload(vb_renderer *r, const uint8_t *scene, size_t scene_len, const vb_layout *layout, const uint32_t *ramps,
                               uint32_t ramp_w, uint32_t ramp_h, const uint8_t *atlas, uint32_t atlas_w, uint32_t atlas_h) {
    if (!r) return VB_E_INVALID;
    int rc = drain_stream(r);
    if (rc) return rc;
    return upload_on(r, r->stream, scene, scene_len, layout, ramps, ramp_w, ramp_h, atlas, atlas_w, atlas_h, true);
}

// ---- images from device memory: Renderer::override_image / register_texture (vello/src/lib.rs:536-603) ----------------------
// An override names an image by its key (the `pixels` pointer of its vb_image / vb_image_patch). The device resolve
// (vb_scene_upload_streams) copies such an image into its atlas slot from the override's device memory with k_atlas_blit and
// records the slot; marking the image dirty later queues the same copy in front of the next frame (refresh_overrides).

// A device image must be memory of this renderer's device (or managed memory), with 4-byte aligned rows of at least 4 * w bytes.
static int check_device_pixels(vb_renderer *r, const void *px, uint32_t w, uint32_t h, size_t pitch) {
    auto bad = [&](const char *why) {
        r->err = std::string("device image: ") + why;
        return VB_E_INVALID;
    };
    if (!w || !h) return bad("a dimension is 0");
    if (vb_texture_key(px)) return bad("a texture or destination key is not device memory");
    if (((uintptr_t)px & 3u) || (pitch & 3u)) return bad("the pointer and the row pitch must be multiples of 4 bytes");
    if (pitch < (size_t)w * 4u) return bad("the row pitch is less than 4 * width");
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, px) != cudaSuccess) {
        cudaGetLastError();
        return bad("not a CUDA pointer");
    }
    if (a.type == cudaMemoryTypeManaged) return VB_OK;
    if (a.type != cudaMemoryTypeDevice || a.device != r->device) return bad("not device memory of the renderer's device");
    return VB_OK;
}

// Copy `rects` into an atlas of atlas_w texels per row with one k_atlas_blit on the renderer's stream. The rectangles reach
// the device through a pinned staging buffer, which is rewritten only once the previous copy out of it has run.
int vb_host::enqueue_blits(vb_renderer *r, std::vector<VbBlitRect> &rects, void *atlas, uint32_t atlas_w) {
    if (rects.empty()) return VB_OK;
    uint64_t units = 0;
    for (VbBlitRect &b : rects) {
        b.spr = vb_atlas_blit_units_per_row(b.w);
        b.unit0 = units;
        units += (uint64_t)b.h * b.spr;
    }
    const size_t bytes = rects.size() * sizeof(VbBlitRect);
    PinnedStage &s = r->pinned[PIN_BLITS];
    uint8_t *h;
    int rc = stage_host(r, s, bytes, &h);
    if (rc) return rc;
    memcpy(h, rects.data(), bytes);
    if ((rc = ensure(r, r->blit_rects, bytes))) return rc;
    CK(cudaMemcpyAsync(r->blit_rects.p, h, bytes, cudaMemcpyHostToDevice, r->stream));
    if ((rc = stage_copied(r, s))) return rc;
    vb_launch_atlas_blit((const VbBlitRect *)r->blit_rects.p, (uint32_t)rects.size(), units, (uint8_t *)atlas, atlas_w, r->stream);
    CK(cudaGetLastError());
    return VB_OK;
}

// Before a frame: copy the dirty overridden images of the current scene slot into their atlas places. The copy runs ahead of
// every kernel of the frame (and outside any captured graph), so a frame that draws its own destination reads the old pixels.
// The atlas does not move, so a captured frame stays valid. Nothing dirty: nothing is enqueued.
int vb_host::refresh_overrides(vb_renderer *r) {
    std::vector<VbBlitRect> rects;
    for (const auto &o : r->cur->overridden)
        if (o.dirty) rects.push_back(VbBlitRect{o.src, o.pitch, 0, o.w, o.h, o.x, o.y, 0, 0});
    if (rects.empty()) return VB_OK;
    const int rc = enqueue_blits(r, rects, r->cur->atlas.p, r->cur->atlas_w);
    if (rc) return rc;
    for (auto &o : r->cur->overridden) o.dirty = false;
    return VB_OK;
}

extern "C" int vb_override_image(vb_renderer *r, const void *key, uint32_t width, uint32_t height, const void *device_pixels,
                                 size_t row_pitch_bytes) {
    if (!r) return VB_E_INVALID;
    if (!key) {
        r->err = "vb_override_image: NULL key";
        return VB_E_INVALID;
    }
    if (device_pixels) {
        CK(cudaSetDevice(r->device));
        const int rc = check_device_pixels(r, device_pixels, width, height, row_pitch_bytes);
        if (rc) return rc;
        r->overrides[key] = vb_renderer::Override{(const uint8_t *)device_pixels, row_pitch_bytes, width, height};
    } else {
        r->overrides.erase(key);
    }
    // recorded atlas places: a new source of the same size is copied before the next frame; a removed override (or one of
    // another size) keeps the pixels copied last and takes effect at the next device resolve
    for (auto &s : r->slot) {
        auto &v = s.overridden;
        v.erase(std::remove_if(v.begin(), v.end(),
                               [&](const auto &o) { return o.key == key && (!device_pixels || o.w != width || o.h != height); }),
                v.end());
        for (auto &o : v)
            if (o.key == key) {
                o.src = (const uint8_t *)device_pixels;
                o.pitch = row_pitch_bytes;
                o.dirty = true;
            }
    }
    return VB_OK;
}

extern "C" int vb_mark_override_image_dirty(vb_renderer *r, const void *key) {
    if (!r) return VB_E_INVALID;
    if (!r->overrides.count(key)) {
        r->err = "vb_mark_override_image_dirty: no override for this key";
        return VB_E_INVALID;
    }
    for (auto &s : r->slot)
        for (auto &o : s.overridden)
            if (o.key == key) o.dirty = true;
    return VB_OK;
}

// Renderer::register_texture / unregister_texture; vb_register_texture / vb_unregister_texture (vb_scene.cpp, which owns vb_image)
// wrap these two.
extern "C" int vb_texture_register(vb_renderer *r, const void *device_pixels, uint32_t width, uint32_t height, size_t row_pitch_bytes,
                                   const void **key_out) {
    if (!r || !key_out) return VB_E_INVALID;
    if (!device_pixels) {
        r->err = "vb_register_texture: NULL pixels";
        return VB_E_INVALID;
    }
    if (!vb_atlas_side_fits(width, height)) {
        r->err = "vb_register_texture: a side over 65535 texels (an image's size is two 16-bit fields)";
        return VB_E_INVALID;
    }
    CK(cudaSetDevice(r->device));
    int rc = check_device_pixels(r, device_pixels, width, height, row_pitch_bytes);
    if (rc) return rc;
    const void *key = new_key(r, KEY_TEXTURE);
    if (!key) {
        r->err = "vb_register_texture: no texture key left";
        return VB_E_INVALID;
    }
    if ((rc = vb_override_image(r, key, width, height, device_pixels, row_pitch_bytes))) return rc;
    *key_out = key;
    return VB_OK;
}

extern "C" int vb_texture_unregister(vb_renderer *r, const void *key) {
    if (!r) return VB_E_INVALID;
    if (!drop_key(r, key, KEY_TEXTURE)) {
        r->err = "vb_unregister_texture: not a texture registered on this renderer";
        return VB_E_INVALID;
    }
    return vb_override_image(r, key, 0, 0, nullptr, 0);
}

// ---- registered destinations: vb_register_destination / vb_unregister_destination ------------------------------------------
// Frames into a destination's key store through k_fine's FI_DST instantiations, except linear RGBA8 with straight alpha, which
// is the default store at another pitch and origin. Every check is made here or in resolve_destination, on the host, before a
// frame is enqueued. The texel size (Destination::texel) sets the alignment, pitch and channel checks and fine's store.
int vb_host::destination_of(vb_renderer *r, const vb_destination *d, const char *who, Destination *out) {
    auto bad = [&](const std::string &why) {
        r->err = std::string(who) + ": " + why;
        return VB_E_INVALID;
    };
    if (d->kind != VB_DEST_LINEAR && d->kind != VB_DEST_ARRAY) return bad("unknown kind");
    const uint32_t fmt = d->format & ~(uint32_t)VB_DEST_PREMULTIPLIED;
    if (fmt > VB_DEST_RGBA32F) return bad("unknown format or flag");
    if (r->grouped || r->xc.configured) return bad("not available for a renderer of a vb_group or with the exchange configured");
    CK(cudaSetDevice(r->device));
    Destination D;
    D.kind = d->kind;
    D.format = fmt;
    D.premul = (d->format & VB_DEST_PREMULTIPLIED) != 0u;
    const uint32_t T = D.texel();
    if (d->kind == VB_DEST_LINEAR) {
        if (!d->ptr) return bad("NULL ptr");
        if ((uintptr_t)d->ptr % T) return bad("ptr is not " + std::to_string(T) + "-byte aligned");
        if (vb_texture_key(d->ptr) || !device_memory_of(r, d->ptr)) return bad("ptr is not device or managed memory of the renderer's device");
        if (d->row_pitch_bytes % T) return bad("row_pitch_bytes is not a multiple of " + std::to_string(T));
        if (d->row_pitch_bytes >= ((size_t)1 << 34)) return bad("row_pitch_bytes is 2^34 or more");
        D.ptr = (uint8_t *)d->ptr;
        D.pitch = d->row_pitch_bytes;
    } else {
        if (!d->array) return bad("NULL array");
        cudaChannelFormatDesc fd;
        cudaExtent ext;
        unsigned int flags = 0;
        if (cudaArrayGetInfo(&fd, &ext, &flags, (cudaArray_t)d->array) != cudaSuccess) {
            cudaGetLastError();
            return bad("not a CUDA array");
        }
        if (ext.depth != 0 || ext.height == 0 || (flags & (cudaArrayLayered | cudaArrayCubemap)))
            return bad("a 1-D, layered, cubemap or 3-D array (a 2-D array is needed)");
        // four channels of T / 4 bytes each: unsigned for the 8-bit formats, float for the others
        const int bits = (int)(2u * T);
        if (fd.f != (T == 4u ? cudaChannelFormatKindUnsigned : cudaChannelFormatKindFloat) || fd.x != bits || fd.y != bits ||
            fd.z != bits || fd.w != bits)
            return bad("the array's channels are not four " + std::to_string(bits) + (T == 4u ? "-bit unsigned ones" : "-bit float ones"));
        if (!(flags & cudaArraySurfaceLoadStore)) return bad("the array was not created with cudaArraySurfaceLoadStore");
        cudaResourceDesc rd;
        memset(&rd, 0, sizeof rd);
        rd.resType = cudaResourceTypeArray;
        rd.res.array.array = (cudaArray_t)d->array;
        CK(cudaCreateSurfaceObject(&D.surf, &rd));
        D.x0 = d->x;
        D.y0 = d->y;
        D.w = ext.width;
        D.h = ext.height;
    }
    *out = D;
    return VB_OK;
}

extern "C" int vb_register_destination(vb_renderer *r, const vb_destination *d, void **key_out) {
    if (!r) return VB_E_INVALID;
    if (!d || !key_out) {
        r->err = "vb_register_destination: NULL destination or key_out";
        return VB_E_INVALID;
    }
    Destination D;
    if (int rc = destination_of(r, d, "vb_register_destination", &D)) return rc;
    const void *key = new_key(r, KEY_DESTINATION);
    if (!key) {
        if (D.surf) cudaDestroySurfaceObject(D.surf);
        r->err = "vb_register_destination: no key left";
        return VB_E_INVALID;
    }
    r->dests[key] = D;
    *key_out = (void *)key;
    return VB_OK;
}

extern "C" int vb_unregister_destination(vb_renderer *r, void *key) {
    if (!r) return VB_E_INVALID;
    auto it = r->dests.find(key);
    if (it == r->dests.end()) {
        r->err = "vb_unregister_destination: not a destination registered on this renderer";
        return VB_E_INVALID;
    }
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream)); // the frames enqueued into it
    if (it->second.surf) CK(cudaDestroySurfaceObject(it->second.surf));
    r->dests.erase(it);
    drop_key(r, key, KEY_DESTINATION);
    return VB_OK;
}

// The frame r prepared goes to d->dev, a key: check that the frame fits the destination, and say where fine stores (d->out).
// A linear destination holds the whole frame, so a window's rows land at their own rows: out[0] is the window's first row.
int vb_host::resolve_destination(vb_renderer *r, Dest *d) {
    auto bad = [&](const std::string &why) {
        r->err = std::string("registered destination: ") + why;
        return VB_E_INVALID;
    };
    const auto it = r->dests.find(d->dev);
    if (it == r->dests.end()) return bad("the key is not a destination registered on this renderer");
    if (d->host) return bad("a key is not host memory");
    if (r->grouped || r->xc.enabled) return bad("not available for a renderer of a vb_group or with the exchange enabled");
    VbConfig &c = r->cfg;
    if (c.n_cells > 1u) return bad("a batch (vb_set_cells with more than one cell) cannot render into a registered destination");
    const Destination &D = it->second;
    VbFineOut o{};
    o.swz = D.format == VB_DEST_BGRA8 ? 0x3012u : 0x3210u;
    o.texel = D.texel();
    o.premul = D.premul;
    o.dst = D.format != VB_DEST_RGBA8 || D.premul || D.kind == VB_DEST_ARRAY;
    if (D.kind == VB_DEST_LINEAR) {
        if (D.pitch < (size_t)c.target_width * o.texel) return bad("the row pitch is below " + std::to_string(o.texel) + " * width");
        c.out_pitch_px = (uint32_t)(D.pitch / o.texel);
        o.out = (uint32_t *)(D.ptr + (size_t)c.out_row0 * D.pitch);
    } else {
        if ((uint64_t)D.x0 + c.target_width > D.w || (uint64_t)D.y0 + fine_rows(c, *d).y1 > D.h)
            return bad("the frame does not fit the array at its origin");
        o.surf = D.surf;
        o.array = 1u;
        o.x0 = D.x0;
        o.y0 = D.y0;
    }
    d->out = o;
    return VB_OK;
}

// ---- backgrounds: vb_set_background -----------------------------------------------------------------------------------------
// The descriptor is checked as vb_register_destination checks it (destination_of); whether it covers a frame, in
// resolve_background. Frames keep the background they were issued with (Frame::bg), so an array's surface object is destroyed
// only once every frame that can read it, a streamed frame's re-run included, has completed. Rule: r->bg never names a
// destroyed surface. Once the old one is released, r->bg is cleared, and the new background is installed only if every step
// succeeded; on a failure the renderer is left without a background.
extern "C" int vb_set_background(vb_renderer *r, const vb_destination *d) {
    if (!r) return VB_E_INVALID;
    Background b;
    if (d) {
        if (int rc = destination_of(r, d, "vb_set_background", &b.d)) return rc;
        b.on = true;
    }
    if (r->bg.d.surf) {
        // complete the frames that read the old array, whatever they report (a streamed frame may have failed for good)
        int rc = drain_stream(r);
        cudaError_t e = cudaSetDevice(r->device);
        if (e == cudaSuccess) e = cudaStreamSynchronize(r->stream);
        // a stream that did not complete may still read the old surface: it is then forgotten, not destroyed
        if (e == cudaSuccess) e = cudaDestroySurfaceObject(r->bg.d.surf);
        r->bg = Background{};
        if (rc == VB_OK && e != cudaSuccess) {
            r->err = std::string("vb_set_background: ") + cudaGetErrorString(e);
            rc = VB_E_CUDA;
        }
        if (rc) {
            if (b.d.surf) cudaDestroySurfaceObject(b.d.surf);
            return rc;
        }
    }
    r->bg = b;
    return VB_OK;
}

// The frame r prepared starts from bg: check that bg covers it, and say what fine reads (d->bg). Like a destination, a
// background holds the whole frame, so a window or a read-back band reads its own rows.
int vb_host::resolve_background(vb_renderer *r, const Background &bg, Dest *d) {
    d->bg = VbFineBg{};
    if (!bg.on) return VB_OK;
    auto bad = [&](const std::string &why) {
        r->err = std::string("background: ") + why;
        return VB_E_INVALID;
    };
    const VbConfig &c = r->cfg;
    const Destination &D = bg.d;
    VbFineBg g{};
    g.on = 1u;
    g.texel = D.texel();
    g.premul = D.premul;
    g.bgra = D.format == VB_DEST_BGRA8;
    if (D.kind == VB_DEST_LINEAR) {
        if (D.pitch < (size_t)c.target_width * g.texel) return bad("the row pitch is below " + std::to_string(g.texel) + " * width");
        g.ptr = D.ptr;
        g.pitch = D.pitch;
    } else {
        if (c.n_cells > 1u) return bad("an array cannot be the background of a batch (vb_set_cells with more than one cell)");
        if ((uint64_t)D.x0 + c.target_width > D.w || (uint64_t)D.y0 + fine_rows(c, *d).y1 > D.h)
            return bad("the frame does not fit the array at its origin");
        g.surf = D.surf;
        g.array = 1u;
        g.x0 = D.x0;
        g.y0 = D.y0;
    }
    d->bg = g;
    return VB_OK;
}

// ---- batches: many scenes of one size in one pass (vb_scene_batch builds the scene) ---------------------------------------
// The offsets split the uploaded scene's draw objects into cells. Validated here against the uploaded draw tags (one download):
// a cell whose clips do not balance would pair a BEGIN_CLIP of one cell with an END_CLIP of the next. What depends on the
// frame size (arena indexing) and on the call (windows) is checked when a frame is prepared.
extern "C" int vb_set_cells(vb_renderer *r, const uint32_t *draw_offsets, uint32_t n_cells) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const std::string &why) {
        r->err = "vb_set_cells: " + why;
        return VB_E_INVALID;
    };
    if (!draw_offsets || n_cells == 0u) return bad("no offsets");
    if (!r->cur->have_scene) return VB_E_NO_SCENE;
    if (r->xc.enabled || r->grouped) return bad("a batch cannot be combined with vb_group or the exchange");
    int rc = drain_stream(r);
    if (rc) return rc;
    CK(cudaSetDevice(r->device));
    const VbLayout &L = r->cur->layout;
    const uint32_t n_draw = L.n_draw_objects;
    if (draw_offsets[0] != 0u || draw_offsets[n_cells] != n_draw) return bad("offsets must start at 0 and end at the scene's draw-object count");
    for (uint32_t c = 0; c < n_cells; c++)
        if (draw_offsets[c + 1] < draw_offsets[c]) return bad("offsets must not decrease");
    r->dmg.epoch++;
    if (n_cells == 1u) { // the whole scene: no batch
        r->cells.clear();
        hit_forget(r);
        return VB_OK;
    }
    std::vector<uint32_t> tags(n_draw);
    if (n_draw) {
        CK(cudaMemcpyAsync(tags.data(), (const uint32_t *)r->cur->scene.p + L.draw_tag_base, (size_t)n_draw * 4, cudaMemcpyDeviceToHost, r->stream));
        CK(cudaStreamSynchronize(r->stream));
    }
    for (uint32_t c = 0; c < n_cells; c++) {
        int64_t depth = 0;
        for (uint32_t i = draw_offsets[c]; i < draw_offsets[c + 1] && depth >= 0; i++)
            depth += tags[i] == VB_DRAWTAG_BEGIN_CLIP ? 1 : tags[i] == VB_DRAWTAG_END_CLIP ? -1 : 0;
        if (depth != 0) return bad("the clips of cell " + std::to_string(c) + " do not balance");
    }
    hit_forget(r); // cell_draw, which the answers read, is rewritten below
    if ((rc = ensure(r, r->cell_draw, ((size_t)n_cells + 1u) * 4u))) return rc;
    r->cells.assign(draw_offsets, draw_offsets + n_cells + 1u);
    // in stream order: a frame still running reads the previous offsets
    CK(cudaMemcpyAsync(r->cell_draw.p, r->cells.data(), r->cells.size() * 4u, cudaMemcpyHostToDevice, r->stream));
    return VB_OK;
}

// ---- Resolver::resolve on the device (resolve.rs:183-399): see include/vello_b200.h and k_resolve.cu ---------------------------
// Streams a resolve can read: a pointer for every stream with elements, stops for every ramp patch, every patch in the draw data.
int vb_host::check_streams(vb_renderer *r, const vb_encoding_streams *e, const char *who) {
    auto bad = [&](const char *why) {
        r->err = std::string(who) + ": " + why;
        return VB_E_INVALID;
    };
    if ((e->n_path_tags && !e->path_tags) || (e->n_path_data && !e->path_data) || (e->n_draw_tags && !e->draw_tags) ||
        (e->n_draw_data && !e->draw_data) || (e->n_transforms && !e->transforms) || (e->n_styles && !e->styles) ||
        (e->n_ramp_patches && !e->ramp_patches) || (e->n_image_patches && !e->image_patches))
        return bad("a stream with elements and no pointer");
    for (uint32_t i = 0; i < e->n_ramp_patches; i++) {
        const vb_ramp_patch &p = e->ramp_patches[i];
        if (!p.n_stops || !p.stops || p.draw_data_offset >= e->n_draw_data) return bad("a ramp patch without stops or outside the draw data");
    }
    for (uint32_t i = 0; i < e->n_image_patches; i++) {
        const vb_image_patch &im = e->image_patches[i];
        if (im.draw_data_offset >= e->n_draw_data) return bad("an image patch outside the draw data");
        if (!vb_atlas_side_fits(im.width, im.height)) return bad("an image with a side over 65535 texels");
    }
    return VB_OK;
}

// The pixels of an image placed at (x, y): with an override on this renderer, a blit from its memory, kept in `over` for
// refresh_overrides (*overridden). Otherwise the caller's to copy; a registered texture has pixels only as an override's.
int vb_host::image_source(vb_renderer *r, const char *who, const void *key, uint32_t w, uint32_t h, uint32_t x, uint32_t y,
                        std::vector<VbBlitRect> &blits, std::vector<vb_renderer::SceneSlot::OverridePlace> &over, bool *overridden) {
    const auto ov = key ? r->overrides.find(key) : r->overrides.end();
    *overridden = ov != r->overrides.end();
    if (*overridden) {
        const vb_renderer::Override &o = ov->second;
        if (o.w != w || o.h != h) {
            r->err = std::string(who) + ": an override's size differs from its image's (" + std::to_string(o.w) + "x" + std::to_string(o.h) + " vs " +
                     std::to_string(w) + "x" + std::to_string(h) + ")";
            return VB_E_INVALID;
        }
        blits.push_back(VbBlitRect{o.src, o.pitch, 0, w, h, x, y, 0, 0});
        over.push_back({key, o.src, o.pitch, w, h, x, y, false});
    } else if (vb_texture_key(key)) {
        r->err = std::string(who) + ": a registered texture has no override on this renderer";
        return VB_E_INVALID;
    }
    return VB_OK;
}

// The installed scene's ramp patches and their encoded stops, for vb_bind_gradient_stops: host copies, no device work.
static void keep_stops(vb_renderer *r, const vb_encoding_streams *e) {
    vb_renderer::SceneSlot &s = *r->cur;
    s.stop_patches.reserve(e->n_ramp_patches);
    for (uint32_t i = 0; i < e->n_ramp_patches; i++) {
        const vb_ramp_patch &p = e->ramp_patches[i];
        s.stop_patches.push_back({p.draw_data_offset, p.n_stops, p.premul_interp ? 1u : 0u, (uint32_t)s.stops.size()});
        s.stops.insert(s.stops.end(), p.stops, p.stops + p.n_stops);
    }
    s.have_stops = true;
}

extern "C" int vb_scene_upload_streams(vb_renderer *r, const vb_encoding_streams *e, vb_layout *layout_out) {
    if (!r || !e) return VB_E_INVALID;
    int rc = check_streams(r, e, "vb_scene_upload_streams");
    if (rc) return rc;
    VbResolvePlan plan;
    const int planned = vb_resolve_plan(*e, &plan);
    if (planned == VB_PLAN_LAYOUT) {
        r->err = "vb_scene_upload_streams: the scene exceeds 32-bit word offsets";
        return VB_E_INVALID;
    }
    VbLayout L;
    memcpy(&L, &plan.layout, sizeof L);
    if ((rc = drain_stream(r))) return rc;
    CK(cudaSetDevice(r->device));
    cudaStream_t st = r->stream;
    // each planned image is filled from an override on this renderer (one k_atlas_blit) or from the host; the images placed
    // before one the atlas refused are checked first, as when each image is placed and checked in turn
    std::vector<VbBlitRect> blits;
    std::vector<vb_renderer::SceneSlot::OverridePlace> over;
    std::vector<const VbResolvePlan::Image *> from_host;
    for (const VbResolvePlan::Image &q : plan.images) {
        bool overridden;
        if ((rc = image_source(r, "device resolve", q.pixels, q.w, q.h, q.x, q.y, blits, over, &overridden))) return rc;
        if (!overridden && q.pixels && q.w && q.h) from_host.push_back(&q);
    }
    if (planned == VB_PLAN_ATLAS) {
        r->err = "device resolve: an image's atlas place or size passes 16 bits (at most 65535 rows of shelves and 65535 "
                 "texels a side)";
        return VB_E_INVALID;
    }
    std::vector<RsRamp> ramps;
    std::vector<vb_ramp_stop> stops;
    for (const vb_ramp_patch *p : plan.ramps) {
        ramps.push_back(RsRamp{(uint32_t)stops.size(), p->n_stops, p->premul_interp ? 1u : 0u, 0u});
        stops.insert(stops.end(), p->stops, p->stops + p->n_stops);
    }
    DiffedUpload guard;
    if ((rc = upload_diff_begin(r, st, L, plan.words, (uint32_t)ramps.size(), plan.atlas_w, plan.atlas_h, guard))) return rc;

    // the six streams go straight to their places in the packed buffer
    if ((rc = ensure(r, r->cur->scene, regions_of(L, plan.words, false, r->view.on, false, false).bytes))) return rc;
    char *base = (char *)r->cur->scene.p;
    if (e->n_path_tags) CK(cudaMemcpyAsync(base, e->path_tags, e->n_path_tags, cudaMemcpyHostToDevice, st));
    if (e->n_path_data) CK(cudaMemcpyAsync(base + (size_t)L.path_data_base * 4, e->path_data, (size_t)e->n_path_data * 4, cudaMemcpyHostToDevice, st));
    if (e->n_draw_tags) CK(cudaMemcpyAsync(base + (size_t)L.draw_tag_base * 4, e->draw_tags, (size_t)e->n_draw_tags * 4, cudaMemcpyHostToDevice, st));
    if (e->n_draw_data) CK(cudaMemcpyAsync(base + (size_t)L.draw_data_base * 4, e->draw_data, (size_t)e->n_draw_data * 4, cudaMemcpyHostToDevice, st));
    if (e->n_transforms) CK(cudaMemcpyAsync(base + (size_t)L.transform_base * 4, e->transforms, (size_t)e->n_transforms * 24, cudaMemcpyHostToDevice, st));
    if (e->n_styles) CK(cudaMemcpyAsync(base + (size_t)L.style_base * 4, e->styles, (size_t)e->n_styles * 8, cudaMemcpyHostToDevice, st));
    // patches, ramp descriptors and stops in one staging buffer
    static_assert(sizeof(RsStop) == sizeof(vb_ramp_stop), "the stops are staged as the caller gave them");
    const size_t pb = plan.patches.size() * sizeof(RsPatch), rb = ramps.size() * sizeof(RsRamp), sb = stops.size() * sizeof(vb_ramp_stop);
    const size_t o_r = (pb + 15) & ~(size_t)15, o_s = (o_r + rb + 15) & ~(size_t)15;
    if ((rc = ensure(r, r->resolve_tmp, o_s + sb + 16))) return rc;
    char *tmp = (char *)r->resolve_tmp.p;
    if (pb) CK(cudaMemcpyAsync(tmp, plan.patches.data(), pb, cudaMemcpyHostToDevice, st));
    if (rb) CK(cudaMemcpyAsync(tmp + o_r, ramps.data(), rb, cudaMemcpyHostToDevice, st));
    if (sb) CK(cudaMemcpyAsync(tmp + o_s, stops.data(), sb, cudaMemcpyHostToDevice, st));
    vb_launch_resolve_finish((uint32_t *)r->cur->scene.p, e->n_path_tags, e->n_open_clips, plan.padded_tags, L.draw_tag_base + e->n_draw_tags,
                             (const RsPatch *)tmp, (uint32_t)plan.patches.size(), st);
    if ((rc = ensure(r, r->cur->ramps, ramps.size() * 512 * 4))) return rc;
    vb_launch_make_ramps((const RsRamp *)(tmp + o_r), (const RsStop *)(tmp + o_s), (uint32_t)ramps.size(), (uint32_t *)r->cur->ramps.p, st);
    if ((rc = ensure(r, r->cur->atlas, (size_t)plan.atlas_w * plan.atlas_h * 4))) return rc;
    CK(cudaMemsetAsync(r->cur->atlas.p, 0, (size_t)plan.atlas_w * plan.atlas_h * 4, st));
    for (const VbResolvePlan::Image *q : from_host)
        CK(cudaMemcpy2DAsync((char *)r->cur->atlas.p + ((size_t)q->y * plan.atlas_w + q->x) * 4, (size_t)plan.atlas_w * 4, q->pixels, (size_t)q->w * 4,
                             (size_t)q->w * 4, q->h, cudaMemcpyHostToDevice, st));
    if ((rc = enqueue_blits(r, blits, r->cur->atlas.p, plan.atlas_w))) return rc;
    CK(cudaGetLastError());
    // the host vectors above are read by the asynchronous copies: they must outlive them
    CK(cudaStreamSynchronize(st));
    set_scene(r, L, plan.words, (uint32_t)ramps.size(), plan.atlas_w, plan.atlas_h, std::move(over), false);
    keep_stops(r, e);
    if (layout_out) memcpy(layout_out, &L, sizeof(vb_layout));
    return VB_OK;
}
