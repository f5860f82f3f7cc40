// vb_compose.cu -- composition of resident fragments: vb_fragment_upload / vb_fragment_free, vb_compose and vb_recompose
// (k_compose.cu, k_recompose.cu), bound instance transforms (vb_bind_instance_transforms), bound draw colours
// (vb_bind_draw_colors, k_colors.cu), bound path points (vb_bind_path_points, k_points.cu), bound gradient stops
// (vb_bind_gradient_stops, k_resolve.cu) and bound transforms (vb_bind_transforms, k_transforms.cu); fragments built from
// device arrays (vb_fragment_from_device_paths, k_device_paths.cu).
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "vb_device.cuh"
#include "vb_diff.h"
#include "vb_renderer.h"
#include "vb_resolve.h"
#include "vb_textures.h"

// ---- composition of resident fragments: vb_fragment_upload / vb_fragment_free / vb_compose (k_compose.cu) ---------------------
// The ramp key of patch p, with one more reference. A key made here is appended to `fresh`: its stops still need a place in
// the stop pool (place_stops).
static RampKey *intern_ramp(vb_renderer *r, const vb_ramp_patch &p, std::vector<RampKey *> &fresh) {
    const bool premul = p.premul_interp != 0u;
    const bool self_equal = vb_same_ramp(p.stops, p.n_stops, premul, p.stops, p.n_stops, premul);
    const uint64_t h = vb_ramp_hash(p.stops, p.n_stops, premul);
    if (self_equal) {
        const auto it = r->ramp_by_hash.find(h);
        if (it != r->ramp_by_hash.end())
            for (RampKey *k : it->second)
                if (vb_same_ramp(k->stops.data(), (uint32_t)k->stops.size(), k->premul, p.stops, p.n_stops, premul)) {
                    k->refs++;
                    return k;
                }
    }
    std::unique_ptr<RampKey> k(new RampKey());
    k->stops.assign(p.stops, p.stops + p.n_stops);
    k->premul = premul;
    k->self_equal = self_equal;
    k->id = r->next_ramp_key++;
    k->refs = 1;
    RampKey *raw = k.get();
    if (self_equal) r->ramp_by_hash[h].push_back(raw);
    r->ramp_keys[raw->id] = std::move(k);
    fresh.push_back(raw);
    return raw;
}
static void release_ramp(vb_renderer *r, RampKey *k) {
    if (--k->refs) return;
    if (k->self_equal) {
        auto it = r->ramp_by_hash.find(vb_ramp_hash(k->stops.data(), (uint32_t)k->stops.size(), k->premul));
        it->second.erase(std::find(it->second.begin(), it->second.end(), k));
        if (it->second.empty()) r->ramp_by_hash.erase(it);
    }
    r->ramp_keys.erase(k->id); // its stops stay in the pool until the pool is rebuilt
}
// An image key names one set of pixels. The caller's buffer need not outlive vb_fragment_upload, so its address may come back
// holding other pixels in a later fragment: host pixels are told apart by a hash of their bytes as well as by the pointer,
// and only a pointer that holds the same pixels again shares an atlas slot. NULL and registered-texture keys are never read
// (hash 0): they are one image per pointer, as in a resolve.
static bool readable_image(const void *key, uint32_t w, uint32_t h) { return key && w && h && !vb_texture_key(key); }
static uint64_t hash_pixels(const void *key, uint32_t w, uint32_t h) {
    const uint8_t *p = (const uint8_t *)key;
    const size_t n = (size_t)w * h * 4u;
    uint64_t a = 0x9e3779b97f4a7c15ull ^ n, b = 0xc2b2ae3d27d4eb4full;
    size_t i = 0;
    for (; i + 16u <= n; i += 16u) {
        uint64_t x, y;
        memcpy(&x, p + i, 8);
        memcpy(&y, p + i + 8, 8);
        a = (a ^ x) * 0xff51afd7ed558ccdull;
        b = (b ^ y) * 0xc4ceb9fe1a85ec53ull;
        a ^= a >> 29;
        b ^= b >> 31;
    }
    for (; i < n; i += 4u) { // w * h * 4 is a multiple of 4
        uint32_t x;
        memcpy(&x, p + i, 4);
        a = (a ^ x) * 0xff51afd7ed558ccdull;
        a ^= a >> 29;
    }
    const uint64_t h64 = (a ^ (b * 0x9e3779b97f4a7c15ull)) * 0xff51afd7ed558ccdull;
    return h64 ^ (h64 >> 32);
}
static ImageKey *intern_image(vb_renderer *r, const void *key, uint32_t w, uint32_t h, uint64_t pixels_hash) {
    std::unique_ptr<ImageKey> &k = r->image_keys[std::make_tuple(key, w, h, pixels_hash)];
    if (!k) {
        k.reset(new ImageKey());
        k->key = key;
        k->w = w;
        k->h = h;
        k->pixels_hash = pixels_hash;
        k->id = r->next_image_key++;
    }
    k->refs++;
    return k.get();
}
static void release_image(vb_renderer *r, ImageKey *k) {
    if (--k->refs == 0u) r->image_keys.erase(std::make_tuple(k->key, k->w, k->h, k->pixels_hash));
}
static void release_keys(vb_renderer *r, const Fragment &f) {
    for (const Fragment::Ramp &x : f.ramps) release_ramp(r, x.key);
    for (const Fragment::Image &x : f.images) release_image(r, x.key);
}

// Copy the stops of new ramp keys into the stop pool. When they do not fit, the pool is made anew from the live keys (their
// stops are on the host), after the work already enqueued, which may read the old pool, has finished.
static int place_stops(vb_renderer *r, const std::vector<RampKey *> &fresh) {
    size_t add = 0;
    for (const RampKey *k : fresh) add += k->stops.size();
    if (add == 0) return VB_OK;
    std::vector<vb_ramp_stop> host;
    size_t first = r->pool_used;
    if ((r->pool_used + add) * sizeof(vb_ramp_stop) <= r->stop_pool.cap) {
        for (RampKey *k : fresh) {
            k->pool = (uint32_t)(first + host.size());
            host.insert(host.end(), k->stops.begin(), k->stops.end());
        }
    } else {
        size_t live = 0;
        for (const auto &e : r->ramp_keys) live += e.second->stops.size();
        if (live > 0x7fffffffu) {
            r->err = "vb_fragment_upload: more gradient stops than 32-bit indices reach";
            return VB_E_INVALID;
        }
        CK(cudaStreamSynchronize(r->stream));
        CK(cudaFree(r->stop_pool.p));
        r->stop_pool = DevBuf{};
        int rc = ensure(r, r->stop_pool, 2 * live * sizeof(vb_ramp_stop));
        if (rc) return rc;
        first = 0;
        for (auto &e : r->ramp_keys) {
            e.second->pool = (uint32_t)host.size();
            host.insert(host.end(), e.second->stops.begin(), e.second->stops.end());
        }
    }
    CK(cudaMemcpy((vb_ramp_stop *)r->stop_pool.p + first, host.data(), host.size() * sizeof(vb_ramp_stop), cudaMemcpyHostToDevice));
    r->pool_used = (uint32_t)(first + host.size());
    return VB_OK;
}

// Release the memory of freed fragments that no enqueued work reads any more.
static void reap_freed(vb_renderer *r) {
    auto &v = r->freed;
    for (size_t i = 0; i < v.size();) {
        if (cudaEventQuery(v[i].done) != cudaSuccess) {
            cudaGetLastError(); // cudaErrorNotReady is not an error of the next call
            i++;
            continue;
        }
        cudaFree(v[i].mem);
        cudaEventDestroy(v[i].done);
        r->fragment_bytes -= v[i].bytes;
        v[i] = v.back();
        v.pop_back();
    }
}

// A fragment's allocation (k_compose.cu reads it): the header of CMP_HEADER_WORDS words, each stream's word offset, then the
// streams back to back in CMP_* order, the path tags padded to whole words. `units` are the streams' lengths as Fragment::len
// counts them (tag bytes, words, draw tags, words, transforms, style words); off[] gets the header and the result is the
// allocation's bytes for them (0 when past 32-bit word offsets), before any image pixels.
static size_t fragment_layout(const uint64_t units[CMP_STREAMS], uint64_t off[CMP_HEADER_WORDS]) {
    const uint64_t words[CMP_STREAMS] = {(units[CMP_TAGS] + 3u) / 4u, units[CMP_PATH_DATA], units[CMP_DRAW_TAGS], units[CMP_DRAW_DATA],
                                         6u * units[CMP_TRANSFORMS], units[CMP_STYLES]};
    uint64_t w = CMP_HEADER_WORDS;
    for (int s = 0; s < (int)CMP_HEADER_WORDS; s++) off[s] = 0u;
    for (int s = 0; s < CMP_STREAMS; s++) {
        off[s] = w;
        w += words[s];
    }
    if (w + 4u > 0xfffffff0ull) return 0u;
    return ((size_t)(w + 4u) * 4u + 15u) & ~(size_t)15u;
}

// Account and register the fragment f, whose allocation holds its streams of lengths `units` (fragment_layout): the renderer
// owns it from now on under a new id, which is returned.
static uint32_t fragment_register(vb_renderer *r, std::unique_ptr<Fragment> f, const uint64_t units[CMP_STREAMS], uint32_t n_paths,
                                  uint32_t n_clips, uint32_t n_open_clips, uint32_t info) {
    for (int s = 0; s < CMP_STREAMS; s++) f->len[s] = (uint32_t)units[s];
    f->n_paths = n_paths;
    f->n_clips = n_clips;
    f->n_open_clips = n_open_clips;
    f->info = info;
    f->id = r->next_fragment++;
    r->fragment_bytes += f->bytes;
    const uint32_t id = f->id;
    r->fragments[id] = std::move(f);
    return id;
}

static size_t up16(size_t v) { return (v + 15u) & ~(size_t)15u; }
// Grow a buffer compose writes. Work already enqueued may read it: growing waits for the renderer's stream.
static int compose_room(vb_renderer *r, DevBuf &b, size_t bytes) {
    if (b.cap >= std::max<size_t>(bytes, 256)) return VB_OK;
    CK(cudaStreamSynchronize(r->stream));
    return ensure(r, b, bytes);
}

extern "C" int vb_fragment_upload(vb_renderer *r, const vb_encoding_streams *e, uint32_t *fragment_out) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const char *why) {
        r->err = std::string("vb_fragment_upload: ") + why;
        return VB_E_INVALID;
    };
    if (!e || !fragment_out) return bad("NULL streams or id");
    if (check_streams(r, e, "vb_fragment_upload")) return VB_E_INVALID;
    // the allocation: header, the six streams, then one copy of each image key's pixels
    uint64_t off[CMP_HEADER_WORDS];
    const uint64_t units[CMP_STREAMS] = {e->n_path_tags, e->n_path_data, e->n_draw_tags, e->n_draw_data, e->n_transforms, 2ull * e->n_styles};
    size_t bytes = fragment_layout(units, off);
    if (!bytes) return bad("the fragment's streams exceed 32-bit word offsets");
    CK(cudaSetDevice(r->device));
    reap_freed(r);
    std::unique_ptr<Fragment> f(new Fragment());
    std::vector<std::pair<size_t, const Fragment::Image *>> copies; // (offset in the allocation, image) per key with pixels
    std::unordered_map<const ImageKey *, size_t> at;
    std::map<std::tuple<const void *, uint32_t, uint32_t>, uint64_t> hashed; // each of this fragment's images is read once
    for (uint32_t i = 0; i < e->n_image_patches; i++) {
        const vb_image_patch &im = e->image_patches[i];
        uint64_t hv = 0;
        if (readable_image(im.pixels, im.width, im.height)) {
            const auto t = std::make_tuple((const void *)im.pixels, im.width, im.height);
            const auto it = hashed.find(t);
            hv = it != hashed.end() ? it->second : (hashed[t] = hash_pixels(im.pixels, im.width, im.height));
        }
        f->images.push_back(Fragment::Image{im.draw_data_offset, intern_image(r, im.pixels, im.width, im.height, hv), nullptr});
    }
    for (Fragment::Image &x : f->images) {
        // a registered texture's key points at nothing: its pixels exist only in device memory (an override, at compose)
        if (!readable_image(x.key->key, x.key->w, x.key->h) || at.count(x.key)) continue;
        at[x.key] = bytes;
        copies.push_back({bytes, &x});
        bytes += ((size_t)x.key->w * x.key->h * 4u + 15u) & ~(size_t)15u;
    }
    std::vector<RampKey *> fresh;
    for (uint32_t i = 0; i < e->n_ramp_patches; i++) {
        const vb_ramp_patch &p = e->ramp_patches[i];
        f->ramps.push_back(Fragment::Ramp{p.draw_data_offset, p.extend, intern_ramp(r, p, fresh)});
    }
    int rc = place_stops(r, fresh);
    cudaError_t ce = rc ? cudaSuccess : cudaMalloc(&f->mem, bytes);
    if (rc || ce != cudaSuccess) {
        release_keys(r, *f);
        if (ce != cudaSuccess) {
            r->err = std::string("vb_fragment_upload: cudaMalloc: ") + cudaGetErrorString(ce);
            return VB_E_CUDA;
        }
        return rc;
    }
    f->bytes = bytes;
    for (Fragment::Image &x : f->images) {
        const auto it = at.find(x.key);
        if (it != at.end()) x.pixels = (const uint8_t *)f->mem + it->second;
    }
    uint32_t header[CMP_HEADER_WORDS];
    for (int s = 0; s < (int)CMP_HEADER_WORDS; s++) header[s] = (uint32_t)off[s];
    char *base = (char *)f->mem;
    const void *src[CMP_STREAMS] = {e->path_tags, e->path_data, e->draw_tags, e->draw_data, e->transforms, e->styles};
    const size_t len_bytes[CMP_STREAMS] = {e->n_path_tags, (size_t)e->n_path_data * 4, (size_t)e->n_draw_tags * 4, (size_t)e->n_draw_data * 4,
                                           (size_t)e->n_transforms * 24, (size_t)e->n_styles * 8};
    cudaStream_t st = r->upload_stream;
    ce = cudaMemcpyAsync(base, header, sizeof header, cudaMemcpyHostToDevice, st);
    for (int s = 0; s < CMP_STREAMS && ce == cudaSuccess; s++)
        if (len_bytes[s]) ce = cudaMemcpyAsync(base + off[s] * 4u, src[s], len_bytes[s], cudaMemcpyHostToDevice, st);
    for (size_t i = 0; i < copies.size() && ce == cudaSuccess; i++) {
        const ImageKey &k = *copies[i].second->key;
        ce = cudaMemcpyAsync(base + copies[i].first, k.key, (size_t)k.w * k.h * 4u, cudaMemcpyHostToDevice, st);
    }
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
        cudaFree(f->mem);
        release_keys(r, *f);
        r->err = std::string("vb_fragment_upload: copying the streams: ") + cudaGetErrorString(ce);
        return VB_E_CUDA;
    }
    *fragment_out = fragment_register(r, std::move(f), units, e->n_paths, e->n_clips, e->n_open_clips,
                                      (uint32_t)vb_draw_info_sum(e->draw_tags, e->n_draw_tags));
    return VB_OK;
}

extern "C" int vb_fragment_free(vb_renderer *r, uint32_t fragment) {
    if (!r) return VB_E_INVALID;
    const auto it = r->fragments.find(fragment);
    if (it == r->fragments.end()) {
        r->err = "vb_fragment_free: unknown or freed fragment " + std::to_string(fragment);
        return VB_E_INVALID;
    }
    CK(cudaSetDevice(r->device));
    reap_freed(r);
    // composes already enqueued read the memory: it is released once the stream has passed this point (reap_freed)
    cudaEvent_t done;
    CK(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    const cudaError_t ce = cudaEventRecord(done, r->stream);
    if (ce != cudaSuccess) {
        cudaEventDestroy(done);
        r->err = std::string("vb_fragment_free: ") + cudaGetErrorString(ce);
        return VB_E_CUDA;
    }
    r->freed.push_back({it->second->mem, it->second->bytes, done});
    release_keys(r, *it->second);
    r->fragments.erase(it);
    return VB_OK;
}

// ---- fragments from device arrays: vb_fragment_from_device_paths / _curves / _dashes (k_device_paths.cu, k_device_dashes.cu) --
// The streams' lengths depend on the data (dropped points, closing lines, cap markers), so the fragment is allocated for the
// worst case of the counts, the four launches write it, and the totals and the error word come back through pinned memory
// after one synchronisation of the renderer's stream.
static const uint32_t STROKE_JOINS[3] = {0u, 0x10000000u, 0x20000000u}, STROKE_CAPS[3] = {0u, 0x01000000u, 0x02000000u}; // path.rs:30-66
static bool one_of(uint32_t v, const uint32_t (&set)[3]) { return v == set[0] || v == set[1] || v == set[2]; }

// What a device check's error word says (VB_DP_ERR_*), naming the first offending row `at`.
static std::string device_paths_error(uint32_t kind, const std::string &at) {
    if (kind == VB_DP_ERR_RING_OFFSETS) return "ring_offsets[" + at + "] breaks the offsets: they start at 0, never decrease and end at n_points";
    if (kind == VB_DP_ERR_PATH_OFFSETS) return "path_offsets[" + at + "] breaks the offsets: they start at 0, never decrease and end at n_rings";
    if (kind == VB_DP_ERR_POINTS) return "point " + at + " is not finite";
    if (kind == VB_DP_ERR_KINDS)
        return "point_kinds[" + at + "] breaks the kinds: each is 0 (on-curve) or 1 (off-curve), a ring starts and ends on-curve, "
               "and at most two off-curve points come in a row";
    if (kind == VB_DP_ERR_DASH_OFFSETS)
        return "the dash offset of path " + at + " is not finite, or is more than 2^24 pattern entries before the pattern's start";
    return "the colour of path " + at + " is not finite";
}

// A dash offset's pre-roll into the pattern (dash_path in vb_scene.cpp): the dash index, bit 31 set when that dash is not drawn,
// and what remains of it; false past the native front end's 2^24 steps.
static bool dash_phase(const double *pattern, uint32_t n, double offset, uint32_t *ix, double *rem) {
    uint32_t i = 0u, inactive = 0u;
    double r = pattern[0] - offset;
    for (uint32_t guard = 0u; r < 0.0; guard++) {
        if (guard > (1u << 24)) return false;
        i = (i + 1u) % n;
        r += pattern[i];
        inactive ^= 1u;
    }
    *ix = i | (inactive << 31);
    *rem = r;
    return true;
}

// The dashes of vb_fragment_from_device_dashes, cut on the device (k_device_dashes.cu) into an intermediate of sub-rings in
// r->dashes_mid: *mid gets d with its points, offsets and counts replaced by the intermediate's, *mid_kinds its point kinds and
// *mid_flags its VB_DP_RING_* flags. The arguments are checked; the device checks the arrays, then the totals come back through
// pinned memory after one synchronisation of the renderer's stream.
static int dash_intermediate(vb_renderer *r, const char *fn, const vb_device_paths *d, const uint8_t *kinds, const vb_dash *dash,
                             vb_device_paths *mid, const uint8_t **mid_kinds, const uint8_t **mid_flags) {
    auto bad = [&](const std::string &why) {
        r->err = std::string(fn) + ": " + why;
        return VB_E_INVALID;
    };
    const uint64_t P = d->n_points, R = d->n_rings, N = d->n_paths, D = dash->n_pattern;
    // the scratch: [err, ring_first] set to all ones; [ring_last, ring_odd, the rings' prefixes and totals, the look-back's
    // leading words] to zero; the rest of the look-back, the ring records, the paths' phases, the pattern
    const uint32_t parts = vb_device_dashes_parts((uint32_t)R);
    const size_t o_first = 16u, o_zero = up16(o_first + 4u * R), o_odd = o_zero + 4u * R, o_excl = up16(o_odd + 4u * R);
    const size_t o_lb = up16(o_excl + 8u * (R + 1u)), o_rec = up16(o_lb + 4u * vb_lookback_words(parts, 2)), o_rem = o_rec + 16u * R;
    const size_t o_ix = o_rem + 8u * N, o_pat = up16(o_ix + 4u * N), scratch = o_pat + 8u * D;
    int rc;
    if ((rc = compose_room(r, r->dashes_tmp, scratch))) return rc;
    char *t = (char *)r->dashes_tmp.p;
    DpArgs c;
    memset(&c, 0, sizeof c);
    c.points = d->points;
    c.kinds = d->n_points ? kinds : nullptr;
    c.ring_offsets = d->ring_offsets;
    c.path_offsets = d->path_offsets;
    c.colors = d->colors;
    c.point_pitch = d->point_pitch_bytes;
    c.color_pitch = d->color_pitch_bytes;
    c.n_points = (uint32_t)P, c.n_rings = (uint32_t)R, c.n_paths = (uint32_t)N;
    c.kind = d->kind;
    c.err = (unsigned long long *)t;
    c.ring_first = (uint32_t *)(t + o_first);
    c.ring_last = (uint32_t *)(t + o_zero);
    c.ring_odd = (uint32_t *)(t + o_odd);
    DdArgs a;
    memset(&a, 0, sizeof a);
    a.points = d->points;
    a.kinds = c.kinds;
    a.ring_offsets = d->ring_offsets;
    a.path_offsets = d->path_offsets;
    a.point_pitch = d->point_pitch_bytes;
    a.n_points = (uint32_t)P, a.n_rings = (uint32_t)R, a.n_paths = (uint32_t)N, a.n_parts = parts;
    a.closed = d->closed ? 1u : 0u, a.n_pattern = (uint32_t)D;
    a.pattern = (const double *)(t + o_pat);
    for (uint32_t k = 0; k < dash->n_pattern; k++) a.pattern_period += dash->pattern[k];
    a.err = c.err;
    a.rec = (uint4 *)(t + o_rec);
    a.excl = (uint2 *)(t + o_excl);
    a.lookback = (uint32_t *)(t + o_lb);
    if (dash->offsets) {
        a.offsets = dash->offsets;
        a.offset_pitch = dash->offset_pitch_bytes;
        a.phase_rem = (double *)(t + o_rem);
        a.phase_ix = (uint32_t *)(t + o_ix);
    } else {
        dash_phase(dash->pattern, dash->n_pattern, dash->offset, &a.scalar_ix, &a.scalar_rem); // checked by the caller
    }
    cudaStream_t st = r->stream;
    PinnedStage &stage = r->pinned[PIN_COMPOSE];
    uint8_t *h;
    if ((rc = stage_host(r, stage, 16u + 8u * D, &h))) return rc;
    memcpy(h + 16u, dash->pattern, 8u * D);
    cudaError_t e2 = cudaMemsetAsync(t, 0xff, o_zero, st);
    if (e2 == cudaSuccess) e2 = cudaMemsetAsync(t + o_zero, 0, o_lb - o_zero + 4u * VB_LB_ZERO_WORDS(parts), st);
    if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(t + o_pat, h + 16u, 8u * D, cudaMemcpyHostToDevice, st);
    if (e2 == cudaSuccess && (rc = stage_copied(r, stage))) return rc;
    if (e2 == cudaSuccess) {
        vb_launch_device_dashes(c, a, st);
        e2 = cudaGetLastError();
    }
    if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(h, t, 8u, cudaMemcpyDeviceToHost, st);
    if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(h + 8u, t + o_excl + 8u * R, 8u, cudaMemcpyDeviceToHost, st);
    if (e2 == cudaSuccess) e2 = cudaStreamSynchronize(st);
    if (e2 != cudaSuccess) {
        r->err = std::string(fn) + ": " + cudaGetErrorString(e2);
        return VB_E_CUDA;
    }
    unsigned long long err;
    uint32_t tot[2];
    memcpy(&err, h, 8u);
    memcpy(tot, h + 8u, 8u);
    if (err != ~0ull) return bad(device_paths_error((uint32_t)(err >> 32), std::to_string((uint32_t)err)));
    if (tot[0] > 0x7fffffffu || tot[1] > 0x7fffffffu) return bad("the dashes' points or sub-rings exceed int32 offsets (a ring is refused before its walk "
                                                                   "when its control polygon's length allows 2^31 dash breaks)");
    // the intermediate: points, ring offsets, path offsets, then the kind and flag bytes
    const uint64_t MP = tot[0], MR = tot[1];
    const size_t o_roff = 8u * MP, o_poff = o_roff + 4u * (MR + 1u), o_kinds = o_poff + 4u * (N + 1u), o_flags = o_kinds + MP;
    if ((rc = compose_room(r, r->dashes_mid, o_flags + MR))) return rc;
    char *m = (char *)r->dashes_mid.p;
    a.out_points = (float *)m;
    a.out_ring_offsets = (int32_t *)(m + o_roff);
    a.out_path_offsets = (int32_t *)(m + o_poff);
    a.out_kinds = (uint8_t *)(m + o_kinds);
    a.out_flags = (uint8_t *)(m + o_flags);
    vb_launch_device_dashes_emit(a, st);
    if ((e2 = cudaGetLastError()) != cudaSuccess) {
        r->err = std::string(fn) + ": " + cudaGetErrorString(e2);
        return VB_E_CUDA;
    }
    *mid = *d;
    mid->points = a.out_points, mid->n_points = (uint32_t)MP, mid->point_pitch_bytes = 8u;
    mid->ring_offsets = a.out_ring_offsets, mid->n_rings = (uint32_t)MR;
    mid->path_offsets = a.out_path_offsets;
    mid->closed = 0u;
    *mid_kinds = a.out_kinds;
    *mid_flags = a.out_flags;
    return VB_OK;
}

// vb_fragment_from_device_paths (kinds NULL: every point on-curve), vb_fragment_from_device_curves and, with `dash`,
// vb_fragment_from_device_dashes; `fn` names the call.
static int from_device(vb_renderer *r, const char *fn, const vb_device_paths *d, const uint8_t *kinds, const vb_dash *dash,
                       uint32_t *fragment_out, uint32_t *n_draw_objects_out) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const std::string &why) {
        r->err = std::string(fn) + ": " + why;
        return VB_E_INVALID;
    };
    if (!d || !fragment_out) return bad("NULL paths or id");
    if (r->grouped || r->xc.enabled || r->xc.configured) return bad("not available for a renderer of a vb_group or with the exchange");
    if (r->frame_pending) return bad("a frame is enqueued and not finished (vb_frame_finish)");
    const uint64_t P = d->n_points, R = d->n_rings, N = d->n_paths;
    if (P > 0x7fffffffu || R > 0x7fffffffu || N > 0x7fffffffu) return bad("n_points, n_rings and n_paths must fit int32 offsets");
    if ((P && !d->points) || ((P || R) && !d->ring_offsets) || (N && !d->colors)) return bad("NULL points, ring_offsets or colors with a non-zero count");
    if (!d->path_offsets && N != R) return bad("without path_offsets every ring is a path: n_paths must equal n_rings");
    if (d->point_pitch_bytes < 8u || d->point_pitch_bytes % 4u || d->point_pitch_bytes > 0xffffffffu)
        return bad("the point pitch must be a multiple of 4 bytes, at least 8 and below 4 GiB");
    if (d->color_pitch_bytes < 16u || d->color_pitch_bytes % 4u || d->color_pitch_bytes > 0xffffffffu)
        return bad("the colour pitch must be a multiple of 4 bytes, at least 16 and below 4 GiB");
    uint32_t flags = 0u, width = 0u;
    if (d->kind == 0u) {
        if (d->fill_rule > 1u) return bad("fill_rule must be 0 (non-zero) or 1 (even-odd)");
        flags = d->fill_rule ? 0x40000000u : 0u; // style_from_fill
    } else if (d->kind == 1u) {
        if (!one_of(d->join, STROKE_JOINS)) return bad("join must be VB_JOIN_BEVEL, VB_JOIN_MITER or VB_JOIN_ROUND");
        if (!one_of(d->start_cap, STROKE_CAPS) || !one_of(d->end_cap, STROKE_CAPS)) return bad("the caps must be VB_CAP_BUTT, VB_CAP_SQUARE or VB_CAP_ROUND");
        if (!(isfinite(d->width) && d->width > 0.0f)) return bad("the stroke width must be finite and > 0");
        if (!isfinite(d->miter_limit)) return bad("the miter limit must be finite");
        flags = 0x80000000u | d->join | (d->start_cap << 2) | d->end_cap | vb_f32_to_f16(d->miter_limit); // style_from_stroke
        memcpy(&width, &d->width, 4);
    } else {
        return bad("kind must be 0 (fill) or 1 (stroke)");
    }
    if (dash) {
        if (d->kind != 1u) return bad("dashes apply to strokes: kind must be 1");
        if (!dash->pattern || !dash->n_pattern) return bad("the dash pattern is empty");
        double sum = 0.0;
        for (uint32_t k = 0; k < dash->n_pattern; k++) {
            if (!(isfinite(dash->pattern[k]) && dash->pattern[k] >= 0.0)) return bad("the dash pattern's entries must be finite and >= 0");
            sum += dash->pattern[k];
        }
        if (!(sum > 0.0)) return bad("the dash pattern's entries sum to 0");
        if (dash->offsets) {
            if (dash->offset_pitch_bytes < 4u || dash->offset_pitch_bytes % 4u || dash->offset_pitch_bytes > 0xffffffffu)
                return bad("the dash offsets' pitch must be a multiple of 4 bytes, at least 4 and below 4 GiB");
        } else {
            uint32_t ix;
            double rem;
            if (!isfinite(dash->offset) || !dash_phase(dash->pattern, dash->n_pattern, dash->offset, &ix, &rem))
                return bad("the dash offset is not finite, or is more than 2^24 pattern entries before the pattern's start");
        }
    }
    // the worst case: a tag per point, the closing line and a cap marker per ring, a PATH tag per path, the TRANSFORM and STYLE
    // tags; 2 words per point and 4 per ring (closing line and cap line, or cap quad); a draw object per path (for dashes, of
    // the intermediate's counts, below)
    uint64_t off[CMP_HEADER_WORDS];
    const uint64_t worst[CMP_STREAMS] = {N ? 2u + P + 2u * R + N : 0u, 2u * P + 4u * R, N, N, N ? 1u : 0u, N ? 2u : 0u};
    size_t bytes = fragment_layout(worst, off);
    if (!bytes && !dash) return bad("the fragment's worst-case streams exceed 32-bit word offsets");
    CK(cudaSetDevice(r->device));
    const void *ptrs[6] = {d->points, d->ring_offsets, d->path_offsets, d->colors, d->draw_index, dash ? dash->offsets : nullptr};
    for (const void *p : ptrs)
        if (p && ((uintptr_t)p % 4u || !device_memory_of(r, p)))
            return bad("every array must be 4-byte aligned device or managed memory of the renderer's device");
    if (kinds && d->n_points && !device_memory_of(r, kinds)) return bad("point_kinds must be device or managed memory of the renderer's device");
    reap_freed(r);

    vb_device_paths mid;
    const uint8_t *ring_flags = nullptr;
    int rc;
    if (dash) {
        if ((rc = dash_intermediate(r, fn, d, kinds, dash, &mid, &kinds, &ring_flags))) return rc;
        d = &mid;
        const uint64_t MP = d->n_points, MR = d->n_rings;
        const uint64_t mworst[CMP_STREAMS] = {N ? 2u + MP + 2u * MR + N : 0u, 2u * MP + 4u * MR, N, N, N ? 1u : 0u, N ? 2u : 0u};
        if (!(bytes = fragment_layout(mworst, off))) return bad("the fragment's worst-case streams exceed 32-bit word offsets");
    }
    const uint64_t MP = d->n_points, MR = d->n_rings;
    // the scratch (DpArgs): [err, ring_first, path_min] set to all ones, [totals, ring_last, ring_odd, path_kept, the look-back's
    // leading words] to zero, then the rest of the look-back, the partitions' prefixes, the ring records and the keep bytes
    const uint32_t parts = vb_device_paths_parts((uint32_t)MP);
    const size_t lb_words = vb_lookback_words(parts, 3);
    const size_t o_first = 16u, o_min = o_first + 4u * MR, o_zero = up16(o_min + (ring_flags ? 4u * N : 0u)), o_last = o_zero + 16u;
    const size_t o_odd = o_last + 4u * MR, o_kept = o_odd + 4u * MR;
    const size_t o_lb = up16(o_kept + 4u * N), o_excl = up16(o_lb + 4u * lb_words), o_rings = up16(o_excl + 12u * parts);
    const size_t o_keep = o_rings + 16u * MR, scratch = o_keep + MP;
    if ((rc = compose_room(r, r->paths_tmp, scratch))) return rc;
    char *t = (char *)r->paths_tmp.p;
    std::unique_ptr<Fragment> f(new Fragment());
    const cudaError_t ce = cudaMalloc(&f->mem, bytes);
    if (ce != cudaSuccess) {
        r->err = std::string(fn) + ": cudaMalloc: " + cudaGetErrorString(ce);
        return VB_E_CUDA;
    }
    f->bytes = bytes;
    DpArgs a;
    memset(&a, 0, sizeof a);
    a.points = d->points;
    a.kinds = d->n_points ? kinds : nullptr;
    a.ring_offsets = d->ring_offsets;
    a.path_offsets = d->path_offsets;
    a.colors = d->colors;
    a.point_pitch = d->point_pitch_bytes;
    a.color_pitch = d->color_pitch_bytes;
    a.n_points = (uint32_t)MP, a.n_rings = (uint32_t)MR, a.n_paths = (uint32_t)N, a.n_parts = parts;
    a.kind = d->kind, a.closed = d->closed ? 1u : 0u, a.style_flags = flags, a.style_width = width;
    a.err = (unsigned long long *)t;
    a.ring_first = (uint32_t *)(t + o_first);
    a.totals = (uint32_t *)(t + o_zero);
    a.ring_last = (uint32_t *)(t + o_last);
    a.ring_odd = (uint32_t *)(t + o_odd);
    a.path_kept = (uint32_t *)(t + o_kept);
    a.lookback = (uint32_t *)(t + o_lb);
    a.part_excl = (uint32_t *)(t + o_excl);
    a.rings = (uint4 *)(t + o_rings);
    a.keep_fix = (uint8_t *)(t + o_keep);
    a.fragment = (uint32_t *)f->mem;
    a.draw_index = d->draw_index;
    a.ring_flags = ring_flags;
    a.path_min = ring_flags ? (uint32_t *)(t + o_min) : nullptr;
    cudaStream_t st = r->stream;
    PinnedStage &stage = r->pinned[PIN_COMPOSE];
    uint8_t *h;
    auto fail = [&](int code) {
        cudaFree(f->mem);
        return code;
    };
    if ((rc = stage_host(r, stage, 32u, &h))) return fail(rc);
    cudaError_t e2 = cudaMemsetAsync(t, 0xff, o_zero, st);
    if (e2 == cudaSuccess) e2 = cudaMemsetAsync(t + o_zero, 0, o_lb - o_zero + 4u * VB_LB_ZERO_WORDS(parts), st);
    if (e2 == cudaSuccess) {
        vb_launch_device_paths(a, st);
        e2 = cudaGetLastError();
    }
    if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(h, t, 8u, cudaMemcpyDeviceToHost, st);
    if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(h + 8u, t + o_zero, 12u, cudaMemcpyDeviceToHost, st);
    if (e2 == cudaSuccess) e2 = cudaStreamSynchronize(st);
    if (e2 != cudaSuccess) {
        r->err = std::string(fn) + ": " + cudaGetErrorString(e2);
        return fail(VB_E_CUDA);
    }
    unsigned long long err;
    uint32_t tot[3];
    memcpy(&err, h, 8u);
    memcpy(tot, h + 8u, 12u);
    if (err != ~0ull) {
        const std::string at = std::to_string((uint32_t)err);
        fail(0);
        // the dashes' intermediate passed the arrays' checks: only a piece's point can fail, rounded to f32 past its range
        if (dash) return bad("point " + at + " of the dashes is not finite in f32");
        return bad(device_paths_error((uint32_t)(err >> 32), at));
    }
    const uint64_t units[CMP_STREAMS] = {N ? 2u + tot[0] : 0u, tot[1], tot[2], tot[2], N ? 1u : 0u, N ? 2u : 0u};
    *fragment_out = fragment_register(r, std::move(f), units, tot[2], 0u, 0u, tot[2]); // FILL_COLOR has one info word
    if (n_draw_objects_out) *n_draw_objects_out = tot[2];
    return VB_OK;
}
extern "C" int vb_fragment_from_device_paths(vb_renderer *r, const vb_device_paths *d, uint32_t *fragment_out, uint32_t *n_draw_objects_out) {
    return from_device(r, "vb_fragment_from_device_paths", d, nullptr, nullptr, fragment_out, n_draw_objects_out);
}
extern "C" int vb_fragment_from_device_curves(vb_renderer *r, const vb_device_paths *d, const uint8_t *point_kinds, uint32_t *fragment_out,
                                              uint32_t *n_draw_objects_out) {
    return from_device(r, "vb_fragment_from_device_curves", d, point_kinds, nullptr, fragment_out, n_draw_objects_out);
}
extern "C" int vb_fragment_from_device_dashes(vb_renderer *r, const vb_device_paths *d, const uint8_t *point_kinds, const vb_dash *dash,
                                              uint32_t *fragment_out, uint32_t *n_draw_objects_out) {
    if (!r) return VB_E_INVALID;
    if (!dash) {
        r->err = "vb_fragment_from_device_dashes: NULL dash";
        return VB_E_INVALID;
    }
    return from_device(r, "vb_fragment_from_device_dashes", d, point_kinds, dash, fragment_out, n_draw_objects_out);
}


// The resident fragment of an id; nullptr when there is none (never uploaded, or freed).
static const Fragment *find_fragment(const vb_renderer *r, uint32_t id) {
    const auto it = r->fragments.find(id);
    return it == r->fragments.end() ? nullptr : it->second.get();
}

// The tables k_compose_streams reads for n instances: [the per-stream exclusive prefix of the instances' lengths,
// CMP_STREAMS x (n + 1) words] [the fragments' addresses, at o_src] [the transforms, at o_xf]; `bytes` in all.
struct CmpTables {
    size_t o_src, o_xf, bytes;
};
static CmpTables cmp_tables(size_t n) {
    CmpTables t;
    t.o_src = up16((size_t)CMP_STREAMS * (n + 1u) * 4u);
    t.o_xf = up16(t.o_src + n * 8u);
    t.bytes = up16(t.o_xf + n * sizeof(CmpXform));
    return t;
}
// Write the tables for instances fr with transforms xf (nullptr: none applied) at h, and return the CmpArgs that read their
// copy at dev. The caller sets the scene, the destinations and the units.
static CmpArgs stage_cmp_tables(const std::vector<const Fragment *> &fr, const CmpXform *xf, uint8_t *h, const char *dev) {
    const uint32_t n = (uint32_t)fr.size();
    const CmpTables t = cmp_tables(n);
    for (int s = 0; s < CMP_STREAMS; s++) {
        uint32_t *P = (uint32_t *)h + (size_t)s * (n + 1u);
        P[0] = 0u;
        for (uint32_t k = 0; k < n; k++) P[k + 1] = P[k] + fr[k]->len[s];
    }
    unsigned long long *srcs = (unsigned long long *)(h + t.o_src);
    for (uint32_t k = 0; k < n; k++) srcs[k] = (unsigned long long)(uintptr_t)fr[k]->mem;
    if (xf) memcpy(h + t.o_xf, xf, (size_t)n * sizeof(CmpXform));
    else memset(h + t.o_xf, 0, (size_t)n * sizeof(CmpXform));
    CmpArgs a;
    memset(&a, 0, sizeof a);
    a.prefix = (const uint32_t *)dev;
    a.src = (const unsigned long long *)(dev + t.o_src);
    a.xf = (const CmpXform *)(dev + t.o_xf);
    a.n = n;
    return a;
}

// vb_compose and vb_recompose. A recompose that damage tracking can follow (a composed base: base_diffable) also matches the
// instances against the current scene's, and begins the diff (diff_begin) with the tables of k_recompose_damage.
static int compose(vb_renderer *r, const char *fn, const vb_instance *inst, uint32_t n, vb_layout *layout_out, uint32_t *draw_offsets,
                   bool recompose) {
    if (!r) return VB_E_INVALID;
    auto bad = [&](const std::string &why) {
        r->err = std::string(fn) + ": " + why;
        return VB_E_INVALID;
    };
    if (n && !inst) return bad("NULL instances");
    if (r->grouped || r->xc.enabled) return bad("not available for a renderer of a vb_group or with the exchange enabled");
    if (r->frame_pending) return bad("a frame is enqueued and not finished (vb_frame_finish)");
    // validate everything and size the scene before anything is written
    std::vector<const Fragment *> fr(n);
    std::vector<CmpXform> xf(n);
    uint64_t tot[CMP_STREAMS] = {}, n_paths = 0, n_clips = 0, n_open = 0, info = 0;
    for (uint32_t k = 0; k < n; k++) {
        if (!(fr[k] = find_fragment(r, inst[k].fragment))) return bad("unknown or freed fragment " + std::to_string(inst[k].fragment));
        memset(&xf[k], 0, sizeof xf[k]);
        xf[k].on = inst[k].has_transform ? 1u : 0u;
        for (int c = 0; c < 6 && xf[k].on; c++) {
            xf[k].m[c] = (float)inst[k].transform[c]; // Transform::from_kurbo
            if (!isfinite(xf[k].m[c])) return bad("instance " + std::to_string(k) + ": the transform must be finite in f32");
        }
        for (int s = 0; s < CMP_STREAMS; s++) tot[s] += fr[k]->len[s];
        n_paths += fr[k]->n_paths;
        n_clips += fr[k]->n_clips;
        n_open += fr[k]->n_open_clips;
        info += fr[k]->info;
    }
    VbLayout L;
    uint32_t padded;
    size_t total_words;
    if (!vb_resolve_layout(tot[CMP_TAGS], tot[CMP_PATH_DATA], tot[CMP_DRAW_TAGS], tot[CMP_DRAW_DATA], tot[CMP_TRANSFORMS], tot[CMP_STYLES] / 2u, n_open,
                           n_paths, n_clips, info, &L, &padded, &total_words))
        return bad("the composed scene exceeds 32-bit word offsets");

    // late-bound ramps and images of every instance in order: the host resolve's de-duplication and shelf placement, keyed
    // by the keys the fragments hold
    const uint64_t seq = ++r->compose_seq;
    std::vector<RsPatch> patches;
    std::vector<RsRamp> ramps;
    std::vector<uint32_t> ramp_ids;
    struct Placed { const ImageKey *key; const uint8_t *src; uint32_t x, y, frag; };
    std::vector<Placed> placed;
    std::vector<uint32_t> img_pre(n + 1u, 0u), img_local; // each instance's images: their place in `placed`
    VbShelfPacker shelf;
    uint32_t dd0 = L.draw_data_base;
    for (uint32_t k = 0; k < n; k++) {
        const Fragment &f = *fr[k];
        img_pre[k + 1] = img_pre[k] + (uint32_t)f.images.size();
        for (const Fragment::Ramp &p : f.ramps) {
            RampKey *key = p.key;
            if (key->stamp != seq || !key->self_equal) {
                key->stamp = seq;
                key->local = (uint32_t)ramps.size();
                ramps.push_back(RsRamp{key->pool, (uint32_t)key->stops.size(), key->premul ? 1u : 0u, 0u});
                ramp_ids.push_back(key->id);
            }
            patches.push_back(RsPatch{dd0 + p.dd, (key->local << 2) | p.extend});
        }
        for (const Fragment::Image &im : f.images) {
            ImageKey *key = im.key;
            if (key->stamp != seq) {
                key->stamp = seq;
                key->local = (uint32_t)placed.size();
                placed.push_back(Placed{key, im.pixels, 0, 0, f.id});
                if (!shelf.place(key->w, key->h, &placed.back().x, &placed.back().y))
                    return bad("the composed atlas places an image below row 65535, past the draw data's 16-bit field");
            }
            const Placed &q = placed[key->local];
            patches.push_back(RsPatch{dd0 + im.dd, (q.x << 16) | q.y});
            img_local.push_back(key->local);
        }
        dd0 += f.len[CMP_DRAW_DATA];
    }
    const uint32_t atlas_w = shelf.width, atlas_h = shelf.height();
    // images with an override on this renderer come from its device memory, the others from their fragment's copy
    std::vector<VbBlitRect> blits;
    std::vector<vb_renderer::SceneSlot::OverridePlace> over;
    std::vector<uint64_t> atlas_keys;
    int rc;
    for (const Placed &q : placed) {
        const ImageKey &k = *q.key;
        bool overridden;
        if ((rc = image_source(r, fn, k.key, k.w, k.h, q.x, q.y, blits, over, &overridden))) return rc;
        if (!overridden && q.src) blits.push_back(VbBlitRect{q.src, (uint64_t)k.w * 4u, 0, k.w, k.h, q.x, q.y, 0, 0});
        // where the slot's pixels come from: the fragment, an override (never a fragment id), or nowhere (a zero region)
        atlas_keys.push_back((uint64_t)k.id << 32 | (overridden ? CMP_FROM_OVERRIDE : q.src ? q.frag : 0u));
    }
    std::vector<ImgPlace> img_place(img_local.size());
    for (size_t t = 0; t < img_local.size(); t++) {
        const Placed &q = placed[img_local[t]];
        img_place[t] = ImgPlace{atlas_keys[img_local[t]], (q.x << 16) | q.y};
    }

    // vb_recompose: match the new instances to the current scene's (vb_diff.h). A matched instance whose images moved in the
    // atlas, or come from an override (copied again by this compose), is unmatched: fine samples in atlas coordinates.
    const vb_renderer::SceneSlot &was = *r->cur;
    const bool arm = recompose && was.composed && was.inst_draw.size() == was.inst_frag.size() + 1u &&
                     was.inst_img.size() == was.inst_frag.size() + 1u && base_diffable(r);
    const uint32_t n_old = arm ? (uint32_t)was.inst_frag.size() : 0u;
    std::vector<uint32_t> match(arm ? n : 0u), unmatched(n_old, 1u);
    if (arm) {
        vb_diff_match(
            n_old, n,
            [&](uint32_t i, uint32_t j) { return was.inst_frag[i] == fr[j]->id && memcmp(&was.inst_xf[i], &xf[j], sizeof(CmpXform)) == 0; },
            match.data());
        for (uint32_t j = 0; j < n; j++) {
            const uint32_t i = match[j];
            if (i == VB_DIFF_NONE) continue;
            const ImgPlace *a = was.img_place.data() + was.inst_img[i], *b = img_place.data() + img_pre[j];
            for (uint32_t t = 0; t < img_pre[j + 1] - img_pre[j] && match[j] != VB_DIFF_NONE; t++)
                if (a[t].key != b[t].key || a[t].xy != b[t].xy || (uint32_t)b[t].key == CMP_FROM_OVERRIDE) match[j] = VB_DIFF_NONE;
            if (match[j] != VB_DIFF_NONE) unmatched[i] = 0u;
        }
    }

    if ((rc = drain_stream(r))) return rc;
    CK(cudaSetDevice(r->device));
    reap_freed(r);
    cudaStream_t st = r->stream;
    vb_renderer::SceneSlot &slot = *r->cur;
    const bool new_ramps = !slot.composed || ramp_ids != slot.ramp_keys;
    const bool new_atlas = !slot.composed || atlas_keys != slot.atlas_keys || !over.empty();
    // the tables, staged through pinned memory: k_compose_streams' (cmp_tables), patches, ramp descriptors
    const size_t o_pat = cmp_tables(n).bytes;
    const size_t o_ramp = up16(o_pat + patches.size() * sizeof(RsPatch)), staged = o_ramp + ramps.size() * sizeof(RsRamp);
    // vb_recompose's tables (vb_rcmp_tables), staged after compose's
    const size_t o_rc = up16(staged), rc_bytes = arm ? vb_rcmp_tables((uint32_t *)nullptr, n_old, n).words * 4u : 0u, host_bytes = o_rc + rc_bytes;
    if ((rc = compose_room(r, r->compose_tmp, staged))) return rc;
    char *tmp = (char *)r->compose_tmp.p;
    PinnedStage &stage = r->pinned[PIN_COMPOSE];
    uint8_t *h;
    if ((rc = stage_host(r, stage, host_bytes, &h))) return rc;
    CmpArgs a = stage_cmp_tables(fr, xf.data(), h, tmp);
    const uint32_t *pre = (const uint32_t *)h;
    if (!patches.empty()) memcpy(h + o_pat, patches.data(), patches.size() * sizeof(RsPatch));
    if (!ramps.empty()) memcpy(h + o_ramp, ramps.data(), ramps.size() * sizeof(RsRamp));
    if (draw_offsets) memcpy(draw_offsets, pre + (size_t)CMP_DRAW_TAGS * (n + 1u), ((size_t)n + 1u) * 4u);
    if (arm) {
        const VbRcmpTables<uint32_t> t = vb_rcmp_tables((uint32_t *)(h + o_rc), n_old, n);
        memcpy(t.old_pre, was.inst_draw.data(), ((size_t)n_old + 1u) * 4u);
        memcpy(t.new_pre, pre + (size_t)CMP_DRAW_TAGS * (n + 1u), ((size_t)n + 1u) * 4u);
        if (n) memcpy(t.map, match.data(), (size_t)n * 4u);
        if (n_old) memcpy(t.unmatched, unmatched.data(), (size_t)n_old * 4u);
    }

    if ((rc = compose_room(r, slot.scene, regions_of(L, total_words, false, r->view.on, false, false).bytes))) return rc;
    if (new_ramps && (rc = compose_room(r, slot.ramps, ramps.size() * 512u * 4u))) return rc;
    if (new_atlas && (rc = compose_room(r, slot.atlas, (size_t)atlas_w * atlas_h * 4u))) return rc;
    if (staged) CK(cudaMemcpyAsync(tmp, h, staged, cudaMemcpyHostToDevice, st));
    if (arm) {
        if ((rc = diff_begin(r, st, false, n_old, n, L.n_draw_objects))) return rc;
        CK(cudaMemcpyAsync((char *)r->dmg_diff.p + r->dmg.diff.o_tables, h + o_rc, rc_bytes, cudaMemcpyHostToDevice, st));
    }
    if ((rc = stage_copied(r, stage))) return rc;
    uint32_t *scene = (uint32_t *)slot.scene.p;
    a.scene = scene;
    const uint32_t dst[CMP_STREAMS] = {L.path_tag_base, L.path_data_base, L.draw_tag_base, L.draw_data_base, L.transform_base, L.style_base};
    const uint32_t units[CMP_STREAMS] = {(uint32_t)((tot[CMP_TAGS] + 3u) / 4u), (uint32_t)tot[CMP_PATH_DATA], (uint32_t)tot[CMP_DRAW_TAGS],
                                         (uint32_t)tot[CMP_DRAW_DATA], (uint32_t)tot[CMP_TRANSFORMS], (uint32_t)tot[CMP_STYLES]};
    memcpy(a.dst, dst, sizeof dst);
    memcpy(a.units, units, sizeof units);
    vb_launch_compose(a, st);
    vb_launch_resolve_finish(scene, (uint32_t)tot[CMP_TAGS], (uint32_t)n_open, padded, L.draw_tag_base + (uint32_t)tot[CMP_DRAW_TAGS],
                             (const RsPatch *)(tmp + o_pat), (uint32_t)patches.size(), st);
    if (new_ramps) {
        vb_launch_make_ramps((const RsRamp *)(tmp + o_ramp), (const RsStop *)r->stop_pool.p, (uint32_t)ramps.size(), (uint32_t *)slot.ramps.p, st);
        slot.ramp_keys = std::move(ramp_ids);
    }
    if (new_atlas) {
        CK(cudaMemsetAsync(slot.atlas.p, 0, (size_t)atlas_w * atlas_h * 4u, st));
        if ((rc = enqueue_blits(r, blits, slot.atlas.p, atlas_w))) return rc;
        slot.atlas_keys = std::move(atlas_keys);
    }
    CK(cudaGetLastError());
    set_scene(r, L, total_words, (uint32_t)ramps.size(), atlas_w, atlas_h, std::move(over), true);
    slot.inst_frag.resize(n);
    for (uint32_t k = 0; k < n; k++) slot.inst_frag[k] = fr[k]->id;
    slot.inst_xf = std::move(xf);
    slot.inst_draw.assign(pre + (size_t)CMP_DRAW_TAGS * (n + 1u), pre + (size_t)(CMP_DRAW_TAGS + 1) * (n + 1u));
    slot.inst_img = std::move(img_pre);
    slot.img_place = std::move(img_place);
    // the instances' ramp patches with their keys' stops, in instance order, for vb_bind_gradient_stops (host copies)
    uint32_t dd_rel = 0u;
    for (uint32_t k = 0; k < n; k++) {
        for (const Fragment::Ramp &p : fr[k]->ramps) {
            const RampKey &key = *p.key;
            slot.stop_patches.push_back({dd_rel + p.dd, (uint32_t)key.stops.size(), key.premul ? 1u : 0u, (uint32_t)slot.stops.size()});
            slot.stops.insert(slot.stops.end(), key.stops.begin(), key.stops.end());
        }
        dd_rel += fr[k]->len[CMP_DRAW_DATA];
    }
    slot.have_stops = true;
    if (layout_out) memcpy(layout_out, &L, sizeof(vb_layout));
    return VB_OK;
}

extern "C" int vb_compose(vb_renderer *r, const vb_instance *inst, uint32_t n, vb_layout *layout_out, uint32_t *draw_offsets) {
    return compose(r, "vb_compose", inst, n, layout_out, draw_offsets, false);
}
extern "C" int vb_recompose(vb_renderer *r, const vb_instance *inst, uint32_t n, vb_layout *layout_out, uint32_t *draw_offsets) {
    const int rc = compose(r, "vb_recompose", inst, n, layout_out, draw_offsets, true);
    if (r) r->dmg.diff.pending = false; // a recompose that failed after diff_begin installed nothing: its diff must not be armed
    return rc;
}
extern "C" uint32_t vb_debug_match_instances(const uint32_t *old_keys, uint32_t n_old, const uint32_t *new_keys, uint32_t n_new, uint32_t *match) {
    return vb_diff_match(n_old, n_new, [&](uint32_t i, uint32_t j) { return old_keys[i] == new_keys[j]; }, match);
}

// ---- bindings to device rows: vb_bind_* -----------------------------------------------------------------------------------------
// A binding points the installed scene at device rows that every frame reads (VbBound). Every kind is bound by one path,
// bind_rows: the checks they share, and what differs between them from BIND_KINDS: the scene a kind needs, how many rows it
// takes and at what pitch, its own checks, and the tables it makes once, here, on the renderer's stream. The tables stay valid
// while the rows are bound, because every scene installation unbinds; every frame after that reads the caller's rows.
using Slot = vb_renderer::SceneSlot;

// The scene a kind binds to, or why there is none (steps 4 and 5 of bind_rows)
static const char *any_scene(const Slot &s) { return s.have_scene ? nullptr : "no scene installed"; }
static const char *composed_scene(const Slot &s) {
    return s.have_scene && s.composed ? nullptr : "the renderer's current scene was not made by vb_compose";
}
static const char *scene_with_stops(const Slot &s) {
    if (!s.have_scene) return "no scene installed";
    if (!s.have_stops)
        return "the scene was installed as packed bytes, whose gradients exist only as resolved ramps; install it from its "
               "streams (vb_scene_upload_streams, vb_scene_upload_device, vb_render_scene) or with vb_compose";
    return nullptr;
}

// The rows a scene takes at most (instances: exactly)
static uint64_t n_instances(const Slot &s) { return s.inst_frag.size(); }
static uint64_t n_draws(const Slot &s) { return s.layout.n_draw_objects; }
static uint64_t n_points(const Slot &s) { return n_path_data(s.layout, s.scene_words) / 2u; }
static uint64_t n_stops(const Slot &s) { return s.stops.size(); }
static uint64_t n_xforms(const Slot &s) { return n_transforms(s.layout, s.scene_words); }

// The kinds' own checks, after the shared ones: why n rows cannot be bound, or nothing
static std::string freed_fragment(const vb_renderer *r, uint32_t) {
    for (uint32_t id : r->cur->inst_frag)
        if (!find_fragment(r, id)) return "fragment " + std::to_string(id) + " of the composed scene was freed";
    return {};
}
static std::string draw_tags_outside(const Slot &s, uint64_t n) {
    if ((uint64_t)s.layout.draw_tag_base + n > s.scene_words) return "the scene's draw tags do not lie inside its words";
    return {};
}
static std::string draw_tags_check(const vb_renderer *r, uint32_t n) { return draw_tags_outside(*r->cur, n); }
static std::string path_tags_outside(const vb_renderer *r, uint32_t) {
    const VbLayout &L = r->cur->layout;
    if (L.path_data_base < L.path_tag_base || L.path_data_base > r->cur->scene_words) return "the scene's path tags do not lie inside its words";
    return {};
}
// bound gradient stops bind the scene's first ramp patches: those with a stop below n (the stops are concatenated in patch order)
static uint32_t bound_grads(const Slot &s, uint32_t n) {
    uint32_t g = 0u;
    while (g < s.stop_patches.size() && s.stop_patches[g].first < n) g++;
    return g;
}
static std::string stops_check(const vb_renderer *r, uint32_t n) {
    const Slot &s = *r->cur;
    if ((uint64_t)s.n_ramps + bound_grads(s, n) > (1ull << 30)) return "the scene's ramps and one per bound gradient pass the 30 bits of the ramp word";
    return draw_tags_outside(s, s.layout.n_draw_objects);
}
static std::string no_check(const vb_renderer *, uint32_t) { return {}; }

// The kinds' bind-time work: the tables of n rows in b. `why` is set for a refusal that only the work finds.

// Bound instance transforms (k_compose.cu): the transform prefix and compose-time transforms from the slot's instance records,
// the untransformed transforms by one k_compose_streams over the transform stream alone (no transforms applied, destination
// 0), and the instances' draw prefix, for damage tracking.
static int instance_tables(vb_renderer *r, uint32_t n, VbBound &b, std::string &) {
    const Slot &slot = *r->cur;
    std::vector<const Fragment *> fr(n);
    for (uint32_t k = 0; k < n; k++) fr[k] = find_fragment(r, slot.inst_frag[k]);
    const uint32_t n_tr = n_transforms(slot.layout, slot.scene_words);
    // staged through pinned memory: [the copy's tables (cmp_tables), with no transforms] [the binding's tables: transform
    // prefix (n + 1), compose-time transforms] [the instances' draw prefix (n + 1)]
    reap_freed(r);
    const size_t tmp_bytes = cmp_tables(n).bytes;
    const size_t o_xf = up16(((size_t)n + 1u) * 4u), o_tr = up16(o_xf + (size_t)n * sizeof(CmpXform));
    const size_t o_draw = up16(o_tr + (size_t)n_tr * 24u), draw_bytes = ((size_t)n + 1u) * 4u; // staged right after the tables
    const size_t staged = tmp_bytes + o_tr + draw_bytes;
    int rc;
    if ((rc = compose_room(r, r->compose_tmp, tmp_bytes))) return rc;
    char *tmp = (char *)r->compose_tmp.p;
    PinnedStage &stage = r->pinned[PIN_COMPOSE];
    uint8_t *h;
    if ((rc = stage_host(r, stage, staged, &h))) return rc;
    CmpArgs a = stage_cmp_tables(fr, nullptr, h, tmp);
    memcpy(h + tmp_bytes, (const uint32_t *)h + (size_t)CMP_TRANSFORMS * (n + 1u), ((size_t)n + 1u) * 4u);
    memcpy(h + tmp_bytes + o_xf, slot.inst_xf.data(), (size_t)n * sizeof(CmpXform));
    memcpy(h + tmp_bytes + o_tr, slot.inst_draw.data(), draw_bytes);

    if ((rc = compose_room(r, r->inst_tables, o_draw + draw_bytes))) return rc;
    cudaStream_t st = r->stream;
    char *tables = (char *)r->inst_tables.p;
    CK(cudaMemcpyAsync(tmp, h, tmp_bytes, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tables, h + tmp_bytes, o_tr, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tables + o_draw, h + tmp_bytes + o_tr, draw_bytes, cudaMemcpyHostToDevice, st));
    if ((rc = stage_copied(r, stage))) return rc;
    a.scene = (uint32_t *)(tables + o_tr);
    a.units[CMP_TRANSFORMS] = n_tr;
    vb_launch_compose(a, st);
    CK(cudaGetLastError());
    b.inst_prefix = (const uint32_t *)tables;
    b.inst_xf = (const CmpXform *)(tables + o_xf);
    b.inst_src = (const uint32_t *)(tables + o_tr);
    b.inst_draw = (const uint32_t *)(tables + o_draw);
    return VB_OK;
}

// Bound path points (k_points.cu): the table of each path's first point, by one k_path_point_slots over the scene's path tags,
// and its 16-bit flag, read back (the call's one synchronisation).
static int point_tables(vb_renderer *r, uint32_t, VbBound &b, std::string &why) {
    const Slot &slot = *r->cur;
    const VbLayout &L = slot.layout;
    int rc;
    if ((rc = compose_room(r, r->point_slots, ((size_t)L.n_paths + 2u) * 4u))) return rc;
    cudaStream_t st = r->stream;
    uint32_t *first = (uint32_t *)r->point_slots.p, *flag = first + L.n_paths + 1u;
    CK(cudaMemsetAsync(first, 0, ((size_t)L.n_paths + 2u) * 4u, st));
    vb_launch_path_point_slots((const uint32_t *)slot.scene.p + L.path_tag_base, L.path_data_base - L.path_tag_base, L.n_paths, first, flag,
                               nullptr, st);
    CK(cudaGetLastError());
    uint32_t i16 = 0u;
    CK(cudaMemcpyAsync(&i16, flag, 4u, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (i16) {
        why = "the scene has 16-bit path segments, whose points are not f32 pairs";
        return VB_E_INVALID;
    }
    b.pt_first = first;
    return VB_OK;
}

// Bound gradient stops (k_resolve.cu): the tables, and the scene's ramps copied into the first rows of stop_ramps. The call's
// one synchronisation waits for the tables' copy. The draw-data slot table follows (bind_rows).
static int stop_tables(vb_renderer *r, uint32_t n, VbBound &b, std::string &) {
    const Slot &slot = *r->cur;
    const VbLayout &L = slot.layout;
    const uint32_t n_grads = bound_grads(slot, n);
    // the tables: [each gradient's ramp word, relative to the draw data] [the gradients (RsRamp), at o_grads] [their stops as
    // encoded, at o_stops] [draw object -> gradient, at o_draw]
    const Slot::StopPatch *last = n_grads ? &slot.stop_patches[n_grads - 1u] : nullptr;
    const size_t s_used = last ? (size_t)last->first + last->n_stops : 0u;
    const size_t o_grads = up16((size_t)n_grads * 4u), o_stops = up16(o_grads + (size_t)n_grads * sizeof(RsRamp));
    const size_t o_draw = up16(o_stops + s_used * sizeof(RsStop)), bytes = o_draw + (size_t)L.n_draw_objects * 4u;
    std::vector<uint8_t> h(bytes, 0u);
    uint32_t *dd = (uint32_t *)h.data();
    RsRamp *grads = (RsRamp *)(h.data() + o_grads);
    for (uint32_t g = 0; g < n_grads; g++) {
        const Slot::StopPatch &p = slot.stop_patches[g];
        grads[g] = RsRamp{p.first, p.n_stops, p.premul, 0u};
        dd[g] = p.dd;
    }
    if (s_used) memcpy(h.data() + o_stops, slot.stops.data(), s_used * sizeof(RsStop));
    memset(h.data() + o_draw, 0xff, (size_t)L.n_draw_objects * 4u);
    int rc;
    if ((rc = compose_room(r, r->stop_tables, bytes))) return rc;
    if ((rc = compose_room(r, r->stop_ramps, ((size_t)slot.n_ramps + n_grads) * 512u * 4u))) return rc;
    cudaStream_t st = r->stream;
    const char *t = (const char *)r->stop_tables.p;
    CK(cudaMemcpyAsync(r->stop_tables.p, h.data(), bytes, cudaMemcpyHostToDevice, st));
    if (slot.n_ramps) CK(cudaMemcpyAsync(r->stop_ramps.p, slot.ramps.p, (size_t)slot.n_ramps * 512u * 4u, cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st)); // h is read by the copy
    b.rs_grads = (const RsRamp *)(t + o_grads);
    b.rs_stops = (const RsStop *)(t + o_stops);
    b.rs_draw = (const uint32_t *)(t + o_draw);
    b.rs_grads_n = n_grads;
    b.rs_ramp0 = slot.n_ramps;
    return VB_OK;
}

// Bound transforms (k_transforms.cu): each path's transform range, which damage tracking reads, by one k_path_point_slots over
// the scene's path tags (the walk bound points use).
static int transform_tables(vb_renderer *r, uint32_t, VbBound &b, std::string &) {
    const VbLayout &L = r->cur->layout;
    int rc;
    if ((rc = compose_room(r, r->xform_ranges, (size_t)L.n_paths * 8u))) return rc;
    cudaStream_t st = r->stream;
    uint2 *range = (uint2 *)r->xform_ranges.p;
    if (L.n_paths) CK(cudaMemsetAsync(range, 0xff, (size_t)L.n_paths * 8u, st));
    vb_launch_path_point_slots((const uint32_t *)r->cur->scene.p + L.path_tag_base, L.path_data_base - L.path_tag_base, L.n_paths, nullptr,
                               nullptr, range, st);
    CK(cudaGetLastError());
    b.xf_range = range;
    return VB_OK;
}

// Bound visibility (k_visibility.cu): only the mask is sized, which every frame packs the caller's rows into, and which flatten
// culls the hidden draw objects' tags by. The call does not synchronise unless the mask grows.
static int visibility_mask(vb_renderer *r, uint32_t, VbBound &, std::string &) {
    return compose_room(r, r->vis_mask, (size_t)vb_vis_words(r->cur->layout) * 4u);
}
// Bound stroke widths (k_widths.cu): only the snapshot is sized, which every frame reads the caller's rows into, and which
// flatten takes the bound strokes' widths from. The call does not synchronise unless the snapshot grows.
static int width_snapshot(vb_renderer *r, uint32_t, VbBound &, std::string &) {
    return compose_room(r, r->width_snap, (size_t)vb_width_entries(r->cur->layout) * 4u);
}
static int no_tables(vb_renderer *, uint32_t, VbBound &, std::string &) { return VB_OK; }

// The draw-data slot table of bound colours, bound gradient stops and bound opacity (k_colors.cu), made from b whenever one
// of them changes and one of them stays bound: every word VB_COLOR_NONE, then one k_draw_data_slots over the draw tags the
// bound rows reach, which also writes the bound gradients' draw objects to rs_draw. The call does not synchronise unless the
// table grows.
static int draw_data_slots(vb_renderer *r, VbBound &b) {
    b.dd_slots = nullptr;
    if (!draw_data_bound(b)) return VB_OK;
    const Slot &slot = *r->cur;
    const VbLayout &L = slot.layout;
    const uint32_t n_dd = n_draw_data(L, slot.scene_words);
    int rc;
    if ((rc = compose_room(r, r->dd_slots, (size_t)n_dd * 4u))) return rc;
    cudaStream_t st = r->stream;
    uint32_t *slots = (uint32_t *)r->dd_slots.p;
    if (n_dd) CK(cudaMemsetAsync(slots, 0xff, (size_t)n_dd * 4u, st));
    const uint32_t *scene = (const uint32_t *)slot.scene.p;
    const uint32_t *grad_dd = b.rows[VB_BIND_STOPS].rows ? (const uint32_t *)r->stop_tables.p : nullptr;
    vb_launch_draw_data_slots(b, scene + L.draw_tag_base, scene + L.draw_data_base, n_dd, L.n_draw_objects, grad_dd, slots, st);
    CK(cudaGetLastError());
    b.dd_slots = slots;
    return VB_OK;
}

// What differs between the kinds of binding, in VB_BIND_* order
struct BindKind {
    const char *fn;                                   // the entry point, which vb_last_error names
    bool enabled_only;                                // refused with the exchange enabled only, not once it is configured
    const char *(*scene)(const Slot &s);              // why the installed scene cannot be bound, or nullptr
    uint64_t (*rows)(const Slot &s);                  // the rows it takes at most (`exact`: exactly)
    bool exact;
    const char *unit;                                 // what a row is, in the row-count error
    uint32_t min_pitch;                               // bytes; 1: byte rows at any pitch and alignment
    bool region;                                      // frames write a region past the scene for it (regions_of)
    std::string (*check)(const vb_renderer *r, uint32_t n);
    int (*tables)(vb_renderer *r, uint32_t n, VbBound &b, std::string &why);
};
static const BindKind BIND_KINDS[VB_N_BINDINGS] = {
    {"vb_bind_instance_transforms", true, composed_scene, n_instances, true, " instances", 24u, true, freed_fragment, instance_tables},
    {"vb_bind_draw_colors", false, any_scene, n_draws, false, " draw objects (1 .. n_draw_objects)", 16u, true, draw_tags_check, no_tables},
    {"vb_bind_path_points", false, any_scene, n_points, false, " points (1 .. n_points)", 8u, true, path_tags_outside, point_tables},
    {"vb_bind_gradient_stops", false, scene_with_stops, n_stops, false, " gradient stops (1 .. n_stops)", 20u, true, stops_check, stop_tables},
    {"vb_bind_transforms", false, any_scene, n_xforms, false, " transforms (1 .. n_transforms)", 24u, true, path_tags_outside, transform_tables},
    {"vb_bind_draw_visibility", false, any_scene, n_draws, false, " draw objects (1 .. n_draw_objects)", 1u, false, no_check, visibility_mask},
    {"vb_bind_stroke_widths", false, any_scene, n_draws, false, " draw objects (1 .. n_draw_objects)", 4u, false, draw_tags_check, width_snapshot},
    {"vb_bind_draw_opacity", false, any_scene, n_draws, false, " draw objects (1 .. n_draw_objects)", 4u, true, draw_tags_check, no_tables},
};

// Unbind `kind` in b: its rows and the tables only it reads
static void unbind(VbBound &b, int kind) {
    b.rows[kind] = VbRows{};
    if (kind == VB_BIND_INSTANCES) b.inst_prefix = b.inst_src = b.inst_draw = nullptr, b.inst_xf = nullptr;
    if (kind == VB_BIND_POINTS) b.pt_first = nullptr;
    if (kind == VB_BIND_STOPS) b.rs_grads = nullptr, b.rs_stops = nullptr, b.rs_draw = nullptr, b.rs_grads_n = b.rs_ramp0 = 0u;
    if (kind == VB_BIND_TRANSFORMS) b.xf_range = nullptr;
}

// Bind n rows of `pitch` bytes from `ptr` as `kind` (null: unbind it), for every frame from now on
static int bind_rows(vb_renderer *r, int kind, const void *ptr, uint32_t n, size_t pitch) {
    if (!r) return VB_E_INVALID;
    const BindKind &K = BIND_KINDS[kind];
    auto bad = [&](const std::string &why) {
        r->err = std::string(K.fn) + ": " + why;
        return VB_E_INVALID;
    };
    if (r->grouped || r->xc.enabled || (!K.enabled_only && r->xc.configured))
        return bad(K.enabled_only ? "not available for a renderer of a vb_group or with the exchange enabled"
                                  : "not available for a renderer of a vb_group or with the exchange");
    if (r->frame_pending) return bad("a frame is enqueued and not finished (vb_frame_finish)");
    VbBound nb = r->bound;
    // the draw-data slot table follows them (draw_data_bound)
    const bool draw_data = kind == VB_BIND_COLORS || kind == VB_BIND_STOPS || kind == VB_BIND_OPACITY;
    int rc;
    if (!ptr) {
        const bool was = nb.rows[kind].rows != nullptr;
        unbind(nb, kind);
        if (draw_data && was) {
            CK(cudaSetDevice(r->device));
            if ((rc = draw_data_slots(r, nb))) return rc;
        }
        r->bound = nb;
        r->dmg.epoch++;
        return VB_OK;
    }
    const Slot &slot = *r->cur;
    if (const char *why = K.scene(slot)) return bad(why);
    const uint64_t max = K.rows(slot);
    if (n == 0u || (K.exact ? n != max : n > max))
        return bad(std::to_string(n) + (K.exact ? " rows for a composed scene of " : " rows for a scene of ") + std::to_string(max) + K.unit);
    if (K.min_pitch == 1u) {
        if (pitch == 0u || pitch > 0xffffffffu) return bad("the row pitch must be at least 1 byte and below 4 GiB");
    } else {
        if ((uintptr_t)ptr & 3u) return bad("the pointer must be 4-byte aligned");
        if ((pitch & 3u) || pitch < K.min_pitch || pitch > 0xfffffffcu)
            return bad("the row pitch must be a multiple of 4 bytes, at least " + std::to_string(K.min_pitch) + " and below 4 GiB");
    }
    CK(cudaSetDevice(r->device));
    if (!device_memory_of(r, ptr)) return bad("the rows must be memory of the renderer's device");
    std::string why = K.check(r, n);
    if (!why.empty()) return bad(why);
    nb.rows[kind] = VbRows{(const uint8_t *)ptr, n, (uint32_t)pitch};
    // a frame writes its regions past the scene (regions_of); both transform regions count, since a view can be set later
    if (K.region && regions_of(slot.layout, slot.scene_words, true, true, draw_data_bound(nb), nb.rows[VB_BIND_POINTS].rows != nullptr).words >
                        0xfffffff0ull)
        return bad("the scene with the regions its frames write past it exceeds 32-bit word offsets");
    if ((rc = K.tables(r, n, nb, why))) return why.empty() ? rc : bad(why);
    if (draw_data && (rc = draw_data_slots(r, nb))) return rc;
    r->bound = nb;
    r->dmg.epoch++;
    return VB_OK;
}

extern "C" int vb_bind_instance_transforms(vb_renderer *r, const float *device_transforms, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_INSTANCES, device_transforms, n, row_pitch_bytes);
}
extern "C" int vb_bind_draw_colors(vb_renderer *r, const float *device_rgba, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_COLORS, device_rgba, n, row_pitch_bytes);
}
extern "C" int vb_bind_path_points(vb_renderer *r, const float *device_xy, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_POINTS, device_xy, n, row_pitch_bytes);
}
extern "C" int vb_bind_gradient_stops(vb_renderer *r, const float *device_stops, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_STOPS, device_stops, n, row_pitch_bytes);
}
extern "C" int vb_bind_transforms(vb_renderer *r, const float *device_affines, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_TRANSFORMS, device_affines, n, row_pitch_bytes);
}
extern "C" int vb_bind_draw_visibility(vb_renderer *r, const uint8_t *device_flags, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_VISIBILITY, device_flags, n, row_pitch_bytes);
}
extern "C" int vb_bind_stroke_widths(vb_renderer *r, const float *device_widths, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_WIDTHS, device_widths, n, row_pitch_bytes);
}
extern "C" int vb_bind_draw_opacity(vb_renderer *r, const float *device_alpha, uint32_t n, size_t row_pitch_bytes) {
    return bind_rows(r, VB_BIND_OPACITY, device_alpha, n, row_pitch_bytes);
}
