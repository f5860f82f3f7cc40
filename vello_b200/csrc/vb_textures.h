// vb_textures.h -- the texture registry of vb_upload.cu, as the native scene front end (vb_scene.cpp) uses it.
// Internal to the library, and plain C++: vb_scene.cpp is built without the CUDA headers.
#ifndef VB_TEXTURES_H
#define VB_TEXTURES_H
#include <stddef.h>
#include <stdint.h>

#include "../../include/vello_b200.h"

extern "C" {
// nonzero for an address of the reserved key range, from which vb_texture_register and vb_register_destination take their
// keys (no host buffer has such an address: the host resolve never reads through it)
int vb_texture_key(const void *key);
// Renderer::register_texture / unregister_texture; vb_register_texture / vb_unregister_texture (vb_scene.cpp) wrap them
int vb_texture_register(vb_renderer *r, const void *device_pixels, uint32_t width, uint32_t height, size_t row_pitch_bytes, const void **key_out);
int vb_texture_unregister(vb_renderer *r, const void *key);
}

#endif
