"""Host-side mirror of the reference's renderer interface over libvello_b200.so (ctypes).

Names follow vello/src/lib.rs: `Renderer` (:330-352), `RendererOptions` (:373-420),
`RenderParams` (:357-369), `AaConfig` (:175-193), `Renderer::render_to_texture` (:474-515).
There is NO CPU fallback: if the CUDA library is missing or no device is present this module
raises -- the oracle under oracle/ is test infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np

from .config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from .encoding import Image, Packed, Scene, resolve

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvello_b200.so")

STAGES = ["pathtag", "flatten", "draw", "clip", "binning", "tile_alloc", "path_count", "backdrop", "coarse",
          "path_tiling", "fine"]


class VelloB200Error(RuntimeError):
    pass


class _Options(C.Structure):
    _fields_ = [("device", C.c_int32), ("timing", C.c_uint32), ("max_retries", C.c_uint32), ("reserved", C.c_uint32)]


class _Layout(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "n_draw_objects", "n_paths", "n_clips", "bin_data_start", "path_tag_base", "path_data_base",
        "draw_tag_base", "draw_data_base", "transform_base", "style_base")]


class _Params(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("base_color", "width", "height", "aa", "bin_row0", "bin_row1", "tile_row0", "tile_row1")]


class FrameStats(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("failed", "binning", "ptcl", "tile", "seg_counts", "segments", "blend", "lines",
                                          "retries", "kernel_launches")] + \
               [("stage_ms", C.c_float * len(STAGES)), ("total_ms", C.c_float), ("arena_bytes", C.c_uint64)]

    def as_dict(self):
        d = {n: int(getattr(self, n)) for n in ("failed", "binning", "ptcl", "tile", "seg_counts", "segments", "blend", "lines",
                                                "retries", "kernel_launches", "arena_bytes")}
        d["stage_ms"] = {s: float(self.stage_ms[i]) for i, s in enumerate(STAGES)}
        d["total_ms"] = float(self.total_ms)
        return d


_lib = None


def load_library() -> C.CDLL:
    """Load libvello_b200.so; raise loudly if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("VELLO_B200_LIB", LIB_PATH)  # development knob: A/B a differently tuned build
    if not os.path.exists(path):
        raise VelloB200Error(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                             "(nvcc, sm_90a). vello_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    vp = C.c_void_p
    lib.vb_renderer_new.argtypes = [C.POINTER(_Options), C.POINTER(vp)]
    lib.vb_renderer_free.argtypes = [vp]
    lib.vb_strerror.restype = C.c_char_p
    lib.vb_last_error.restype = C.c_char_p
    lib.vb_last_error.argtypes = [vp]
    lib.vb_scene_upload.argtypes = [vp, vp, C.c_size_t, C.POINTER(_Layout), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.c_uint32]
    lib.vb_render_resident.argtypes = [vp, C.POINTER(_Params), vp, C.POINTER(FrameStats)]
    lib.vb_render_enqueue.argtypes = [vp, C.POINTER(_Params), vp]
    lib.vb_frame_finish.argtypes = [vp, C.POINTER(FrameStats)]
    lib.vb_render.argtypes = [vp, vp, C.c_size_t, C.POINTER(_Layout), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.c_uint32,
                              C.POINTER(_Params), vp, C.c_uint32, C.POINTER(FrameStats)]
    lib.vb_render_begin.argtypes = [vp, vp, C.c_size_t, C.POINTER(_Layout), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.c_uint32,
                                    C.POINTER(_Params), vp, C.POINTER(FrameStats)]
    lib.vb_readback_wait.argtypes = [vp]
    lib.vb_set_readback_bands.argtypes = [vp, C.c_uint32]
    lib.vb_set_cuda_graph.argtypes = [vp, C.c_int]
    lib.vb_set_timing.argtypes = [vp, C.c_int]
    lib.vb_target.restype = vp
    lib.vb_target.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.vb_copy_to_host.argtypes = [vp, vp, vp, C.c_size_t]
    lib.vb_stream.restype = vp
    lib.vb_stream.argtypes = [vp]
    lib.vb_run_stages.argtypes = [vp, C.POINTER(_Params), C.c_int, C.c_int, vp]
    lib.vb_debug_download.argtypes = [vp, C.c_char_p, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.vb_debug_upload.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    lib.vb_debug_limit_arena.argtypes = [vp, C.c_char_p, C.c_uint32]
    lib.vb_set_occlusion_cull.argtypes = [vp, C.c_int]
    lib.vb_debug_fine_traffic.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.vb_last_frame_ms.restype = C.c_float
    lib.vb_last_frame_ms.argtypes = [vp]
    lib.vb_frame_alloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
    lib.vb_frame_free.argtypes = [vp, vp]
    lib.vb_ipc_export.argtypes = [vp, vp, C.c_char_p]
    lib.vb_ipc_open.argtypes = [vp, C.c_char_p, C.POINTER(vp)]
    lib.vb_ipc_close.argtypes = [vp, vp]
    lib.vb_group_new.argtypes = [C.POINTER(C.c_int32), C.c_uint32, C.POINTER(_Options), C.POINTER(vp)]
    lib.vb_group_free.argtypes = [vp]
    lib.vb_group_size.restype = C.c_uint32
    lib.vb_group_size.argtypes = [vp]
    lib.vb_group_renderer.restype = vp
    lib.vb_group_renderer.argtypes = [vp, C.c_uint32]
    lib.vb_group_last_error.restype = C.c_char_p
    lib.vb_group_last_error.argtypes = [vp]
    lib.vb_group_render.argtypes = [vp, vp, C.c_size_t, C.POINTER(_Layout), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.c_uint32,
                                    C.POINTER(_Params), vp, C.c_uint32, vp]
    lib.vb_group_scene_upload.argtypes = [vp, vp, C.c_size_t, C.POINTER(_Layout), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.c_uint32]
    lib.vb_group_render_resident.argtypes = [vp, C.POINTER(_Params), vp, vp]
    lib.vb_group_frame.restype = vp
    lib.vb_group_frame.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.vb_group_stripes.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
    lib.vb_group_set_balancing.argtypes = [vp, C.c_int]
    lib.vb_group_set_exchange.argtypes = [vp, C.c_int]
    lib.vb_exchange_configure.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(vp), C.POINTER(C.c_size_t)]
    lib.vb_exchange_attach.argtypes = [vp, C.c_uint32, vp]
    lib.vb_exchange_set_bounds.argtypes = [vp, C.POINTER(C.c_uint32)]
    lib.vb_exchange_enable.argtypes = [vp, C.c_int]
    lib.vb_override_image.argtypes = [vp, vp, C.c_uint32, C.c_uint32, vp, C.c_size_t]
    lib.vb_mark_override_image_dirty.argtypes = [vp, vp]
    lib.vb_set_cells.argtypes = [vp, vp, C.c_uint32]
    lib.vb_render_uploaded.argtypes = [vp, C.POINTER(_Params), vp, C.c_uint32, C.POINTER(FrameStats)]
    _lib = lib
    return lib


EXPORTED_SYMBOLS = ["vb_renderer_new", "vb_renderer_free", "vb_strerror", "vb_last_error", "vb_scene_upload",
                    "vb_render_resident", "vb_render_enqueue", "vb_frame_finish", "vb_render", "vb_target", "vb_copy_to_host", "vb_stream",
                    "vb_run_stages", "vb_debug_download", "vb_debug_upload", "vb_debug_limit_arena", "vb_debug_fine_traffic", "vb_set_occlusion_cull", "vb_render_begin", "vb_readback_wait", "vb_set_readback_bands", "vb_set_cuda_graph", "vb_set_timing",
                    "vb_scene_upload_streams", "vb_render_uploaded", "vb_last_frame_ms", "vb_frame_alloc", "vb_frame_free", "vb_ipc_export", "vb_ipc_open", "vb_ipc_close",
                    "vb_group_new", "vb_group_free", "vb_group_size", "vb_group_renderer", "vb_group_last_error", "vb_group_render",
                    "vb_group_scene_upload", "vb_group_render_resident", "vb_group_frame", "vb_group_stripes", "vb_group_set_balancing",
                    "vb_group_set_exchange", "vb_exchange_configure", "vb_exchange_attach", "vb_exchange_set_bounds", "vb_exchange_enable",
                    "vb_override_image", "vb_mark_override_image_dirty", "vb_set_cells"]


def _device_image(t):
    """(pointer, height, width, row pitch in bytes) of an (H, W, 4) uint8 array in device memory, from its
    `__cuda_array_interface__` (a torch CUDA tensor, or a slice of one): texels 4 bytes apart, rows any multiple of 4 apart."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{type(t).__name__} has no __cuda_array_interface__: a device image is needed")
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) != 3 or shape[2] != 4 or cai["typestr"] not in ("|u1", "<u1", ">u1"):
        raise ValueError(f"a device image is (H, W, 4) uint8, not shape {shape} of type {cai['typestr']}")
    strides = cai.get("strides") or (shape[1] * 4, 4, 1)
    if tuple(strides[1:]) != (4, 1) or strides[0] % 4:
        raise ValueError(f"a device image has texel strides (4, 1) and a row stride that is a multiple of 4, not {tuple(strides)}")
    return int(cai["data"][0]), shape[0], shape[1], int(strides[0])


@dataclass
class RendererOptions:
    """vello::RendererOptions restricted to what applies (lib.rs:373-420): there is no `use_cpu`."""
    device: int = 0
    timing: bool = False
    max_retries: int = 6


def _params_struct(p: RenderParams, bin_rows=(0, 0), tile_rows=(0, 0)) -> _Params:
    return _Params(p.base_color.premul_rgba8_u32(), int(p.width), int(p.height), int(p.antialiasing_method),
                   int(bin_rows[0]), int(bin_rows[1]), int(tile_rows[0]), int(tile_rows[1]))


class Renderer:
    """`vello::Renderer`: `Renderer(options)`, then `render_to_texture(scene, params)`."""

    def __init__(self, options: Optional[RendererOptions] = None):
        self.lib = load_library()
        options = options or RendererOptions()
        self.handle = C.c_void_p()
        opt = _Options(options.device, 1 if options.timing else 0, options.max_retries, 0)
        rc = self.lib.vb_renderer_new(C.byref(opt), C.byref(self.handle))
        if rc != 0:
            raise VelloB200Error(f"vb_renderer_new failed: {self.lib.vb_strerror(rc).decode()} "
                                 "(a CUDA device is required; there is no CPU fallback)")
        self.options = options
        self.last_stats: Optional[FrameStats] = None
        self._keep = None
        self._owner = None
        self._device_images = {}  # key -> the device array an override of this renderer reads (kept alive while in use)

    @classmethod
    def _borrowed(cls, lib, handle: int, owner):
        """A view of a renderer owned by someone else (a RendererGroup): closing it frees nothing."""
        r = cls.__new__(cls)
        r.lib, r.handle, r.options, r.last_stats, r._keep = lib, C.c_void_p(handle), None, None, None
        r._owner = owner
        r._device_images = {}
        return r

    def close(self):
        if getattr(self, "_owner", None) is None and getattr(self, "handle", None) and self.handle.value:
            self.lib.vb_renderer_free(self.handle)
        self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise VelloB200Error(f"{what}: {self.lib.vb_strerror(rc).decode()} [{self.lib.vb_last_error(self.handle).decode()}]")

    # -- scene -----------------------------------------------------------------------------------
    def upload(self, packed: Packed):
        scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
        ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
        atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
        lay = _Layout(*[int(v) for v in packed.layout.as_array()])
        self._keep = (scene, ramps, atlas)
        rc = self.lib.vb_scene_upload(self.handle, scene.ctypes.data, scene.nbytes, C.byref(lay),
                                      ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                      atlas.ctypes.data, atlas.shape[1], atlas.shape[0])
        self._check(rc, "vb_scene_upload")

    # -- images from device memory (Renderer::override_image / register_texture, vello/src/lib.rs:536-603) ---------------------
    # Overrides apply where the scene is resolved on the device (NativeScene.upload_device); a host-packed scene (upload,
    # render_to_texture, render_stream) ignores them. The caller orders its writes to a device array before the call that
    # copies it (a torch.cuda.synchronize(), or work on `self.stream`).
    def register_texture(self, t) -> Image:
        """Draw the device array `t` ((H, W, 4) uint8, RGBA8 with straight alpha; e.g. a torch CUDA tensor or a column slice
        of one) as an `Image`: a fresh key with an override of `t`. `t` is held until `unregister_texture`. The image's
        sampler fields (quality, extends, alpha, format, alpha_type) are the caller's to change."""
        from .scene_native import _Image, _lib as _scene_lib
        ptr, h, w, pitch = _device_image(t)
        im = _Image()
        self._check(_scene_lib().vb_register_texture(self.handle, C.c_void_p(ptr), w, h, pitch, C.byref(im)), "vb_register_texture")
        self._device_images[int(im.pixels)] = t
        zeros = np.lib.stride_tricks.as_strided(np.zeros(4, dtype=np.uint8), shape=(h, w, 4), strides=(0, 0, 1))
        return Image(zeros, key=int(im.pixels))

    def unregister_texture(self, image: Image):
        from .scene_native import _Image, _lib as _scene_lib
        im = _Image(C.c_void_p(image.key) if image.key is not None else None, image.width, image.height)
        self._check(_scene_lib().vb_unregister_texture(self.handle, C.byref(im)), "vb_unregister_texture")
        self._device_images.pop(image.key, None)

    def override_image(self, image: Image, t=None):
        """Supply the pixels of `image` from the device array `t` at the next device resolve and the frames after it
        (`mark_override_image_dirty` to copy them again); `t=None` removes the override. A host image without a key gets one
        here: its data becomes a private contiguous copy whose address is the key."""
        if t is None:
            if image.key is not None:
                self._check(self.lib.vb_override_image(self.handle, C.c_void_p(image.key), 0, 0, None, 0), "vb_override_image")
                self._device_images.pop(image.key, None)
            return
        ptr, h, w, pitch = _device_image(t)
        if image.key is None:
            image.data = np.ascontiguousarray(image.data, dtype=np.uint8).copy()
            image.key = int(image.data.ctypes.data)
        self._check(self.lib.vb_override_image(self.handle, C.c_void_p(image.key), w, h, C.c_void_p(ptr), pitch), "vb_override_image")
        self._device_images[image.key] = t

    def mark_override_image_dirty(self, image: Image):
        """Copy the overridden image's device pixels into the atlas again, in front of the next frame."""
        if image.key is None:
            raise ValueError("mark_override_image_dirty: the image has no override")
        self._check(self.lib.vb_mark_override_image_dirty(self.handle, C.c_void_p(image.key)), "vb_mark_override_image_dirty")

    # -- rendering ---------------------------------------------------------------------------------
    def render_to_texture(self, scene, params: RenderParams, bin_rows=(0, 0), tile_rows=(0, 0)) -> np.ndarray:
        """Render `scene` (a `Scene`, or an already resolved `Packed`) and return the RGBA8 image
        (h, w, 4) -- un-premultiplied, like the reference's Rgba8Unorm storage texture. Goes through
        the one-call C entry point `vb_render` with host buffers (upload + render + readback)."""
        packed = scene if isinstance(scene, Packed) else resolve(scene.encoding)
        scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
        ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
        atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
        lay = _Layout(*[int(v) for v in packed.layout.as_array()])
        ps = _params_struct(params, bin_rows, tile_rows)
        h0, h1 = self.stripe_rows(params, bin_rows, tile_rows)
        out = np.zeros((h1 - h0, params.width, 4), dtype=np.uint8)
        st = FrameStats()
        rc = self.lib.vb_render(self.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay),
                                ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), out.ctypes.data, 0, C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_render")
        return out

    def render_stream(self, scenes, params: RenderParams):
        """Render a sequence of scenes through the streaming entry points (vb_render_begin / vb_readback_wait): a generator
        of RGBA8 images, each complete when yielded. Three frames are in flight (upload | rasterise | read back), so frame k-2
        is yielded after frame k has been submitted."""
        outs = []
        for k, scene in enumerate(scenes):
            packed = scene if isinstance(scene, Packed) else resolve(scene.encoding)
            scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
            ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
            atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
            lay = _Layout(*[int(v) for v in packed.layout.as_array()])
            ps = _params_struct(params, (0, 0))
            out = np.zeros((params.height, params.width, 4), dtype=np.uint8)
            outs.append(out)
            st = FrameStats()
            rc = self.lib.vb_render_begin(self.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay),
                                          ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                          atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), out.ctypes.data, C.byref(st))
            self.last_stats = st
            self._check(rc, "vb_render_begin")
            if k >= 2:
                yield outs[k - 2]  # complete: vb_render_begin returned for the frame two later
                outs[k - 2] = None
        if outs:
            self._check(self.lib.vb_readback_wait(self.handle), "vb_readback_wait")
            for o in outs[-2:]:
                if o is not None:
                    yield o

    # -- batches: many scenes of one size in one pass (vb_set_cells) ---------------------------------------------------------
    def set_cells(self, offsets):
        """Split the uploaded scene's draw objects into cells (`offsets`: len = cells + 1, from `encoding.batch` or
        `NativeScene.batch`): the following frames render cell c into frame c of an [N, H, W, 4] destination. A new upload
        resets the renderer to one cell."""
        arr = np.ascontiguousarray(offsets, dtype=np.uint32)
        if arr.ndim != 1 or arr.size < 2:
            raise ValueError("set_cells: offsets need at least two entries (cells + 1)")
        self._check(self.lib.vb_set_cells(self.handle, arr.ctypes.data, arr.size - 1), "vb_set_cells")

    def render_batch(self, scenes, params: RenderParams, out=None):
        """Render every scene of `scenes` (all `Scene`s, or all `NativeScene`s, which are resolved on the device) at
        params.width x params.height in ONE pass and return the [N, H, W, 4] RGBA8 frames: into `out` when it is a CUDA array
        of that shape (`__cuda_array_interface__`, e.g. a torch uint8 tensor), else a new numpy array."""
        from .encoding import batch
        from .scene_native import NativeScene
        scenes = list(scenes)
        n, h, w = len(scenes), int(params.height), int(params.width)
        if n == 0:
            raise ValueError("render_batch: no scenes")
        if all(isinstance(s, NativeScene) for s in scenes):
            b = NativeScene()
            offsets = b.batch(scenes)
            b.upload_device(self)
        else:
            bs, offsets = batch(scenes)
            self.upload(resolve(bs.encoding))
        self.set_cells(offsets)
        ps = _params_struct(params)
        st = FrameStats()
        if out is not None and hasattr(out, "__cuda_array_interface__"):
            cai = out.__cuda_array_interface__
            shape = tuple(int(v) for v in cai["shape"])
            if shape != (n, h, w, 4) or cai["typestr"] not in ("|u1", "<u1", ">u1") or cai.get("strides") not in (None, (h * w * 4, w * 4, 4, 1)):
                raise ValueError(f"render_batch: out must be a contiguous uint8 ({n}, {h}, {w}, 4) array, not {shape} {cai['typestr']}")
            rc = self.lib.vb_render_uploaded(self.handle, C.byref(ps), C.c_void_p(int(cai["data"][0])), 1, C.byref(st))
        else:
            out = np.zeros((n, h, w, 4), dtype=np.uint8)
            rc = self.lib.vb_render_uploaded(self.handle, C.byref(ps), C.c_void_p(out.ctypes.data), 0, C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_render_uploaded")
        return out

    @staticmethod
    def stripe_rows(params: RenderParams, bin_rows=(0, 0), tile_rows=(0, 0)):
        if tile_rows[1] > tile_rows[0]:
            return min(tile_rows[0] * 16, params.height), min(tile_rows[1] * 16, params.height)
        if bin_rows[1] > bin_rows[0]:
            return min(bin_rows[0] * 256, params.height), min(bin_rows[1] * 256, params.height)
        return 0, params.height

    def render_resident(self, params: RenderParams, out_device_ptr: int = 0, bin_rows=(0, 0), tile_rows=(0, 0)) -> FrameStats:
        """Render the uploaded scene into a device buffer (0 = the renderer's own target)."""
        ps = _params_struct(params, bin_rows, tile_rows)
        st = FrameStats()
        rc = self.lib.vb_render_resident(self.handle, C.byref(ps), C.c_void_p(out_device_ptr or None), C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_render_resident")
        return st

    def enqueue(self, params: RenderParams, out_device_ptr: int = 0, bin_rows=(0, 0), tile_rows=(0, 0)):
        ps = _params_struct(params, bin_rows, tile_rows)
        self._check(self.lib.vb_render_enqueue(self.handle, C.byref(ps), C.c_void_p(out_device_ptr or None)), "vb_render_enqueue")

    def finish(self) -> FrameStats:
        st = FrameStats()
        rc = self.lib.vb_frame_finish(self.handle, C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_frame_finish")
        return st

    @property
    def stream(self) -> int:
        return int(self.lib.vb_stream(self.handle) or 0)

    def target_ptr(self) -> int:
        n = C.c_size_t(0)
        return int(self.lib.vb_target(self.handle, C.byref(n)) or 0)

    # -- stage-level access (parity tests) -----------------------------------------------------------
    def run_stages(self, params: RenderParams, first: str, last: str, out_device_ptr: int = 0, bin_rows=(0, 0)):
        ps = _params_struct(params, bin_rows)
        rc = self.lib.vb_run_stages(self.handle, C.byref(ps), STAGES.index(first), STAGES.index(last), C.c_void_p(out_device_ptr or None))
        self._check(rc, "vb_run_stages")

    def download(self, name: str, dtype) -> np.ndarray:
        n = C.c_size_t(0)
        self._check(self.lib.vb_debug_download(self.handle, name.encode(), None, 0, C.byref(n)), f"download {name}")
        buf = np.zeros(n.value, dtype=np.uint8)
        if n.value:
            self._check(self.lib.vb_debug_download(self.handle, name.encode(), buf.ctypes.data, n.value, C.byref(n)), f"download {name}")
        return buf.view(dtype)

    def upload_buffer(self, name: str, arr: np.ndarray):
        a = np.ascontiguousarray(arr)
        self._check(self.lib.vb_debug_upload(self.handle, name.encode(), a.ctypes.data, a.nbytes), f"upload {name}")

    # the guard byte vb_debug_limit_arena writes past a limited arena's limit (VB_GUARD_BYTE)
    GUARD_BYTE = 0xA5
    NO_LIMIT = 0xFFFFFFFF

    def limit_arena(self, name: str, limit: int):
        """Test-only: the kernels see at most `limit` of arena `name` ("lines", "binning", "tiles", "seg_counts", "segments",
        "blend", "ptcl"; ptcl in words of the whole arena) until an attempt overflows it. `NO_LIMIT` clears it. The bytes of
        the allocation past the limit are filled with GUARD_BYTE (see download_guard)."""
        self._check(self.lib.vb_debug_limit_arena(self.handle, name.encode(), int(limit)), f"vb_debug_limit_arena {name}")

    def download_guard(self, name: str) -> np.ndarray:
        """The guard region past a limited arena's limit as bytes ("lines", ..., "ptcl", "line_scratch", "flatten_jobs")."""
        return self.download(f"{name}.guard", np.uint8)

    def set_cuda_graph(self, on: bool):
        """Replay whole frames as CUDA graphs (default on)."""
        self._check(self.lib.vb_set_cuda_graph(self.handle, 1 if on else 0), "vb_set_cuda_graph")

    def set_occlusion_cull(self, on: bool):
        """fine skips the commands under a tile's last opaque full-tile cover (identical pixels). Default on."""
        self._check(self.lib.vb_set_occlusion_cull(self.handle, 1 if on else 0), "vb_set_occlusion_cull")

    def fine_traffic(self):
        """(ptcl_words, segment_refs, fill_cmds) of the last frame -- inputs of the fine roofline."""
        a, b, c = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.vb_debug_fine_traffic(self.handle, C.byref(a), C.byref(b), C.byref(c)), "vb_debug_fine_traffic")
        return int(a.value), int(b.value), int(c.value)

    def download_target(self, params: RenderParams, bin_rows=(0, 0), device_ptr: int = 0, tile_rows=(0, 0)) -> np.ndarray:
        """Copy the last frame's target (or `device_ptr`) to the host."""
        h0, h1 = self.stripe_rows(params, bin_rows, tile_rows)
        out = np.zeros((h1 - h0, params.width, 4), dtype=np.uint8)
        src = device_ptr or self.target_ptr()
        self._check(self.lib.vb_copy_to_host(self.handle, C.c_void_p(src), C.c_void_p(out.ctypes.data), C.c_size_t(out.nbytes)),
                    "vb_copy_to_host")
        return out


class RendererGroup:
    """One frame on several GPUs of one box from one process (`vb_group`): the frame is cut into cost-balanced stripes of tile
    rows, every device renders one, and `fine` on device k stores its pixels straight into the frame on devices[0] over
    NVLink peer mapping (or every device reads its stripe back over its own PCIe link for a host destination)."""

    def __init__(self, devices, options: Optional[RendererOptions] = None):
        self.lib = load_library()
        options = options or RendererOptions()
        self.devices = [int(d) for d in devices]
        arr = (C.c_int32 * len(self.devices))(*self.devices)
        opt = _Options(self.devices[0], 1 if options.timing else 0, options.max_retries, 0)
        self.handle = C.c_void_p()
        rc = self.lib.vb_group_new(arr, len(self.devices), C.byref(opt), C.byref(self.handle))
        if rc != 0:
            raise VelloB200Error(f"vb_group_new failed: {self.lib.vb_strerror(rc).decode()}")
        self.last_stats = None

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.vb_group_free(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise VelloB200Error(f"{what}: {self.lib.vb_strerror(rc).decode()} [{self.lib.vb_group_last_error(self.handle).decode()}]")

    def renderer(self, i: int) -> Renderer:
        """The i-th device's renderer (statistics, debugging); it belongs to the group and lives as long as the group."""
        h = self.lib.vb_group_renderer(self.handle, int(i))
        if not h:
            raise VelloB200Error(f"vb_group_renderer: no renderer {i}")
        return Renderer._borrowed(self.lib, h, self)

    def set_balancing(self, on: bool):
        self._check(self.lib.vb_group_set_balancing(self.handle, 1 if on else 0), "vb_group_set_balancing")

    def set_exchange(self, on: bool):
        """Shard `flatten` by tag range across the devices and exchange lines / path boxes through peer memory
        (k_exchange.cu) instead of flattening the whole scene on every device."""
        self._check(self.lib.vb_group_set_exchange(self.handle, 1 if on else 0), "vb_group_set_exchange")

    def upload(self, packed: Packed):
        scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
        ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
        atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
        lay = _Layout(*[int(v) for v in packed.layout.as_array()])
        self._keep = (scene, ramps, atlas)
        self._check(self.lib.vb_group_scene_upload(self.handle, scene.ctypes.data, scene.nbytes, C.byref(lay),
                                                   ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                                   atlas.ctypes.data, atlas.shape[1], atlas.shape[0]), "vb_group_scene_upload")

    def render_resident(self, params: RenderParams, out_device_ptr: int = 0):
        ps = _params_struct(params)
        st = (FrameStats * len(self.devices))()
        self._check(self.lib.vb_group_render_resident(self.handle, C.byref(ps), C.c_void_p(out_device_ptr or None), st), "vb_group_render_resident")
        self.last_stats = list(st)
        return self.last_stats

    def render_to_texture(self, scene, params: RenderParams) -> np.ndarray:
        """ONE call, ONE frame: upload to every device, render the stripes, assemble in the caller's host buffer."""
        packed = scene if isinstance(scene, Packed) else resolve(scene.encoding)
        scene_w = np.ascontiguousarray(packed.scene, dtype=np.uint32)
        ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
        atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
        lay = _Layout(*[int(v) for v in packed.layout.as_array()])
        ps = _params_struct(params)
        out = np.zeros((params.height, params.width, 4), dtype=np.uint8)
        st = (FrameStats * len(self.devices))()
        rc = self.lib.vb_group_render(self.handle, scene_w.ctypes.data, scene_w.nbytes, C.byref(lay),
                                      ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                      atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(ps), out.ctypes.data, 0, st)
        self.last_stats = list(st)
        self._check(rc, "vb_group_render")
        return out

    def frame_to_host(self, params: RenderParams) -> np.ndarray:
        """Copy the group's assembled frame (on devices[0]) to the host."""
        n = C.c_size_t(0)
        ptr = self.lib.vb_group_frame(self.handle, C.byref(n))
        out = np.zeros((params.height, params.width, 4), dtype=np.uint8)
        r0 = self.lib.vb_group_renderer(self.handle, 0)
        rc = self.lib.vb_copy_to_host(r0, C.c_void_p(ptr), C.c_void_p(out.ctypes.data), C.c_size_t(out.nbytes))
        self._check(rc, "vb_copy_to_host")
        return out

    def stripes(self):
        n = len(self.devices)
        b = (C.c_uint32 * (n + 1))()
        ms = (C.c_float * n)()
        self._check(self.lib.vb_group_stripes(self.handle, b, ms), "vb_group_stripes")
        return list(b), list(ms)
