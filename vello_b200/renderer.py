"""Host-side mirror of the reference's renderer interface over libvello_b200.so (ctypes).

Names follow vello/src/lib.rs: `Renderer` (:330-352), `RendererOptions` (:373-420),
`RenderParams` (:357-369), `AaConfig` (:175-193), `Renderer::render_to_texture` (:474-515).
There is NO CPU fallback: if the CUDA library is missing or no device is present this module
raises -- the oracle under oracle/ is test infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref
from dataclasses import dataclass
from typing import Optional

import numpy as np

from .config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from .encoding import Image, Packed, Scene, resolve
from .shapes import Affine

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


class _RampStop(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("offset", "r", "g", "b", "a")]


class _RampPatch(C.Structure):
    _fields_ = [("draw_data_offset", C.c_uint32), ("extend", C.c_uint32), ("premul_interp", C.c_uint32), ("n_stops", C.c_uint32),
                ("stops", C.c_void_p)]


class _ImagePatch(C.Structure):
    _fields_ = [("draw_data_offset", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32), ("pixels", C.c_void_p)]


class _EncodingStreams(C.Structure):
    _fields_ = [("path_tags", C.c_void_p), ("n_path_tags", C.c_uint32), ("path_data", C.c_void_p), ("n_path_data", C.c_uint32),
                ("draw_tags", C.c_void_p), ("n_draw_tags", C.c_uint32), ("draw_data", C.c_void_p), ("n_draw_data", C.c_uint32),
                ("transforms", C.c_void_p), ("n_transforms", C.c_uint32), ("styles", C.c_void_p), ("n_styles", C.c_uint32),
                ("n_paths", C.c_uint32), ("n_clips", C.c_uint32), ("n_open_clips", C.c_uint32),
                ("ramp_patches", C.c_void_p), ("n_ramp_patches", C.c_uint32), ("image_patches", C.c_void_p), ("n_image_patches", C.c_uint32)]


class _DevicePaths(C.Structure):
    _fields_ = [("points", C.c_void_p), ("n_points", C.c_uint32), ("point_pitch_bytes", C.c_size_t),
                ("ring_offsets", C.c_void_p), ("n_rings", C.c_uint32), ("path_offsets", C.c_void_p), ("n_paths", C.c_uint32),
                ("colors", C.c_void_p), ("color_pitch_bytes", C.c_size_t), ("kind", C.c_uint32), ("fill_rule", C.c_uint32),
                ("width", C.c_float), ("miter_limit", C.c_float), ("join", C.c_uint32), ("start_cap", C.c_uint32),
                ("end_cap", C.c_uint32), ("closed", C.c_uint32), ("draw_index", C.c_void_p)]


class _Dash(C.Structure):
    _fields_ = [("pattern", C.c_void_p), ("n_pattern", C.c_uint32), ("offset", C.c_double), ("offsets", C.c_void_p),
                ("offset_pitch_bytes", C.c_size_t)]


class _Instance(C.Structure):
    _fields_ = [("fragment", C.c_uint32), ("has_transform", C.c_uint32), ("transform", C.c_double * 6)]


class _Destination(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("format", C.c_uint32), ("ptr", C.c_void_p), ("row_pitch_bytes", C.c_size_t),
                ("array", C.c_void_p), ("x", C.c_uint32), ("y", C.c_uint32)]


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
    lib.vb_debug_lookback.argtypes = [vp, C.c_int, C.c_uint32, vp, vp, vp]
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
    lib.vb_set_view.argtypes = [vp, C.POINTER(C.c_double)]
    lib.vb_group_set_view.argtypes = [vp, C.POINTER(C.c_double)]
    lib.vb_debug_graph_captures.argtypes = [vp, C.POINTER(C.c_uint64)]
    lib.vb_hit_test.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32]
    lib.vb_hit_map.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, C.c_size_t, C.c_uint32]
    lib.vb_fragment_upload.argtypes = [vp, C.POINTER(_EncodingStreams), C.POINTER(C.c_uint32)]
    lib.vb_fragment_free.argtypes = [vp, C.c_uint32]
    lib.vb_fragment_from_device_paths.argtypes = [vp, C.POINTER(_DevicePaths), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    lib.vb_fragment_from_device_curves.argtypes = [vp, C.POINTER(_DevicePaths), vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    lib.vb_fragment_from_device_dashes.argtypes = [vp, C.POINTER(_DevicePaths), vp, C.POINTER(_Dash), C.POINTER(C.c_uint32),
                                                   C.POINTER(C.c_uint32)]
    lib.vb_compose.argtypes = [vp, vp, C.c_uint32, C.POINTER(_Layout), vp]
    lib.vb_recompose.argtypes = [vp, vp, C.c_uint32, C.POINTER(_Layout), vp]
    lib.vb_debug_match_instances.argtypes = [vp, C.c_uint32, vp, C.c_uint32, vp]
    lib.vb_debug_match_instances.restype = C.c_uint32
    lib.vb_bind_instance_transforms.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_draw_colors.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_path_points.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_gradient_stops.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_transforms.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_draw_visibility.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_stroke_widths.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_bind_draw_opacity.argtypes = [vp, vp, C.c_uint32, C.c_size_t]
    lib.vb_set_damage_tracking.argtypes = [vp, C.c_int]
    lib.vb_set_upload_diff.argtypes = [vp, C.c_int]
    lib.vb_add_damage.argtypes = [vp, vp, C.c_uint32]
    lib.vb_last_damage.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_uint32)]
    lib.vb_register_destination.argtypes = [vp, C.POINTER(_Destination), C.POINTER(vp)]
    lib.vb_unregister_destination.argtypes = [vp, vp]
    lib.vb_set_background.argtypes = [vp, C.POINTER(_Destination)]
    _lib = lib
    return lib


EXPORTED_SYMBOLS = ["vb_renderer_new", "vb_renderer_free", "vb_strerror", "vb_last_error", "vb_scene_upload",
                    "vb_render_resident", "vb_render_enqueue", "vb_frame_finish", "vb_render", "vb_target", "vb_copy_to_host", "vb_stream",
                    "vb_run_stages", "vb_debug_download", "vb_debug_upload", "vb_debug_limit_arena", "vb_debug_fine_traffic", "vb_debug_lookback", "vb_set_occlusion_cull", "vb_render_begin", "vb_readback_wait", "vb_set_readback_bands", "vb_set_cuda_graph", "vb_set_timing",
                    "vb_scene_upload_streams", "vb_render_uploaded", "vb_last_frame_ms", "vb_frame_alloc", "vb_frame_free", "vb_ipc_export", "vb_ipc_open", "vb_ipc_close",
                    "vb_group_new", "vb_group_free", "vb_group_size", "vb_group_renderer", "vb_group_last_error", "vb_group_render",
                    "vb_group_scene_upload", "vb_group_render_resident", "vb_group_frame", "vb_group_stripes", "vb_group_set_balancing",
                    "vb_group_set_exchange", "vb_exchange_configure", "vb_exchange_attach", "vb_exchange_set_bounds", "vb_exchange_enable",
                    "vb_override_image", "vb_mark_override_image_dirty", "vb_set_cells", "vb_set_view", "vb_group_set_view",
                    "vb_debug_graph_captures", "vb_hit_test", "vb_hit_map", "vb_fragment_upload", "vb_fragment_free", "vb_compose",
                    "vb_bind_instance_transforms", "vb_set_damage_tracking", "vb_add_damage", "vb_last_damage",
                    "vb_recompose", "vb_set_upload_diff", "vb_register_destination", "vb_unregister_destination",
                    "vb_bind_draw_colors", "vb_bind_path_points", "vb_bind_gradient_stops", "vb_bind_transforms",
                    "vb_set_background", "vb_bind_draw_visibility", "vb_bind_stroke_widths", "vb_bind_draw_opacity",
                    "vb_fragment_from_device_paths", "vb_fragment_from_device_curves",
                    "vb_fragment_from_device_dashes"]


def _device_rows(t, who: str, what: str, cols: int, vector: bool = False, empty: bool = False):
    """(pointer, rows, row pitch in bytes) of an (n, cols) float32 device array bound by a `bind_*` method, from its
    `__cuda_array_interface__` (a torch CUDA tensor, or columns of a larger one): columns 4 bytes apart and rows any multiple of
    4 bytes, at least 4 * cols, apart. With `vector` (cols = 1) an (n,) array is taken as (n, 1), so a column of a larger
    tensor such as `state[:, 5]` binds with its row stride. With `empty`, n = 0 is taken (a null pointer and the least pitch).
    `who` names the method and `what` the rows in the errors."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{type(t).__name__} has no __cuda_array_interface__: device {what} are needed")
    shape = tuple(int(v) for v in cai["shape"])
    strides = cai.get("strides")
    rows = shape
    if vector and len(shape) == 1:
        rows, strides = shape + (1,), strides and (strides[0], 4)
    if len(rows) != 2 or (rows[0] == 0 and not empty) or rows[1] != cols or cai["typestr"] != "<f4":
        form = f"(n,) or (n, {cols})" if vector else f"(n, {cols})"
        raise ValueError(f"{who}: {what} must be {form} float32, not {shape} {cai['typestr']}")
    if rows[0] == 0:
        return None, 0, 4 * cols
    shape = rows
    strides = strides or (4 * cols, 4)
    pitch = int(strides[0]) if shape[0] > 1 else 4 * cols  # the pitch of a single row is never used
    if int(strides[1]) != 4 or pitch % 4 or pitch < 4 * cols:
        raise ValueError(f"{who}: columns 4 bytes apart and rows a multiple of 4 bytes, at least {4 * cols}, apart; "
                         f"not strides {tuple(strides)}")
    return C.c_void_p(int(cai["data"][0])), shape[0], pitch


def _device_offsets(t, who: str, what: str, dtype: str = "<i4"):
    """(pointer, entries) of a contiguous 1-D int32 device array, from its `__cuda_array_interface__`. int64 offsets (torch's
    default integer type) are refused with the conversion to make. `who` names the method and `what` the array in the errors."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{who}: {type(t).__name__} has no __cuda_array_interface__: device {what} are needed")
    shape = tuple(int(v) for v in cai["shape"])
    if cai["typestr"] == "<i8" and dtype == "<i4":
        raise ValueError(f"{who}: {what} are int64; convert them to int32 (e.g. `t.to(torch.int32)`)")
    if len(shape) != 1 or cai["typestr"] != dtype:
        raise ValueError(f"{who}: {what} must be a 1-D int32 array, not {shape} {cai['typestr']}")
    strides = cai.get("strides")
    if strides is not None and shape[0] > 1 and tuple(strides) != (4,):
        raise ValueError(f"{who}: {what} must be contiguous, not strides {tuple(strides)}")
    return (C.c_void_p(int(cai["data"][0])) if shape[0] else None), shape[0]


def _device_flags(t, who: str):
    """(pointer, rows, row pitch in bytes) of a 1-D bool or uint8 device array bound by a `bind_*` method, from its
    `__cuda_array_interface__` (a torch CUDA tensor, or a column of a larger uint8 one): one byte per row, rows any positive
    number of bytes apart. `who` names the method in the errors."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{type(t).__name__} has no __cuda_array_interface__: device flags are needed")
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) != 1 or shape[0] == 0 or cai["typestr"] not in ("|b1", "|u1", "<u1", ">u1"):
        raise ValueError(f"{who}: flags must be (n,) bool or uint8, not {shape} {cai['typestr']}")
    strides = cai.get("strides") or (1,)
    pitch = int(strides[0]) if shape[0] > 1 else 1  # the pitch of a single row is never used
    if pitch <= 0:
        raise ValueError(f"{who}: rows a positive number of bytes apart, not strides {tuple(strides)}")
    return C.c_void_p(int(cai["data"][0])), shape[0], pitch


def _device_kinds(t, n_points: int, who: str):
    """The pointer of `point_kinds`: a contiguous 1-D uint8 or bool device array of `n_points` entries, from its
    `__cuda_array_interface__` (0 on-curve, 1 off-curve; True is 1)."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{who}: {type(t).__name__} has no __cuda_array_interface__: device point_kinds are needed")
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) != 1 or cai["typestr"] not in ("|b1", "|u1", "<u1", ">u1"):
        raise ValueError(f"{who}: point_kinds must be a 1-D uint8 or bool array, not {shape} {cai['typestr']}")
    if shape[0] != n_points:
        raise ValueError(f"{who}: point_kinds has {shape[0]} entries for {n_points} points")
    strides = cai.get("strides")
    if strides is not None and shape[0] > 1 and tuple(strides) != (1,):
        raise ValueError(f"{who}: point_kinds must be contiguous, not strides {tuple(strides)}")
    return C.c_void_p(int(cai["data"][0])) if shape[0] else None


def _device_image(t, typestr="|u1"):
    """(pointer, height, width, row pitch in bytes) of an (H, W, 4) device array of element type `typestr` ("|u1" uint8,
    "<f2" float16 or "<f4" float32), from its `__cuda_array_interface__` (a torch CUDA tensor, or a slice of one): elements
    e bytes apart, texels 4e bytes apart, rows any multiple of 4e apart. Device images (uint8) and linear destinations
    (`Renderer.register_destination`) are read this way."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{type(t).__name__} has no __cuda_array_interface__: a device image is needed")
    shape = tuple(int(v) for v in cai["shape"])
    same = ("|u1", "<u1", ">u1") if typestr == "|u1" else (typestr,)
    if len(shape) != 3 or shape[2] != 4 or cai["typestr"] not in same:
        name = {"|u1": "uint8", "<f2": "float16", "<f4": "float32"}[typestr]
        raise ValueError(f"a device image is (H, W, 4) {name}, not shape {shape} of type {cai['typestr']}")
    e = int(typestr[2:])
    strides = cai.get("strides") or (shape[1] * 4 * e, 4 * e, e)
    if tuple(strides[1:]) != (4 * e, e) or strides[0] % (4 * e):
        raise ValueError(f"a device image has texel strides ({4 * e}, {e}) and a row stride that is a multiple of {4 * e}, "
                         f"not {tuple(strides)}")
    return int(cai["data"][0]), shape[0], shape[1], int(strides[0])


def _background_image(t, typestr):
    """(pointer, row pitch in bytes) of a background (`Renderer.set_background`): an (H, W, 4) device array as `_device_image`
    reads it, or an (N, H, W, 4) one whose cells are H row pitches apart."""
    cai = getattr(t, "__cuda_array_interface__", None)
    if cai is None or len(cai["shape"]) != 4:
        ptr, _, _, pitch = _device_image(t, typestr)
        return ptr, pitch
    shape = tuple(int(v) for v in cai["shape"])
    e = int(typestr[2:])
    strides = tuple(int(v) for v in (cai.get("strides") or (shape[1] * shape[2] * 4 * e, shape[2] * 4 * e, 4 * e, e)))

    class _Cell:
        __cuda_array_interface__ = dict(cai, shape=shape[1:], strides=strides[1:])
    ptr, h, _, pitch = _device_image(_Cell(), typestr)
    if shape[0] > 1 and strides[0] != h * pitch:
        raise ValueError(f"set_background: the cells of an (N, H, W, 4) background are H row pitches ({h * pitch} bytes) apart, "
                         f"not {strides[0]}")
    return ptr, pitch


def _device_vector(t, width, typestrs, what):
    """(pointer, rows) of a contiguous (rows, width) -- or (rows,) for width 1 -- device array from its
    `__cuda_array_interface__`."""
    cai = t.__cuda_array_interface__
    shape = tuple(int(v) for v in cai["shape"])
    want = 2 if width > 1 else 1
    if len(shape) != want or (width > 1 and shape[1] != width) or cai["typestr"] not in typestrs:
        raise ValueError(f"hit_test: {what} must be {'(n, %d)' % width if width > 1 else '(n,)'} {typestrs[0]}, "
                         f"not {shape} {cai['typestr']}")
    item = int(cai["typestr"][2:])
    strides = cai.get("strides")
    if strides is not None and tuple(strides) != ((width * item, item) if width > 1 else (item,)) and shape[0] > 1:
        raise ValueError(f"hit_test: {what} must be contiguous, not strides {tuple(strides)}")
    return int(cai["data"][0]), shape[0]


@dataclass
class RendererOptions:
    """vello::RendererOptions restricted to what applies (lib.rs:373-420): there is no `use_cpu`."""
    device: int = 0
    timing: bool = False
    max_retries: int = 6


def _view_coeffs(affine: Optional[Affine]):
    """The kurbo Affine coefficients [a b c d e f] as vb_set_view takes them (None: clear the view)."""
    return None if affine is None else (C.c_double * 6)(*[float(v) for v in affine.coeffs])


def _encoding_streams(enc, key_of):
    """`enc` (an `encoding.Encoding`) as vb_encoding_streams, and the arrays it points into (keep them alive for the call).
    key_of(image) gives the pointer an image is keyed and read by."""
    from .encoding import _f32_bits, _path_data_array
    tags = np.asarray(enc.path_tags, dtype=np.uint8)
    pd = _path_data_array(enc.path_data).view(np.uint32)
    dtags = np.asarray(enc.draw_tags, dtype=np.uint32)
    ddata = np.asarray(enc.draw_data, dtype=np.uint32)
    tr = np.asarray(enc.transforms, dtype=np.float32).reshape(-1)
    st = np.zeros(2 * len(enc.styles), dtype=np.uint32)
    for i, (fl, lw) in enumerate(enc.styles):
        st[2 * i], st[2 * i + 1] = fl, _f32_bits(lw)
    keep = [tags, pd, dtags, ddata, tr, st]
    rps = (_RampPatch * max(len(enc.ramp_patches), 1))()
    for i, p in enumerate(enc.ramp_patches):
        stops = (_RampStop * len(p["stops"]))(*[_RampStop(o, c.r, c.g, c.b, c.a) for o, c in p["stops"]])
        keep.append(stops)
        rps[i] = _RampPatch(p["draw_data_offset"], p["extend"], 1 if p["premul"] else 0, len(p["stops"]), C.cast(stops, C.c_void_p))
    ips = (_ImagePatch * max(len(enc.image_patches), 1))()
    for i, p in enumerate(enc.image_patches):
        im = p["image"]
        ips[i] = _ImagePatch(p["draw_data_offset"], im.width, im.height, key_of(im))
    keep += [rps, ips]
    ptr = lambda a: a.ctypes.data if a.size else None  # noqa: E731
    e = _EncodingStreams(ptr(tags), tags.size, ptr(pd), pd.size, ptr(dtags), dtags.size, ptr(ddata), ddata.size, ptr(tr), len(enc.transforms),
                         ptr(st), len(enc.styles), enc.n_paths, enc.n_clips, enc.n_open_clips, C.cast(rps, C.c_void_p), len(enc.ramp_patches),
                         C.cast(ips, C.c_void_p), len(enc.image_patches))
    return e, keep


def _params_struct(p: RenderParams, bin_rows=(0, 0), tile_rows=(0, 0)) -> _Params:
    return _Params(p.base_color.premul_rgba8_u32(), int(p.width), int(p.height), int(p.antialiasing_method),
                   int(bin_rows[0]), int(bin_rows[1]), int(tile_rows[0]), int(tile_rows[1]))


class Renderer:
    """`vello::Renderer`: `Renderer(options)`, then `render_to_texture(scene, params)`."""

    # the device arrays the bind_* methods hold while bound (_bind), None while unbound: of bind_instance_transforms,
    # bind_draw_colors, bind_path_points, bind_gradient_stops, bind_transforms, bind_draw_visibility, bind_stroke_widths and
    # bind_draw_opacity
    _bound = _colors = _points = _stops = _xforms = _visibility = _widths = _opacity = None

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
        self._fragment_pixels = {}  # id(pixel array) -> its contiguous copy while it lives: keys of upload_fragment's non-contiguous images
        self._destinations = {}  # key -> the device array a registered destination writes (kept alive while registered)
        self._background = None  # the device array of set_background
        self._background_shape = None  # (cells, H, W, 4-D) of a linear background: what _check_background compares frames with
        self._frame_size = None  # (width, height) of the last frame that succeeded: the shape of last_damage
        self._cells = 1  # cells of the installed scene (set_cells; every installation is one cell)
        self._hit_extent = None  # (width, cells * height) of the last frame that succeeded: hit_map's whole frame

    @classmethod
    def _borrowed(cls, lib, handle: int, owner):
        """A view of a renderer owned by someone else (a RendererGroup): closing it frees nothing."""
        r = cls.__new__(cls)
        r.lib, r.handle, r.options, r.last_stats, r._keep = lib, C.c_void_p(handle), None, None, None
        r._owner = owner
        r._device_images = {}
        r._fragment_pixels = {}
        r._destinations = {}
        r._background = None
        r._background_shape = None
        r._frame_size = None
        r._cells = 1
        r._hit_extent = None
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
        self._cells = 1
        rc = self.lib.vb_scene_upload(self.handle, scene.ctypes.data, scene.nbytes, C.byref(lay),
                                      ramps.ctypes.data if ramps.size else None, 512, ramps.shape[0],
                                      atlas.ctypes.data, atlas.shape[1], atlas.shape[0])
        self._check(rc, "vb_scene_upload")

    def upload_scene(self, scene) -> "Layout":
        """Resolve the `Scene` `scene` on the device and install it (`vb_scene_upload_streams`), keeping its gradient stops, so
        that `bind_gradient_stops` can bind them (a packed `upload` keeps only resolved ramps). Returns its Layout."""
        from .encoding import Layout
        e, keep = _encoding_streams(scene.encoding, self._image_key)
        L = _Layout()
        self._check(self.lib.vb_scene_upload_streams(self.handle, C.byref(e), C.byref(L)), "vb_scene_upload_streams")
        self._cells = 1
        return Layout(L.n_draw_objects, L.n_paths, L.n_clips, L.bin_data_start, L.path_tag_base, L.path_data_base, L.draw_tag_base,
                      L.draw_data_base, L.transform_base, L.style_base)

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

    # -- composition: frames built on the device from resident fragments (vb_fragment_upload / vb_compose) -------------------
    def upload_fragment(self, scene) -> int:
        """Copy `scene` (a `Scene` or a `NativeScene`) to the device as a fragment, with its images' pixels and its gradient
        stops, and return its id for `compose`. The scene is not needed afterwards; editing it does not change the fragment."""
        from .scene_native import NativeScene, _lib as _scene_lib
        fid = C.c_uint32(0)
        if isinstance(scene, NativeScene):
            self._check(_scene_lib().vb_scene_upload_fragment(self.handle, scene.handle, C.byref(fid)), "vb_scene_upload_fragment")
            return int(fid.value)
        e, keep = _encoding_streams(scene.encoding, self._image_key)
        self._check(self.lib.vb_fragment_upload(self.handle, C.byref(e), C.byref(fid)), "vb_fragment_upload")
        return int(fid.value)

    def _image_key(self, im: Image) -> Optional[int]:
        """The pointer an image of a `Scene` is keyed and read by: its key, else its pixel array (as resolve keys images by
        the array's identity; for a non-contiguous array, a contiguous copy kept while the array lives, so that the key stays the
        same)."""
        if im.key is not None:
            return int(im.key)
        d = im.data
        if isinstance(d, np.ndarray) and d.dtype == np.uint8 and d.flags.c_contiguous:
            return int(d.ctypes.data)
        copy = self._fragment_pixels.get(id(d))
        if copy is None:
            copy = np.ascontiguousarray(d, dtype=np.uint8).copy()
            try:  # held while `d` lives, so that the key stays the same for it (and no other array can have its id)
                weakref.finalize(d, self._fragment_pixels.pop, id(d), None)
                self._fragment_pixels[id(d)] = copy
            except TypeError:  # not weakly referenceable: a copy for this upload only
                pass
        return int(copy.ctypes.data)

    def upload_device_paths(self, points, ring_offsets, colors, *, path_offsets=None, style=0, closed: bool = True,
                            draw_index=None, point_kinds=None):
        """Build a fragment on the device from ragged device arrays (`vb_fragment_from_device_paths`) and return (fragment id,
        draw objects). `points` is float32 (P, 2) x y rows, `ring_offsets` int32 (R + 1,): ring r is points ring_offsets[r] ..
        ring_offsets[r + 1] - 1; `path_offsets` int32 (N + 1,) over rings (None: each ring is a path); `colors` float32 (N, 4)
        straight-alpha r g b a, one row per path. Arrays come through `__cuda_array_interface__` (e.g. torch CUDA tensors); points
        and colours may be columns of larger arrays (rows any multiple of 4 bytes apart), offsets are contiguous. `style` is a
        fill rule (FILL_NON_ZERO, FILL_EVEN_ODD) or an undashed `Stroke`; `closed` closes a stroke's rings (fills always close).
        The fragment is word for word `upload_fragment` of a Scene that fills (or strokes) each path i with Color(colors[i]) under
        the identity, its shape being, per ring, a move to the first point, lines to the others and, when closed, a close.
        `draw_index` (optional, int32 (N,) device array) receives each path's draw object in the fragment, or -1 for a path that
        encodes nothing. `point_kinds` (optional, uint8 or bool (P,) device array) makes the paths curved
        (`vb_fragment_from_device_curves`): 0 marks an on-curve point, 1 an off-curve one, and each on-curve point after a ring's
        first ends a segment chosen by the off-curve points in front of it: none a line, one a quad, two a cubic. A ring starts
        and ends on-curve; a curved closing segment ends on a repeat of the first point. None makes every point on-curve. Write
        the arrays on `self.stream` (or synchronise) before the call; it returns once the fragment is built."""
        from .encoding import Stroke
        who = "upload_device_paths"
        d, kinds = self._device_paths(who, points, ring_offsets, colors, path_offsets, draw_index, point_kinds)
        if isinstance(style, Stroke):
            if style.dash_pattern:
                raise ValueError(f"{who}: dashed strokes are built by upload_device_dashes (or encode them with Scene.stroke)")
            self._device_stroke(d, style, closed)
        else:
            d.kind, d.fill_rule = 0, int(style)
        fid, n_draws = C.c_uint32(0), C.c_uint32(0)
        if point_kinds is None:
            self._check(self.lib.vb_fragment_from_device_paths(self.handle, C.byref(d), C.byref(fid), C.byref(n_draws)),
                        "vb_fragment_from_device_paths")
        else:
            self._check(self.lib.vb_fragment_from_device_curves(self.handle, C.byref(d), kinds, C.byref(fid), C.byref(n_draws)),
                        "vb_fragment_from_device_curves")
        return int(fid.value), int(n_draws.value)

    def upload_device_dashes(self, points, ring_offsets, colors, stroke, *, path_offsets=None, closed: bool = True,
                             draw_index=None, point_kinds=None, dash_offsets=None):
        """Build a fragment of dashed strokes on the device (`vb_fragment_from_device_dashes`) and return (fragment id, draw
        objects). The arrays are those of `upload_device_paths` (with `point_kinds`, curved paths); `stroke` is a dashed
        `Stroke`, whose pattern and offset cut every path, or, with `dash_offsets` (float32 (N,) device array, or a column of a
        larger one), path i's offset is dash_offsets[i]: an animated offset is a new fragment per frame. The fragment is word for
        word `upload_fragment` of a Scene that strokes each path i with Color(colors[i]) under the identity, with `stroke` and
        dash offset float(dash_offsets[i]) (or stroke.dash_offset), its shape being `upload_device_paths`' with the rings of fewer
        than two points left out. Write the arrays on `self.stream` (or synchronise) before the call; it returns once the
        fragment is built."""
        from .encoding import Stroke
        who = "upload_device_dashes"
        if not isinstance(stroke, Stroke) or not stroke.dash_pattern:
            raise ValueError(f"{who}: stroke must be a Stroke with a dash pattern")
        d, kinds = self._device_paths(who, points, ring_offsets, colors, path_offsets, draw_index, point_kinds)
        self._device_stroke(d, stroke, closed)
        pattern = (C.c_double * len(stroke.dash_pattern))(*(float(v) for v in stroke.dash_pattern))
        dash = _Dash(C.cast(pattern, C.c_void_p), len(stroke.dash_pattern), float(stroke.dash_offset), None, 4)
        if dash_offsets is not None:
            ptr, n, pitch = _device_rows(dash_offsets, who, "dash offsets", 1, vector=True, empty=True)
            if n != d.n_paths:
                raise ValueError(f"{who}: {n} dash offsets for {d.n_paths} paths")
            dash.offsets, dash.offset_pitch_bytes = ptr, pitch
        fid, n_draws = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.vb_fragment_from_device_dashes(self.handle, C.byref(d), kinds, C.byref(dash), C.byref(fid),
                                                            C.byref(n_draws)), "vb_fragment_from_device_dashes")
        return int(fid.value), int(n_draws.value)

    @staticmethod
    def _device_paths(who, points, ring_offsets, colors, path_offsets, draw_index, point_kinds):
        """The checked arrays of `upload_device_paths` and `upload_device_dashes`: (_DevicePaths without its style, kinds)."""
        pts, n_pts, pitch = _device_rows(points, who, "points", 2, empty=True)
        rings, n_roff = _device_offsets(ring_offsets, who, "ring_offsets")
        if n_roff == 0:
            raise ValueError(f"{who}: ring_offsets has n_rings + 1 entries, at least 1")
        paths, n_poff = (None, n_roff) if path_offsets is None else _device_offsets(path_offsets, who, "path_offsets")
        if n_poff == 0:
            raise ValueError(f"{who}: path_offsets has n_paths + 1 entries, at least 1")
        cols, n_cols, cpitch = _device_rows(colors, who, "colours", 4, empty=True)
        if n_cols != n_poff - 1:
            raise ValueError(f"{who}: {n_cols} colours for {n_poff - 1} paths")
        kinds = None if point_kinds is None else _device_kinds(point_kinds, n_pts, who)
        d = _DevicePaths(pts, n_pts, pitch, rings, n_roff - 1, paths, n_poff - 1, cols, cpitch)
        if draw_index is not None:
            idx, n_idx = _device_offsets(draw_index, who, "draw_index")
            if n_idx != n_poff - 1:
                raise ValueError(f"{who}: draw_index has {n_idx} entries for {n_poff - 1} paths")
            d.draw_index = idx
        return d, kinds

    @staticmethod
    def _device_stroke(d, stroke, closed):
        d.kind, d.width, d.miter_limit = 1, stroke.width, stroke.miter_limit
        d.join, d.start_cap, d.end_cap, d.closed = stroke.join, stroke.start_cap, stroke.end_cap, 1 if closed else 0

    def free_fragment(self, fragment: int):
        """Release a fragment (after the work already enqueued that reads it). Composed scenes are copies: they stay."""
        self._check(self.lib.vb_fragment_free(self.handle, int(fragment)), "vb_fragment_free")

    def compose(self, instances):
        """Make the renderer's scene `Scene()` with every `(fragment id, Affine or None)` of `instances` appended in order,
        resolved, built on the device from the resident fragments (`vb_compose`; asynchronous on `self.stream`). Returns
        (Layout, draw_offsets): instance k's draws are draw objects draw_offsets[k] .. draw_offsets[k + 1] - 1."""
        return self._compose(instances, "vb_compose")

    def recompose(self, instances):
        """`compose`, after which the next frame repaints only what changed (`vb_recompose`): with damage tracking on and the
        last frame rendered from the composition being replaced, the old and new instance lists are matched in order, and only
        the tiles of the instances added, removed or changed (and of draws whose enclosing clip changed) are damaged. Otherwise,
        and for `compose` itself, the next frame is full. Same return value as `compose`."""
        return self._compose(instances, "vb_recompose")

    def _compose(self, instances, fn):
        from .encoding import Layout
        inst = list(instances)
        arr = (_Instance * max(len(inst), 1))()
        for k, (fid, t) in enumerate(inst):
            arr[k].fragment = int(fid)
            if t is not None:
                arr[k].has_transform = 1
                for i, v in enumerate(t.coeffs):
                    arr[k].transform[i] = float(v)
        L = _Layout()
        offs = (C.c_uint32 * (len(inst) + 1))()
        self._check(getattr(self.lib, fn)(self.handle, arr, len(inst), C.byref(L), offs), fn)
        self._cells = 1
        lay = Layout(L.n_draw_objects, L.n_paths, L.n_clips, L.bin_data_start, L.path_tag_base, L.path_data_base, L.draw_tag_base,
                     L.draw_data_base, L.transform_base, L.style_base)
        return lay, [int(v) for v in offs]

    def _bind(self, name, held, t, rows_of):
        """The body of the bind_* methods: bind `t` with vb_<name>, from the (pointer, rows, row pitch) that rows_of(t) checks
        and returns, or unbind for None; and hold `t` in the attribute `held` while it is bound."""
        fn = "vb_" + name
        ptr, n, pitch = (None, 0, 0) if t is None else rows_of(t)
        self._check(getattr(self.lib, fn)(self.handle, ptr, n, pitch), fn)
        setattr(self, held, t)

    def bind_instance_transforms(self, t):
        """Render instance k of the last `compose` under row k of the device array `t` in every frame from now on, read when
        the frame runs (`vb_bind_instance_transforms`): `t` is float32 (n, 6) [a b c d e f] rows, one per composed instance, with
        `__cuda_array_interface__` (e.g. a torch CUDA tensor, or columns of a larger one such as `state[:, 2:8]`). Write it on
        `self.stream` (or synchronise) before a frame, never while one runs; frames then need no further call. A row that is not
        finite leaves its instance as composed. `t` is held while bound; None unbinds. A new scene (upload, compose) unbinds."""
        self._bind("bind_instance_transforms", "_bound", t, lambda t: _device_rows(t, "bind_instance_transforms", "transforms", 6))

    def bind_draw_colors(self, t):
        """Render draw object k of the installed scene, for every row k of the device array `t`, as if it had been encoded with
        `Color(row k)`, in every frame from now on, read when the frame runs (`vb_bind_draw_colors`): `t` is float32 (n, 4)
        straight-alpha r g b a rows, n at most `Scene.n_draw_objects`, with `__cuda_array_interface__` (e.g. a torch CUDA tensor,
        or columns of a larger one such as `state[:, 3:7]`). Row k belongs to draw object k, the index `hit_test` returns (global
        in a composed scene or a batch). It applies to solid fills, strokes and blurred rectangles; rows of other draw objects
        are ignored, and draw objects from n on keep their encoded colour, as does one whose row is not finite. Write it on
        `self.stream` (or synchronise) before a frame, never while one runs; frames then need no further call. `t` is held
        while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_draw_colors", "_colors", t, lambda t: _device_rows(t, "bind_draw_colors", "colours", 4))

    def bind_path_points(self, t):
        """Take point k of the installed scene's path data from row k of the device array `t` in every frame from now on, read
        when the frame runs (`vb_bind_path_points`): `t` is float32 (n, 2) x y rows, n at most the scene's `Scene.n_points`, with `__cuda_array_interface__` (e.g. a torch CUDA tensor, or columns of a larger one such as
        `state[:, 4:6]`). Row k is path-data words 2k and 2k + 1 (global in a composed scene or a batch), in the coordinates the
        point was encoded in: the path's transform, bound instance transforms and a view still apply. Every frame renders what
        uploading the scene with those words overwritten would render; points from n on, and a point whose row is not finite,
        keep their encoded values. Write it on `self.stream` (or synchronise) before a frame, never while one runs; frames then
        need no further call. `t` is held while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_path_points", "_points", t, lambda t: _device_rows(t, "bind_path_points", "points", 2))

    def bind_gradient_stops(self, t):
        """Take stop k of the installed scene's gradients from row k of the device array `t` in every frame from now on, read
        when the frame runs (`vb_bind_gradient_stops`): `t` is float32 (n, 5) offset r g b a rows (straight alpha, after the
        brush alpha), n at most the scene's `Scene.n_stops`, with `__cuda_array_interface__` (e.g. a torch CUDA tensor, or
        columns of a larger one such as `state[:, 2:7]`). Row k is stop k of the ramp patches in draw-data order (global in a
        composed scene or a batch). Every frame renders what uploading the scene's streams with those stops would render; stops
        from n on, and a stop whose row is not finite, keep their encoded values. The scene must have been installed with its
        stops (`upload_scene`, `NativeScene.upload_device`, `compose`), not as packed bytes. Write it on `self.stream` (or
        synchronise) before a frame, never while one runs; frames then need no further call. `t` is held while bound; None
        unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_gradient_stops", "_stops", t, lambda t: _device_rows(t, "bind_gradient_stops", "stops", 5))

    def bind_transforms(self, t):
        """Take transform-stream entry k of the installed scene from row k of the device array `t` in every frame from now on,
        read when the frame runs (`vb_bind_transforms`): `t` is float32 (n, 6) [a b c d e f] rows (kurbo Affine order), n at
        most the scene's `Scene.n_transforms`, with `__cuda_array_interface__` (e.g. a torch CUDA tensor, or columns of a larger
        one such as `state[:, 2:8]`). Row k is entry k of the transform stream (global in a composed scene or a batch): calls
        with equal consecutive transforms share one entry, and a brush transform is an entry of its own holding `transform *
        brush_transform`. Every frame renders what installing the scene with those entries overwritten would render; entries
        from n on, and an entry whose row is not finite, keep the value the frame would read unbound. Bound instance transforms
        and a view still apply (a view on top). Any installed scene can be bound, packed ones included. Write it on
        `self.stream` (or synchronise) before a frame, never while one runs; frames then need no further call. `t` is held
        while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_transforms", "_xforms", t, lambda t: _device_rows(t, "bind_transforms", "transforms", 6))

    def bind_draw_visibility(self, t):
        """Show draw object k of the installed scene only while byte k of the device array `t` is nonzero, in every frame from
        now on, read when the frame runs (`vb_bind_draw_visibility`): `t` is a 1-D bool or uint8 array of n flags, n at most
        the scene's `Scene.n_draw_objects`, with `__cuda_array_interface__` and any positive byte stride (e.g. a torch CUDA
        tensor, or a column of a larger uint8 state tensor such as `state[:, 3]`). Index k is the draw object of `hit_test`,
        global in a composed scene (instance i owns `draw_offsets[i] ..`) or a batch; draw objects from n on are shown. Every
        frame renders what uploading the scene re-encoded without the hidden draw objects would render. Hiding a push_*_layer's
        draw object hides the whole layer, up to its pop_layer (whose flag is ignored), and its blend; hide the layer's own
        draws too to skip their flattening. Hit tests and hit maps
        never return a hidden draw object. Write `t` on `self.stream` (or synchronise) before a frame; frames then need no
        further call. Per instance of a composed scene, one device op makes the flags from an (instances,) bool mask and the
        instances' draw counts (`counts = draw_offsets[1:] - draw_offsets[:-1]` as a device tensor):

            r.bind_draw_visibility(mask_inst.repeat_interleave(counts))

        `t` is held while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_draw_visibility", "_visibility", t, lambda t: _device_flags(t, "bind_draw_visibility"))

    def bind_stroke_widths(self, t):
        """Stroke draw object k of the installed scene with the line width in row k of the device array `t`, in every frame from
        now on, read when the frame runs (`vb_bind_stroke_widths`): `t` is float32 (n,) or (n, 1), n at most the scene's
        `Scene.n_draw_objects`, with `__cuda_array_interface__` and rows any multiple of 4 bytes apart (e.g. a torch CUDA
        tensor, or a column of a larger one such as `state[:, 5]`). Index k is the draw object of `hit_test`, global in a
        composed scene or a batch. A row is a width in the stroke's own coordinates, as `Stroke.width` is: the path's transform,
        bound transforms and a view still apply (for a constant on-screen width under a zoom z, write w / z). It applies to
        strokes only; rows of other draw objects are ignored, and draw objects from n on, and a stroke whose row is not finite
        and > 0, keep their encoded width. Joins, caps, miter limit and dashes keep theirs. Every frame renders what the scene
        re-encoded with those widths renders. Write `t` on `self.stream` (or synchronise) before a frame; frames then need no
        further call. `t` is held while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_stroke_widths", "_widths", t, lambda t: _device_rows(t, "bind_stroke_widths", "widths", 1, vector=True))

    def bind_draw_opacity(self, t):
        """Draw layer or image k of the installed scene with the alpha in row k of the device array `t`, in every frame from now
        on, read when the frame runs (`vb_bind_draw_opacity`): `t` is float32 (n,) or (n, 1), n at most the scene's
        `Scene.n_draw_objects`, with `__cuda_array_interface__` and rows any multiple of 4 bytes apart (e.g. a torch CUDA
        tensor, or a column of a larger one such as `state[:, 5]`). Index k is the draw object of `hit_test`, global in a
        composed scene or a batch. A finite row is clamped to [0, 1] and becomes the alpha of a push_*_layer's draw object (the
        pop_layer's row is ignored) or of an image (in place of the image's alpha times the brush alpha). A push_clip_layer with
        a row below 1 is drawn as push_layer(MIX_NORMAL, COMPOSE_SRC_OVER, row), so its whole layer fades; at 1 it is drawn as
        encoded. Rows of fills, strokes, gradients and blurred rectangles are ignored, and draw objects from n on, and a row
        that is not finite, keep their encoded values. Every frame renders what the scene re-encoded with those alphas renders;
        hit tests do not change. Write `t` on `self.stream` (or synchronise) before a frame; frames then need no further call.
        `t` is held while bound; None unbinds. A new scene (any upload, compose or recompose) unbinds."""
        self._bind("bind_draw_opacity", "_opacity", t, lambda t: _device_rows(t, "bind_draw_opacity", "alphas", 1, vector=True))

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
        self._check_background(params, 1)
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
        self._frame_size = (int(params.width), int(params.height))
        self._cells, self._hit_extent = 1, self._frame_size
        return out

    def render_stream(self, scenes, params: RenderParams):
        """Render a sequence of scenes through the streaming entry points (vb_render_begin / vb_readback_wait): a generator
        of RGBA8 images, each complete when yielded. Three frames are in flight (upload | rasterise | read back), so frame k-2
        is yielded after frame k has been submitted."""
        self._check_background(params, 1)
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
            self._cells, self._hit_extent = 1, (int(params.width), int(params.height))  # once it completes
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
        self._cells = arr.size - 1

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
        self._check_background(params, n)
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
        self._frame_size = (w, h)
        self._hit_extent = (w, n * h)
        return out

    @staticmethod
    def stripe_rows(params: RenderParams, bin_rows=(0, 0), tile_rows=(0, 0)):
        if tile_rows[1] > tile_rows[0]:
            return min(tile_rows[0] * 16, params.height), min(tile_rows[1] * 16, params.height)
        if bin_rows[1] > bin_rows[0]:
            return min(bin_rows[0] * 256, params.height), min(bin_rows[1] * 256, params.height)
        return 0, params.height

    # format: (vb_destination.format, element type of a linear target)
    DEST_FORMATS = {"rgba8": (0, "|u1"), "bgra8": (1, "|u1"), "rgba16f": (2, "<f2"), "rgba32f": (3, "<f4")}
    DEST_ALPHA = {"straight": 0, "premultiplied": 0x100}

    def register_destination(self, target=None, *, array=None, format: str = "rgba8", alpha: str = "straight",
                             origin=(0, 0)) -> int:
        """Register where frames can be rendered straight to (`vb_register_destination`) and return its key, which goes
        wherever `out_device_ptr` goes (`render_resident`, `enqueue`, `run_stages`).

        `target`: an (H, W, 4) uint8 device array (`__cuda_array_interface__`: a torch CUDA tensor, or a slice of a larger
        one) with strides (pitch, 4, 1), or float16 / float32 for the float formats, with strides (pitch, 8, 2) /
        (pitch, 16, 4); pixel (x, y) of a frame lands at element [y, x]. It must hold the frames rendered into it: the row
        pitch is checked at each frame, the rows are the caller's to provide. `array`: an integer `cudaArray_t` handle of a
        2-D array created with `cudaArraySurfaceLoadStore` (such as level 0 of an imported Vulkan image), of four channels
        that match the format (8-bit unsigned, 16-bit float or 32-bit float); pixel (x, y) lands at texel
        (origin[0] + x, origin[1] + y), and a frame that does not fit is refused. `format`: "rgba8" (vello's byte order),
        "bgra8", "rgba16f" or "rgba32f". `alpha`: "straight" (vello's) or "premultiplied". The values are fine's f32 pixels
        clamped to [0, 1], rounded to 8 bits or to halves for the narrower formats (see `vb_register_destination`). A
        bin_row / tile_row window writes its rows at their own rows. Damage-tracked frames into the same key are
        incremental."""
        if format not in self.DEST_FORMATS:
            raise ValueError(f"register_destination: format is one of {sorted(self.DEST_FORMATS)}, not {format!r}")
        if alpha not in self.DEST_ALPHA:
            raise ValueError(f"register_destination: alpha is one of {sorted(self.DEST_ALPHA)}, not {alpha!r}")
        fmt, typestr = self.DEST_FORMATS[format]
        fmt |= self.DEST_ALPHA[alpha]
        if (target is None) == (array is None):
            raise ValueError("register_destination: give either a target or an array")
        if target is not None:
            ptr, _, _, pitch = _device_image(target, typestr)
            d = _Destination(0, fmt, ptr, pitch, None, 0, 0)
        else:
            d = _Destination(1, fmt, None, 0, int(array), int(origin[0]), int(origin[1]))
        key = C.c_void_p()
        self._check(self.lib.vb_register_destination(self.handle, C.byref(d), C.byref(key)), "vb_register_destination")
        self._destinations[int(key.value)] = target
        return int(key.value)

    def unregister_destination(self, key: int):
        """Unregister a destination (`vb_unregister_destination`), once the frames enqueued into it have completed."""
        self._check(self.lib.vb_unregister_destination(self.handle, C.c_void_p(key)), "vb_unregister_destination")
        self._destinations.pop(int(key), None)

    def set_background(self, target=None, *, array=None, format: str = "rgba8", alpha: str = "straight", origin=(0, 0)):
        """Draw the frames enqueued from now on over a background instead of over the base colour (`vb_set_background`);
        with neither `target` nor `array`, clear it.

        `target`: an (H, W, 4) device array (`__cuda_array_interface__`) of the format's element type, as
        `register_destination` takes it, or an (N, H, W, 4) one whose cells are H row pitches apart: cell c of a batch
        (`set_cells`) starts from target[c]. Pixel (x, y) of a frame starts from element [y, x]. `array`: an integer
        `cudaArray_t` handle, read at texel (origin[0] + x, origin[1] + y). `format` and `alpha` describe the texels as
        for `register_destination`. Each texel is read as f32, clamped to [0, 1] and, for straight alpha, premultiplied. The
        background may be the frame's destination itself. It must stay alive, with its pixels as the frames should see them,
        until the frames that read it have completed. A target's shape must cover the frames rendered over it: every
        rendering method refuses a frame (ValueError) whose rows, columns or cells it does not hold (`_check_background`).
        An array's extent is checked by the library."""
        if format not in self.DEST_FORMATS:
            raise ValueError(f"set_background: format is one of {sorted(self.DEST_FORMATS)}, not {format!r}")
        if alpha not in self.DEST_ALPHA:
            raise ValueError(f"set_background: alpha is one of {sorted(self.DEST_ALPHA)}, not {alpha!r}")
        fmt, typestr = self.DEST_FORMATS[format]
        fmt |= self.DEST_ALPHA[alpha]
        if target is not None and array is not None:
            raise ValueError("set_background: give a target, an array or neither")
        if target is None and array is None:
            self._background, self._background_shape = None, None
            self._check(self.lib.vb_set_background(self.handle, None), "vb_set_background")
            return
        shape = None
        if target is not None:
            ptr, pitch = _background_image(target, typestr)
            d = _Destination(0, fmt, ptr, pitch, None, 0, 0)
            dims = tuple(int(v) for v in target.__cuda_array_interface__["shape"])
            shape = (dims[0], dims[1], dims[2], True) if len(dims) == 4 else (1, dims[0], dims[1], False)
        else:
            d = _Destination(1, fmt, None, 0, int(array), int(origin[0]), int(origin[1]))
        # a failed call leaves the renderer without a background when it had to release an array's (vb_set_background)
        self._background, self._background_shape = None, None
        self._check(self.lib.vb_set_background(self.handle, C.byref(d)), "vb_set_background")
        self._background, self._background_shape = target, shape

    def _check_background(self, params: RenderParams, cells: int):
        """A linear background must hold every row of every cell a frame reads; the C descriptor has no height, so the shape
        of the target given to set_background is compared here. Cell c is read from row c * height: an (H, W, 4) target
        needs cells * height rows, and an (N, H, W, 4) one N >= cells and, with more than one cell, H == height."""
        if self._background_shape is None:
            return
        n, h, w, four_d = self._background_shape
        height, width = int(params.height), int(params.width)
        fits = w >= width and (h >= height and n >= cells and (cells == 1 or h == height) if four_d else h >= cells * height)
        if not fits:
            have = f"({n}, {h}, {w}, 4)" if four_d else f"({h}, {w}, 4)"
            raise ValueError(f"set_background: a {have} background cannot hold {cells} cell(s) of {width}x{height}")

    def render_resident(self, params: RenderParams, out_device_ptr: int = 0, bin_rows=(0, 0), tile_rows=(0, 0)) -> FrameStats:
        """Render the uploaded scene into a device buffer (0 = the renderer's own target)."""
        self._check_background(params, self._cells)
        ps = _params_struct(params, bin_rows, tile_rows)
        st = FrameStats()
        rc = self.lib.vb_render_resident(self.handle, C.byref(ps), C.c_void_p(out_device_ptr or None), C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_render_resident")
        self._frame_size = (int(params.width), int(params.height))
        self._hit_extent = (int(params.width), self._cells * int(params.height))
        return st

    def enqueue(self, params: RenderParams, out_device_ptr: int = 0, bin_rows=(0, 0), tile_rows=(0, 0)):
        self._check_background(params, self._cells)
        ps = _params_struct(params, bin_rows, tile_rows)
        self._check(self.lib.vb_render_enqueue(self.handle, C.byref(ps), C.c_void_p(out_device_ptr or None)), "vb_render_enqueue")
        self._enqueued_size = (int(params.width), int(params.height))
        self._enqueued_extent = (int(params.width), self._cells * int(params.height))

    def finish(self) -> FrameStats:
        st = FrameStats()
        rc = self.lib.vb_frame_finish(self.handle, C.byref(st))
        self.last_stats = st
        self._check(rc, "vb_frame_finish")
        self._frame_size = getattr(self, "_enqueued_size", self._frame_size)
        self._hit_extent = getattr(self, "_enqueued_extent", self._hit_extent)
        return st

    @property
    def stream(self) -> int:
        return int(self.lib.vb_stream(self.handle) or 0)

    def target_ptr(self) -> int:
        n = C.c_size_t(0)
        return int(self.lib.vb_target(self.handle, C.byref(n)) or 0)

    # -- stage-level access (parity tests) -----------------------------------------------------------
    def run_stages(self, params: RenderParams, first: str, last: str, out_device_ptr: int = 0, bin_rows=(0, 0)):
        if last == "fine":
            self._check_background(params, self._cells)
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

    # look-back monoids of debug_lookback (VB_LOOKBACK_*) and their words per partition
    LOOKBACK_SUM1, LOOKBACK_SUM5, LOOKBACK_BACKDROP, LOOKBACK_AFFINE = 0, 1, 2, 3
    LOOKBACK_WORDS = {0: 1, 1: 5, 2: 3, 3: 2}
    LOOKBACK_MAX_DELAY_NS = 1_000_000

    def debug_lookback(self, op: int, agg: np.ndarray, delay_ns=None) -> np.ndarray:
        """Test-only: the device look-back alone (vb_debug_lookback) over len(agg) partitions, partition p waiting delay_ns[p]
        before it publishes agg[p] ((n_parts, K) u32). Returns every partition's exclusive prefix, (n_parts, K) u32."""
        a = np.ascontiguousarray(agg, dtype=np.uint32)
        n = a.shape[0]
        if a.shape != (n, self.LOOKBACK_WORDS[op]):
            raise ValueError(f"debug_lookback: agg must be (n_parts, {self.LOOKBACK_WORDS[op]}), not {a.shape}")
        d = None if delay_ns is None else np.ascontiguousarray(delay_ns, dtype=np.uint32)
        if d is not None and d.shape != (n,):
            raise ValueError("debug_lookback: one delay per partition")
        out = np.zeros_like(a)
        self._check(self.lib.vb_debug_lookback(self.handle, op, n, a.ctypes.data, None if d is None else d.ctypes.data, out.ctypes.data),
                    "vb_debug_lookback")
        return out

    def set_cuda_graph(self, on: bool):
        """Replay whole frames as CUDA graphs (default on)."""
        self._check(self.lib.vb_set_cuda_graph(self.handle, 1 if on else 0), "vb_set_cuda_graph")

    def set_view(self, affine: Optional[Affine]):
        """Render the uploaded scene under `affine` from the next frame on, as `Scene().append(scene, affine)` would render,
        without uploading it again (pan / zoom of a resident scene). Frames already enqueued keep their view; the view
        survives uploads. Flatten then culls what lies above, below or right of the frame. None clears it."""
        self._check(self.lib.vb_set_view(self.handle, _view_coeffs(affine)), "vb_set_view")

    def hit_test(self, points, out=None):
        """The topmost draw object under each point of the last frame that completed (`vb_hit_test`): for every (x, y) in
        pixel coordinates of that frame (a batch's tall [N * H, W] frame), the index of the last draw object in draw order
        whose outline covers the point inside all its enclosing clips (`Scene.n_draw_objects` tells which index a call got),
        or -1. Alpha and blend modes do not matter; clips are never returned; points outside the frame and NaN give -1.

        A numpy (n, 2) float32 array (or anything numpy turns into one) returns a numpy int32 (n,) array (into `out` when it
        is one), synchronously. A device array (`__cuda_array_interface__`, e.g. a torch CUDA tensor) of n x 2 float32 needs
        `out`, a device int32 array of n: the work is enqueued on `self.stream` and `out` is returned at once (order the
        points' writes before the call and synchronise with that stream before reading `out`)."""
        if hasattr(points, "__cuda_array_interface__"):
            ptr, n = _device_vector(points, 2, ("<f4",), "points")
            if out is None or not hasattr(out, "__cuda_array_interface__"):
                raise ValueError("hit_test: device points need a device int32 array `out`")
            optr, m = _device_vector(out, 1, ("<i4",), "out")
            if m != n:
                raise ValueError(f"hit_test: out holds {m} answers for {n} points")
            self._check(self.lib.vb_hit_test(self.handle, C.c_void_p(ptr), n, C.c_void_p(optr), 1), "vb_hit_test")
            return out
        pts = np.ascontiguousarray(points, dtype=np.float32)
        if pts.ndim != 2 or pts.shape[1] != 2:
            raise ValueError(f"hit_test: points must be (n, 2), not {pts.shape}")
        n = pts.shape[0]
        if out is None:
            out = np.empty(n, dtype=np.int32)
        elif not (isinstance(out, np.ndarray) and out.dtype == np.int32 and out.shape == (n,) and out.flags.c_contiguous):
            raise ValueError(f"hit_test: out must be a contiguous int32 numpy array of shape ({n},)")
        if n:
            self._check(self.lib.vb_hit_test(self.handle, pts.ctypes.data, n, out.ctypes.data, 0), "vb_hit_test")
        return out

    def hit_map(self, rect=None, out=None):
        """`hit_test` at every pixel centre of a rectangle of the last frame that completed (`vb_hit_map`): element [j, i] is
        the answer for the point (x0 + i + 0.5, y0 + j + 0.5), equal int for int. `rect` = (x0, y0, w, h) must lie inside that
        frame; None is the whole frame, (0, 0, W, N * H) for a batch of N cells (reshape it to (N, H, W)).

        With no `out`, or a numpy `out` (int32 (h, w) with element stride 4, so a slice of a larger array works), the call is
        synchronous and returns the numpy map. A device `out` (`__cuda_array_interface__`, e.g. a torch int32 CUDA tensor or a
        row slice of one) of the same shape and element stride gets the map enqueued on `self.stream` and is returned at once
        (synchronise with that stream before reading it). Only the h rows of w answers are written."""
        if rect is None:
            if self._hit_extent is None:
                raise VelloB200Error("hit_map: no frame has completed on this renderer")
            rect = (0, 0) + tuple(self._hit_extent)
        x0, y0, w, h = (int(v) for v in rect)
        if not all(0 <= v < 2 ** 32 for v in (x0, y0, w, h)):
            raise ValueError(f"hit_map: rect must be four unsigned 32-bit integers, not {tuple(rect)}")
        device = out is not None and hasattr(out, "__cuda_array_interface__")
        if device:
            cai = out.__cuda_array_interface__
            shape, typestr, ptr = tuple(int(v) for v in cai["shape"]), cai["typestr"], int(cai["data"][0])
            strides = cai.get("strides") or (4 * w, 4)
        else:
            if out is None:
                out = np.empty((h, w), dtype=np.int32)
            if not isinstance(out, np.ndarray):
                raise ValueError("hit_map: out must be a numpy array or a device array")
            shape, typestr, ptr, strides = out.shape, out.dtype.str, out.ctypes.data, out.strides
        if shape != (h, w) or typestr != "<i4":
            raise ValueError(f"hit_map: out must be int32 of shape ({h}, {w}), not {shape} {typestr}")
        pitch = int(strides[0]) if h > 1 else 4 * w  # one row: its pitch is never used
        if (w > 1 and strides[1] != 4) or (h > 1 and (pitch % 4 or pitch < 4 * w)):
            raise ValueError(f"hit_map: out needs element stride 4 and a row stride of at least 4 * w, not strides {tuple(strides)}")
        self._check(self.lib.vb_hit_map(self.handle, x0, y0, w, h, C.c_void_p(ptr), pitch, 1 if device else 0), "vb_hit_map")
        return out

    def debug_graph_captures(self) -> int:
        """Test-only: whole-frame CUDA graphs this renderer has instantiated so far."""
        n = C.c_uint64(0)
        self._check(self.lib.vb_debug_graph_captures(self.handle, C.byref(n)), "vb_debug_graph_captures")
        return int(n.value)

    def set_occlusion_cull(self, on: bool):
        """fine skips the commands under a tile's last opaque full-tile cover (identical pixels). Default on."""
        self._check(self.lib.vb_set_occlusion_cull(self.handle, 1 if on else 0), "vb_set_occlusion_cull")

    def set_damage_tracking(self, on: bool):
        """Damage tracking (`vb_set_damage_tracking`, default off): a frame rendered into the same device destination as the
        last successful one, with the same scene, size, AA, base colour and view, repaints only the tiles that changed and
        writes no other pixel. With bound instance transforms, the instances whose transforms changed are found on the device;
        `add_damage` names anything else. Switching it on (again) makes the next frame full."""
        self._check(self.lib.vb_set_damage_tracking(self.handle, 1 if on else 0), "vb_set_damage_tracking")

    def set_upload_diff(self, on: bool):
        """Diff re-uploaded scenes against the scene the last tracked frame rendered (`vb_set_upload_diff`, default off): with
        damage tracking on, the frame after `upload`, `NativeScene.upload_device` or a device-destination `vb_render` repaints
        only the tiles of the draw objects that were added, removed or changed, found on the device. Turning it off frees the
        spare scene buffers it keeps."""
        self._check(self.lib.vb_set_upload_diff(self.handle, 1 if on else 0), "vb_set_upload_diff")

    def add_damage(self, rects):
        """Add half-open pixel rectangles (x0, y0, x1, y1), an (n, 4) array, to the next frame's damage (`vb_add_damage`),
        in stream order. Clamped to the frame; no effect while tracking is off."""
        arr = np.ascontiguousarray(rects, dtype=np.uint32).reshape(-1, 4)
        self._check(self.lib.vb_add_damage(self.handle, arr.ctypes.data if arr.size else None, arr.shape[0]), "vb_add_damage")

    def last_damage(self) -> np.ndarray:
        """The tiles the last successful frame rendered (`vb_last_damage`): bool [tiles_h, tiles_w], all True for a full frame."""
        if self._frame_size is None:
            raise VelloB200Error("last_damage: no frame rendered yet")
        w, h = self._frame_size
        out = np.zeros(((h + 15) // 16, (w + 15) // 16), dtype=np.uint8)
        n = C.c_uint32(0)
        self._check(self.lib.vb_last_damage(self.handle, out.ctypes.data, out.size, C.byref(n)), "vb_last_damage")
        return out.astype(bool)

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

    def set_view(self, affine: Optional[Affine]):
        """`Renderer.set_view` on every device's renderer."""
        self._check(self.lib.vb_group_set_view(self.handle, _view_coeffs(affine)), "vb_group_set_view")

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
