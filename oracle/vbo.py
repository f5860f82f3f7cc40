"""ctypes binding for the CPU oracle (oracle/libvbo.so).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module; the product (vello_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

STAGES = ["pathtag", "flatten", "draw", "clip", "binning", "tile_alloc", "path_count", "backdrop",
          "coarse", "path_tiling", "fine"]

DTYPES = {
    "tag_monoids": np.dtype([("trans_ix", "<u4"), ("pathseg_ix", "<u4"), ("pathseg_offset", "<u4"),
                             ("style_ix", "<u4"), ("path_ix", "<u4")]),
    "path_bboxes": np.dtype([("x0", "<i4"), ("y0", "<i4"), ("x1", "<i4"), ("y1", "<i4"),
                             ("draw_flags", "<u4"), ("trans_ix", "<u4")]),
    "lines": np.dtype([("path_ix", "<u4"), ("pad", "<u4"), ("p0", "<f4", 2), ("p1", "<f4", 2)]),
    "draw_monoids": np.dtype([("path_ix", "<u4"), ("clip_ix", "<u4"), ("scene_offset", "<u4"),
                              ("info_offset", "<u4")]),
    "info_bin_data": np.dtype("<u4"),
    "clip_inp": np.dtype([("ix", "<u4"), ("path_ix", "<i4")]),
    "clip_bboxes": np.dtype([("x0", "<f4"), ("y0", "<f4"), ("x1", "<f4"), ("y1", "<f4")]),
    "draw_bboxes": np.dtype([("x0", "<f4"), ("y0", "<f4"), ("x1", "<f4"), ("y1", "<f4")]),
    "bin_headers": np.dtype([("element_count", "<u4"), ("chunk_offset", "<u4")]),
    "paths": np.dtype([("bbox", "<u4", 4), ("tiles", "<u4"), ("pad", "<u4", 3)]),
    "tiles": np.dtype([("backdrop", "<i4"), ("segment_count_or_ix", "<u4")]),
    "seg_counts": np.dtype([("line_ix", "<u4"), ("counts", "<u4")]),
    "segments": np.dtype([("p0", "<f4", 2), ("p1", "<f4", 2), ("y_edge", "<f4"), ("pad", "<u4")]),
    "ptcl": np.dtype("<u4"),
    "blend_spill": np.dtype("<u4"),
    "tile_counts": np.dtype("<u4"),
    "bump": np.dtype([("failed", "<u4"), ("binning", "<u4"), ("ptcl", "<u4"), ("tile", "<u4"),
                      ("seg_counts", "<u4"), ("segments", "<u4"), ("blend", "<u4"), ("lines", "<u4")]),
    "config": np.dtype("<u4"),
}


class _Layout(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "n_draw_objects", "n_paths", "n_clips", "bin_data_start", "path_tag_base", "path_data_base",
        "draw_tag_base", "draw_data_base", "transform_base", "style_base")]


class _Params(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("width", "height", "base_color", "aa", "bin_row0", "bin_row1")]


def build(force: bool = False) -> None:
    """Compile the oracle (gcc). Building the checker is not using it."""
    if force or not all(os.path.exists(os.path.join(_HERE, n)) for n in ("libvbo.so", "libvbo_libm.so")):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))


_libs = {}


def _load(libm: bool):
    key = bool(libm)
    if key not in _libs:
        build()
        lib = C.CDLL(os.path.join(_HERE, "libvbo_libm.so" if libm else "libvbo.so"))
        lib.vbo_create.restype = C.c_void_p
        lib.vbo_destroy.argtypes = [C.c_void_p]
        lib.vbo_bind.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(_Layout), C.c_void_p, C.c_uint32,
                                 C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(_Params)]
        lib.vbo_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lib.vbo_buffer.restype = C.c_void_p
        lib.vbo_buffer.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_size_t)]
        lib.vbo_set_buffer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        lib.vbo_set_threads.argtypes = [C.c_void_p, C.c_int]
        lib.vbo_math.restype = C.c_float
        lib.vbo_math.argtypes = [C.c_int, C.c_float, C.c_float]
        _libs[key] = lib
    return _libs[key]


class Oracle:
    """One oracle context. `render()` runs the whole pipeline; `run()` runs a stage range."""

    def __init__(self, libm: bool = False, threads: int = 1):
        self.lib = _load(libm)
        self.ctx = C.c_void_p(self.lib.vbo_create())
        self.lib.vbo_set_threads(self.ctx, threads)
        self._keep = None

    def __del__(self):
        try:
            self.lib.vbo_destroy(self.ctx)
        except Exception:
            pass

    def bind(self, packed, width: int, height: int, base_color_u32: int = 0xFF000000, aa: int = 0,
             bin_rows=(0, 0)):
        scene = np.ascontiguousarray(packed.scene, dtype=np.uint32)
        ramps = np.ascontiguousarray(packed.ramps, dtype=np.uint32)
        atlas = np.ascontiguousarray(packed.atlas, dtype=np.uint8)
        lay = _Layout(*[int(v) for v in packed.layout.as_array()])
        par = _Params(width, height, base_color_u32, aa, bin_rows[0], bin_rows[1])
        self._keep = (scene, ramps, atlas, lay, par)
        self.width, self.height = width, height
        rc = self.lib.vbo_bind(self.ctx, scene.ctypes.data, scene.size, C.byref(lay),
                               ramps.ctypes.data if ramps.size else None, ramps.shape[0],
                               atlas.ctypes.data, atlas.shape[1], atlas.shape[0], C.byref(par))
        assert rc == 0

    def run(self, first="pathtag", last="fine") -> Optional[np.ndarray]:
        f, l = STAGES.index(first), STAGES.index(last)
        out = None
        if l == len(STAGES) - 1:
            out = np.zeros((self.height, self.width, 4), dtype=np.uint8)
        rc = self.lib.vbo_run(self.ctx, f, l, out.ctypes.data if out is not None else None)
        assert rc == 0, rc
        return out

    def render(self, packed, width, height, base_color_u32=0xFF000000, aa=0, bin_rows=(0, 0)) -> np.ndarray:
        self.bind(packed, width, height, base_color_u32, aa, bin_rows)
        return self.run()

    def buffer(self, name: str) -> np.ndarray:
        n = C.c_size_t(0)
        p = self.lib.vbo_buffer(self.ctx, name.encode(), C.byref(n))
        dt = DTYPES[name]
        if not p or n.value == 0:
            return np.zeros(0, dtype=dt)
        raw = (C.c_uint8 * n.value).from_address(p)
        return np.frombuffer(raw, dtype=np.uint8).copy().view(dt)

    def set_buffer(self, name: str, arr: np.ndarray):
        a = np.ascontiguousarray(arr)
        rc = self.lib.vbo_set_buffer(self.ctx, name.encode(), a.ctypes.data, a.nbytes)
        assert rc == 0

    def math(self, fn: int, a: float, b: float = 0.0) -> float:
        return float(self.lib.vbo_math(fn, a, b))
