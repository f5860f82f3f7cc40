"""The CPU oracle's fine with per-pixel starting values and an f32 output (test infrastructure only).

Backgrounds (vb_set_background) change only where fine's tiles start: at each pixel's background value instead of the base
colour. This module builds a private copy of the oracle, as tests/oracle_f32.py does (the oracle's own sources and CFLAGS,
in a scratch directory), with tests/oracle_f32.py's f32 store and one more addition to fine, found by its text: when starting
values are set (`F32BgOracle.bg`, the (height, width, 4) float32 premultiplied values of the frame), each tile starts pixel
(x, y) at them. The values come from the float32 numpy restatement of the load (`start_values`). Nothing under oracle/ is
written, and every other stage is the oracle's."""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

import numpy as np

from . import oracle_f32
from .oracle_f32 import ORACLE, F32Oracle

# the tile start of fine_tile, and what the copy puts in its place
INIT = "    for (int i = 0; i < 256; i++) { rgba[i] = base; area[i] = 0.0f; }\n"
BG_INIT = """    for (int i = 0; i < 256; i++) {
        rgba[i] = base;
        area[i] = 0.0f;
        const uint32_t bx = tile_x * 16u + ((uint32_t)i & 15u), by = tile_y * 16u + ((uint32_t)i >> 4);
        if (g_bg && bx < cfg->target_width && by < cfg->target_height) {
            const float *b = g_bg + ((size_t)by * cfg->target_width + bx) * 4u;
            rgba[i].r = b[0]; rgba[i].g = b[1]; rgba[i].b = b[2]; rgba[i].a = b[3];
        }
    }
"""
GLOBALS = """
static const float *g_bg;
void vbo_set_fine_bg(const float *bg) { g_bg = bg; }
"""


def build(workdir: str) -> str:
    """Compile the copy into `workdir` and return the library's path."""
    src = open(os.path.join(ORACLE, "vbo_fine.c")).read()
    assert src.count(oracle_f32.STORE) == 1 and src.count(INIT) == 1, "fine is not what this copy expects (oracle/vbo_fine.c changed)"
    inc = '#include "vbo_internal.h"\n'
    assert src.count(inc) == 1
    src = src.replace(inc, inc + oracle_f32.GLOBALS + GLOBALS).replace(oracle_f32.STORE, oracle_f32.STORE + oracle_f32.TAP)
    src = src.replace(INIT, BG_INIT)
    fine = os.path.join(workdir, "vbo_fine_bg.c")
    with open(fine, "w") as f:
        f.write(src)
    cflags = re.search(r"^CFLAGS\s*=\s*(.*)$", open(os.path.join(ORACLE, "Makefile")).read(), re.M).group(1).split()
    lib = os.path.join(workdir, "libvbo_bg.so")
    subprocess.check_call([os.environ.get("CC", "gcc"), *cflags, "-I", ORACLE, "-o", lib, os.path.join(ORACLE, "vbo_stages.c"), fine,
                           "-lm", "-lpthread"])
    return lib


class F32BgOracle(F32Oracle):
    """An F32Oracle whose fine starts from `bg(values)` while they are set."""

    def __init__(self, lib_path: str, threads: int = 1):
        super().__init__(lib_path, threads)
        self.lib.vbo_set_fine_bg.argtypes = [C.c_void_p]
        self._bg = None

    def bg(self, values: np.ndarray | None):
        assert values is None or (values.dtype == np.float32 and values.flags.c_contiguous and values.shape[-1] == 4)
        self._bg = values
        self.lib.vbo_set_fine_bg(None if values is None else values.ctypes.data)


def clamp01(v):
    """fminf(1, fmaxf(0, v)) as the device computes it: NaN gives 0, and -0 gives +0 (numpy's fmax may keep -0; adding +0
    makes it +0 and changes no other value)."""
    return np.fmin(np.float32(1.0), np.fmax(np.float32(0.0), v)) + np.float32(0.0)


def start_values(texels: np.ndarray, fmt: str, premultiplied: bool) -> np.ndarray:
    """The load of vb_set_background in float32: texels ((..., 4) uint8, float16 or float32 as stored) -> fine's starting
    premultiplied pixels. Each channel as f32 (byte / 255.0f, r and b swapped back for bgra8; the half exactly; the float as
    it is), clamp01 (NaN gives 0), then for straight alpha each colour channel times alpha."""
    if fmt in ("rgba8", "bgra8"):
        v = texels.astype(np.float32) / np.float32(255.0)
        if fmt == "bgra8":
            v = v[..., [2, 1, 0, 3]]
    else:
        v = texels.astype(np.float32)
    v = clamp01(v).astype(np.float32)
    if not premultiplied:
        v[..., :3] = v[..., :3] * v[..., 3:4]
    return np.ascontiguousarray(v)


def unorm8(v):
    return np.floor(np.float32(0.5) + np.float32(255.0) * clamp01(v)).astype(np.uint8)


def store_rgba8_straight(pre: np.ndarray) -> np.ndarray:
    """fine's RGBA8 straight store of premultiplied f32 pixels."""
    a_inv = np.float32(1.0) / np.fmax(pre[..., 3:], np.float32(1e-6))
    out = np.empty(pre.shape, np.uint8)
    out[..., :3] = unorm8(pre[..., :3] * a_inv)
    out[..., 3] = unorm8(pre[..., 3])
    return out
