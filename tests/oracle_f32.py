"""The CPU oracle's fine with a second output: the f32 values its RGBA8 store rounds (test infrastructure only).

Float destinations store fine's pixel before quantisation, so their tests need that value from an independent computation,
not only its rounding. The oracle (oracle/vbo_fine.c) computes it and rounds it in the same statement. This module builds a
private copy of the oracle in a scratch directory: the oracle's own sources, compiled with the oracle's own CFLAGS (read from
oracle/Makefile), with one addition to fine's store, found by its text. Beside each RGBA8 texel the copy writes, when an f32
output is set:

* premultiplied: clamp01(c), fine's premultiplied pixel c clamped as unorm8 clamps (fminf(1, fmaxf(0, v)); NaN gives 0);
* straight: clamp01(c.rgb * a_inv) with the store's own a_inv = 1 / fmaxf(c.a, 1e-6f), and clamp01(c.a).

Nothing under oracle/ is written; the RGBA8 output and every other stage are the oracle's, unchanged."""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

import numpy as np

from oracle.vbo import Oracle, _Layout, _Params

ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")

# fine's store, the last statement of its per-pixel loop, and what the copy adds after it
STORE = "            o[3] = (uint8_t)unorm8(fg.a);\n"
TAP = """            if (g_f32) {
                float *f = g_f32 + ((size_t)py * cfg->target_width + px) * 4u;
                const float k = g_f32_straight ? a_inv : 1.0f;
                f[0] = fminf(1.0f, fmaxf(0.0f, fg.r * k));
                f[1] = fminf(1.0f, fmaxf(0.0f, fg.g * k));
                f[2] = fminf(1.0f, fmaxf(0.0f, fg.b * k));
                f[3] = fminf(1.0f, fmaxf(0.0f, fg.a));
            }
"""
# fine is not re-entrant (one context renders at a time, vbo_fine.c), so the output is one global, as its thread table is
GLOBALS = """
static float *g_f32;
static int g_f32_straight;
void vbo_set_fine_f32(float *out, int straight) { g_f32 = out; g_f32_straight = straight; }
"""


def build(workdir: str) -> str:
    """Compile the copy into `workdir` and return the library's path."""
    src = open(os.path.join(ORACLE, "vbo_fine.c")).read()
    assert src.count(STORE) == 1, "fine's RGBA8 store is not where this copy expects it (oracle/vbo_fine.c changed)"
    inc = '#include "vbo_internal.h"\n'
    assert src.count(inc) == 1
    src = src.replace(inc, inc + GLOBALS).replace(STORE, STORE + TAP)
    fine = os.path.join(workdir, "vbo_fine_f32.c")
    with open(fine, "w") as f:
        f.write(src)
    cflags = re.search(r"^CFLAGS\s*=\s*(.*)$", open(os.path.join(ORACLE, "Makefile")).read(), re.M).group(1).split()
    lib = os.path.join(workdir, "libvbo_f32.so")
    subprocess.check_call([os.environ.get("CC", "gcc"), *cflags, "-I", ORACLE, "-o", lib, os.path.join(ORACLE, "vbo_stages.c"), fine,
                           "-lm", "-lpthread"])
    return lib


class F32Oracle(Oracle):
    """An Oracle on the copy's library: bind / run / set_buffer as the oracle's, plus `f32(out, straight)`."""

    def __init__(self, lib_path: str, threads: int = 1):
        lib = C.CDLL(lib_path)
        lib.vbo_create.restype = C.c_void_p
        lib.vbo_destroy.argtypes = [C.c_void_p]
        lib.vbo_bind.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(_Layout), C.c_void_p, C.c_uint32,
                                 C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(_Params)]
        lib.vbo_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lib.vbo_buffer.restype = C.c_void_p
        lib.vbo_buffer.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_size_t)]
        lib.vbo_set_buffer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        lib.vbo_set_threads.argtypes = [C.c_void_p, C.c_int]
        lib.vbo_set_fine_f32.argtypes = [C.c_void_p, C.c_int]
        self.lib = lib
        self.ctx = C.c_void_p(lib.vbo_create())
        lib.vbo_set_threads(self.ctx, threads)
        self._keep = None

    def f32(self, out: np.ndarray | None, straight: bool = False):
        """Write the f32 values of every following fine run into `out` ((height, width, 4) float32), or stop (None)."""
        assert out is None or (out.dtype == np.float32 and out.flags.c_contiguous)
        self.lib.vbo_set_fine_f32(None if out is None else out.ctypes.data, int(straight))
