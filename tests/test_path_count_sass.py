"""Static checks of the compiled k_path_count (cuobjdump on the object `build()` produces, no GPU needed), beside the table
in test_compiled_kernels.py.

k_path_count touches every line of a frame: it keeps everything in registers (no stack, no local memory) at 40 registers or
fewer, so that six CTAs of 256 threads share an SM, and its shared memory (the per-line state of a 768-line step) lets six
CTAs share an SM too."""
import os
import re
import shutil
import subprocess

import pytest

from .test_compiled_kernels import SMEM_PER_SM, _key, built  # noqa: F401  (fixture)

OBJ = "k_path_count.o"
CTAS, THREADS, REGS = 6, 256, 40

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


def test_path_count_budget(built):  # noqa: F811
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, OBJ)], capture_output=True, text=True, check=True).stdout
    found = [(fn, tuple(map(int, vals))) for fn, *vals in
             re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res) if _key(fn)[0] == "k_path_count"]
    assert len(found) == 1, f"expected one k_path_count in {OBJ}:\n{res}"
    reg, stack, shared, local = found[0][1]
    assert stack == 0 and local == 0, f"k_path_count: {stack} bytes of stack, {local} bytes of local memory"
    assert reg <= REGS, f"k_path_count: {reg} registers, more than {REGS}"
    assert reg * THREADS * CTAS <= 65536
    assert shared * CTAS <= SMEM_PER_SM, f"k_path_count: {shared} B of shared memory, fewer than {CTAS} CTAs per SM"

