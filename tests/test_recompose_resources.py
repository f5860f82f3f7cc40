"""Static check of the compiled sm_90a code of recompose damage (k_recompose.cu; cuobjdump on the object `build()` produces; no GPU
needed). The kernel runs one warp per draw object of the old and the new composition in the first frame after vb_recompose; a
local array or a spill would add a round trip through local memory for each of them, so it must keep everything in registers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_recompose.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


def test_recompose_kernel_has_no_local_memory_or_stack():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_recompose_damage\S*):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert len(found) == 1, f"expected the k_recompose_damage kernel in:\n{res}"
    for fn, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
