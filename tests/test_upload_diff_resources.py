"""Static check of the compiled sm_90a code of the upload diff (k_upload_diff.cu; cuobjdump on the object `build()` produces; no
GPU needed). Its kernels run in the first frame after a diffed upload, one thread per draw object and one warp per pair of draw
objects; a local array or a spill would add a round trip through local memory for each of them."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_upload_diff.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


def test_upload_diff_kernels_have_no_local_memory_or_stack():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_upload_\S*):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert len(found) == 3, f"expected the three k_upload_* kernels in:\n{res}"
    for fn, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
