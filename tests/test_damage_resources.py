"""Static check of the compiled sm_90a code of damage tracking (k_damage.cu; cuobjdump on the object `build()` produces; no GPU
needed). Its kernels run in every tracked frame, one thread per transform and one warp per draw object; a local array or a spill
would add a round trip through local memory for each of them, so they must keep everything in registers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_damage.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


def test_damage_kernels_have_no_local_memory_or_stack():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_damage\S*):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert len(found) == 5, f"expected the five k_damage kernels in:\n{res}"
    for fn, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, f"{fn}: {stack} bytes of stack, {local} bytes of local memory"
