"""Static check of the compiled sm_90a code of the flatten tag pass (cuobjdump on the object `build()` produces; no GPU
needed). `k_flatten_lean` runs most partitions of a map-like scene; it exists to run at a higher occupancy than the general
`k_flatten` (128 registers), so it must stay within its register budget and keep everything in registers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_flatten.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")

THREADS = 256        # FL_THREADS
MIN_CTAS_PER_SM = 4  # FL_LEAN_MINB
REGS_PER_SM = 65536


@pytest.fixture(scope="module")
def usage():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    return {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res)}


def _lean(usage):
    found = [v for fn, v in usage.items() if "k_flatten_lean" in fn]
    assert len(found) == 1, f"k_flatten_lean not found in {sorted(usage)}"
    return found[0]


def test_lean_tag_pass_has_no_local_memory(usage):
    _, stack = _lean(usage)
    assert stack == 0, f"k_flatten_lean uses {stack} bytes of stack (spills or a local array)"


def test_lean_tag_pass_register_budget(usage):
    reg, _ = _lean(usage)
    assert reg * THREADS * MIN_CTAS_PER_SM <= REGS_PER_SM, f"k_flatten_lean: {reg} registers, fewer than {MIN_CTAS_PER_SM} CTAs per SM"
