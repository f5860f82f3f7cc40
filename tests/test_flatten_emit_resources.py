"""Static check of the compiled sm_90a code of `k_flatten_emit` (cuobjdump on the object `build()` produces; no GPU needed).
It runs every lean partition of the frame again, after the scan, to write their lines straight to their final positions,
so it is held to the same budget as `k_flatten_lean`: four 256-thread CTAs per SM and everything in registers."""
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
SMEM_PER_SM = 228 * 1024  # sm_90: 228 KB of shared memory per SM (cuobjdump counts the 1 KB each CTA reserves)


@pytest.fixture(scope="module")
def usage():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_flatten_emit\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)
    assert len(found) == 1, f"k_flatten_emit not found once in {res}"
    _, reg, stack, shared = found[0]
    return int(reg), int(stack), int(shared)


def test_emit_pass_has_no_local_memory(usage):
    _, stack, _ = usage
    assert stack == 0, f"k_flatten_emit uses {stack} bytes of stack (spills or a local array)"


def test_emit_pass_register_budget(usage):
    reg, _, _ = usage
    assert reg * THREADS * MIN_CTAS_PER_SM <= REGS_PER_SM, f"k_flatten_emit: {reg} registers, fewer than {MIN_CTAS_PER_SM} CTAs per SM"


def test_emit_pass_shared_memory_budget(usage):
    _, _, shared = usage
    assert shared * MIN_CTAS_PER_SM <= SMEM_PER_SM, f"k_flatten_emit: {shared} B of shared memory, fewer than {MIN_CTAS_PER_SM} CTAs per SM"
