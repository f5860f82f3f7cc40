"""Static check of the compiled sm_90a code of the path tag scan (cuobjdump on the object `build()` produces; no GPU needed).
`k_pathtag_scan` keeps each thread's tag words and monoids in registers and stages the partition's monoids in shared memory,
so that its stores are whole 16-byte words; a spill or a local array would put them back in memory, per thread."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_pathtag.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def usage():
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", OBJ], capture_output=True, text=True, check=True).stdout
    return {fn: (int(reg), int(stack), int(shared))
            for fn, reg, stack, shared in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)}


def _scan(usage):
    found = [v for fn, v in usage.items() if "k_pathtag_scan" in fn]
    assert len(found) == 1, f"k_pathtag_scan not found in {sorted(usage)}"
    return found[0]


def test_pathtag_scan_has_no_local_memory(usage):
    _, stack, _ = _scan(usage)
    assert stack == 0, f"k_pathtag_scan uses {stack} bytes of stack (spills or a local array)"


@pytest.fixture(scope="module")
def sass(usage):
    """The object's SASS: k_pathtag_scan is its only kernel."""
    assert len(usage) == 1, f"k_pathtag.o holds more than the scan: {sorted(usage)}"
    return subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout


def test_pathtag_scan_has_no_local_accesses(sass):
    assert not re.search(r"\b(LDL|STL)\b", sass), "k_pathtag_scan loads or stores local memory"


def test_pathtag_scan_stores_16_byte_words(sass):
    """The monoids leave the CTA as 128-bit stores, and the tag words arrive as 128-bit loads."""
    assert re.search(r"\bSTG\.E\.128\b", sass), "no 128-bit global store in k_pathtag_scan"
    assert re.search(r"\bLDG\.E\.128", sass), "no 128-bit global load in k_pathtag_scan"
