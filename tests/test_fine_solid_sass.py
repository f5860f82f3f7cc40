"""Static checks of the compiled k_fine_solid (cuobjdump on the object `build()` produces, no GPU needed), beside the table in
test_compiled_kernels.py.

k_fine_solid paints the tiles that run only FILL / SOLID / COLOR / JUMP. It exists to hold more resident warps than k_fine (20
per SM at 96 registers): its registers let FI_SOLID_MINB CTAs of FI_SOLID_WARPS warps share an SM, and so does its shared
memory (mask LUT, and per warp the command windows and the MSAA state). It has no blend stack and no brush copies: what
stack it has is a few spilled words of the tile loop (at most STACK bytes, against k_fine's 320+), and it holds all three AA
modes."""
import os
import re
import shutil
import subprocess

import pytest

from .test_compiled_kernels import FINE_SRC, SMEM_PER_SM, _key, built  # noqa: F401  (fixture)

OBJ = "k_fine.o"
REGS_PER_SM = 65536
MAX_SMEM_PER_CTA = 227 * 1024  # sm_90: the most dynamic shared memory one CTA may opt in to
STACK = 32

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")


def _macro(name):
    return int(re.search(rf"#define {name} (\d+)", open(FINE_SRC).read()).group(1))


def _smem_bytes(aa, warps):
    """FineSmem<aa>::bytes(warps) of k_fine.cu: the mask LUT, its mbarrier, and per warp WarpIo (+ WarpMs<aa> for MSAA)."""
    lut = {0: 0, 1: 256, 2: 2048}[aa] * 4
    io = 2 * 64 * 4 + 2 * 8
    ms = 0 if aa == 0 else 4 * (256 * (4 if aa == 2 else 2) + 64 + 16 + 4 + 4 + 8 + 32 + 64) + 256
    return lut + 16 + warps * (io + ms)


def test_fine_solid_budget(built):  # noqa: F811
    warps, minb = _macro("FI_SOLID_WARPS"), _macro("FI_SOLID_MINB")
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, OBJ)], capture_output=True, text=True, check=True).stdout
    found = {_key(fn)[1]: tuple(map(int, vals)) for fn, *vals in
             re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res) if _key(fn)[0] == "k_fine_solid"}
    assert sorted(found) == ["Li0E", "Li1E", "Li2E"], f"expected k_fine_solid<0>, <1> and <2> in {OBJ}: {sorted(found)}"
    for args, (reg, stack, shared, local) in found.items():
        assert stack <= STACK and local == 0, f"k_fine_solid<{args}>: {stack} bytes of stack, {local} bytes of local memory"
        assert reg * 32 * warps * minb <= REGS_PER_SM, f"k_fine_solid<{args}>: {reg} registers, fewer than {minb} x {warps} warps per SM"
    for aa in (0, 1, 2):
        smem = _smem_bytes(aa, warps)
        assert smem <= MAX_SMEM_PER_CTA and (smem + 1024) * minb <= SMEM_PER_SM, f"k_fine_solid<{aa}>: {smem} B of shared memory per CTA"


def test_fine_solid_sass(built):  # noqa: F811
    """The lean kernel stages its command windows and mask LUT with bulk copies on mbarriers, like k_fine."""
    full = subprocess.run(["cuobjdump", "-sass", os.path.join(built, OBJ)], capture_output=True, text=True, check=True).stdout
    parts = [p for p in full.split("Function : ")[1:] if "k_fine_solid" in p.split("\n", 1)[0]]
    assert len(parts) == 3, f"{len(parts)} k_fine_solid functions in the disassembly"
    for sass in parts:
        assert "UBLKCP" in sass and "SYNCS" in sass, "k_fine_solid does not stage with bulk copies on mbarriers"
