"""Static checks of fine's registered-destination instantiations (k_fine<2 + FI_DST> and k_fine<2 + FI_DST + FI_DMG>, MSAA16
into a BGRA8 buffer or a CUDA array; cuobjdump / nvdisasm on the objects `build()` produces, no GPU needed). They differ from
their counterparts only at the store, so they keep the counterparts' guards: no local-memory instruction in the MSAA fill or in
the interpreter's CMD_FILL / CMD_SOLID / CMD_COLOR cases, no more 128-bit local accesses than tests/test_damage_sass.py
allows, and no more stack (spill slots included) than the counterpart."""
import os
import re
import shutil
import subprocess

import pytest

from .test_damage_sass import BUILD, _line_range, _sass_by_line

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvdisasm") is None, reason="CUDA binary utilities not installed")

FI_DMG, FI_DST = 16, 32


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@pytest.mark.parametrize("mode", [2 + FI_DST, 2 + FI_DST + FI_DMG])
def test_destination_fine_hot_path_has_no_local_memory(built, tmp_path_factory, mode):
    sass = _sass_by_line(built, tmp_path_factory, "k_fine.o", f"k_fineILi{mode}E", "k_fine.cu")
    assert len(sass) > 5000, f"k_fine<{mode}> not found in the disassembly"
    fill = _line_range("__device__ void fill_path_ms(", "// ---------------- blend.wgsl")
    interp = _line_range("case VB_CMD_FILL: {", "case VB_CMD_BEGIN_CLIP: {")
    bad = [(ln, ins) for ln, ins in sass if ln is not None and re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\b", ins)
           and (fill[0] <= ln < fill[1] or interp[0] <= ln < interp[1])]
    assert not bad, f"local-memory instructions in k_fine<{mode}>'s fill / colour path: {bad[:5]}"
    wide = [ins for _, ins in sass if re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\.128\b", ins)]
    assert len(wide) <= 100, f"{len(wide)} 128-bit local loads/stores in k_fine<{mode}>: rgba[] is probably back in local memory"
    stores = [ins for _, ins in sass if re.match(r"(@!?U?P\d+\s+)?SUST\b", ins)]
    assert any(".128" in ins for ins in stores), "the array store is not two 128-bit surface stores per lane"


def test_destination_fine_stack_matches_counterpart(built):
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, "k_fine.o")], capture_output=True, text=True, check=True).stdout
    stack = {int(m): int(s) for m, s in re.findall(r"Function \S*k_fineILi(\d+)E\S*:\s*\n\s*REG:\d+ STACK:(\d+)", res)}
    for base in (0, 1, 2, FI_DMG, 1 + FI_DMG, 2 + FI_DMG):
        assert base + FI_DST in stack, f"k_fine<{base} + FI_DST> missing from k_fine.o"
        assert stack[base + FI_DST] <= stack[base], f"k_fine<{base} + FI_DST>: {stack[base + FI_DST]} bytes of stack, {stack[base]} without"

