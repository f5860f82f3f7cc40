"""Static checks of the damage-tracking instantiations of coarse and fine (cuobjdump / nvdisasm on the objects `build()`
produces; no GPU needed), the same guards tests/test_sass_guards.py keeps on the default ones:

* `k_fine<2 + FI_DMG>` (MSAA16, damaged tiles only) keeps the lane's pixels in registers: no local-memory instruction in the
  MSAA fill or in the interpreter's CMD_FILL / CMD_SOLID / CMD_COLOR cases, and only the known few 128-bit local accesses.
* `k_coarse<true>` does not spill (the default one does not either)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
SRC = os.path.join(ROOT, "vello_b200", "csrc", "k_fine.cu")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvdisasm") is None, reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


def _sass_by_line(built, tmp_path_factory, obj, fn_mark, src_name):
    """[(source line of src_name or None, instruction text)] of the function whose mangled name contains fn_mark."""
    d = tmp_path_factory.mktemp("cubin")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(built, obj)], cwd=d, check=True, capture_output=True)
    cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
    assert cubins, f"no cubin in {obj}"
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(d, cubins[0])], capture_output=True, text=True, check=True).stdout
    out, cur, in_fn = [], None, False
    for ln in dis.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", ln)
        if m:
            in_fn = fn_mark in m.group(1)
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = int(m.group(2)) if m.group(1).endswith(src_name) else None
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
        if m and in_fn:
            out.append((cur, m.group(1).strip()))
    return out


def _line_range(pattern_start, pattern_end):
    src = open(SRC).read().splitlines()
    a = next(i for i, l in enumerate(src) if pattern_start in l) + 1
    b = next(i for i, l in enumerate(src) if i + 1 > a and pattern_end in l) + 1
    return a, b


def test_tracked_fine_hot_path_has_no_local_memory(built, tmp_path_factory):
    sass = _sass_by_line(built, tmp_path_factory, "k_fine.o", "k_fineILi18E", "k_fine.cu")
    assert len(sass) > 5000, "k_fine<2 + FI_DMG> not found in the disassembly"
    fill = _line_range("__device__ void fill_path_ms(", "// ---------------- blend.wgsl")
    interp = _line_range("case VB_CMD_FILL: {", "case VB_CMD_BEGIN_CLIP: {")
    bad = [(ln, ins) for ln, ins in sass if ln is not None and re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\b", ins)
           and (fill[0] <= ln < fill[1] or interp[0] <= ln < interp[1])]
    assert not bad, f"local-memory instructions in the tracked fine's fill / colour path: {bad[:5]}"
    wide = [ins for _, ins in sass if re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\.128\b", ins)]
    assert len(wide) <= 100, f"{len(wide)} 128-bit local loads/stores in k_fine<2 + FI_DMG>: rgba[] is probably back in local memory"


def test_tracked_coarse_does_not_spill(built):
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, "k_coarse.o")], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_coarse\S*):\s*\n\s*REG:\d+ STACK:(\d+)", res)
    assert len(found) == 2, f"expected k_coarse<false> and k_coarse<true> in:\n{res}"
    for fn, stack in found:
        assert int(stack) == 0, f"{fn}: {stack} bytes of stack"
