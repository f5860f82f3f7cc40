"""Static checks of the compiled sm_90a code (cuobjdump / nvdisasm on the objects `build()` produces; no GPU needed).

* `k_fine` must keep the lane's pixels in registers: no local-memory instruction may be attributed to the MSAA fill
  (`fill_path_ms`) or to the interpreter's CMD_FILL / CMD_SOLID / CMD_COLOR cases. Four `#pragma unroll 1` brush loops
  once kept `rgba[]` / `area[]` in local memory, which made local traffic the kernel's top stall.
* `k_fine` stages its mask LUT and command windows with bulk copies signalled on mbarriers (SASS UBLKCP / SYNCS), the
  Hopper (sm_90a) path DESIGN.md claims.
* no kernel of the pipeline spills more than a few registers."""
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


def _fine_sass_by_line(built, tmp_path_factory):
    """[(source line of k_fine.cu or None, instruction text)] of k_fine<2>, from nvdisasm's line info."""
    d = tmp_path_factory.mktemp("cubin")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(built, "k_fine.o")], cwd=d, check=True, capture_output=True)
    cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
    assert cubins, "no cubin in k_fine.o"
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(d, cubins[0])], capture_output=True, text=True, check=True).stdout
    out, cur, in_fn = [], None, False
    for ln in dis.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", ln)
        if m:
            in_fn = "k_fineILi2E" in m.group(1)
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = int(m.group(2)) if m.group(1).endswith("k_fine.cu") else None
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
        if m and in_fn:
            out.append((cur, m.group(1).strip()))
    assert len(out) > 5000, "k_fine<2> not found in the disassembly"
    return out


def _line_range(pattern_start, pattern_end):
    src = open(SRC).read().splitlines()
    a = next(i for i, l in enumerate(src) if pattern_start in l) + 1
    b = next(i for i, l in enumerate(src) if i + 1 > a and pattern_end in l) + 1
    return a, b


def test_fine_hot_path_has_no_local_memory(built, tmp_path_factory):
    sass = _fine_sass_by_line(built, tmp_path_factory)
    fill = _line_range("__device__ void fill_path_ms(", "// ---------------- blend.wgsl")
    interp = _line_range("case VB_CMD_FILL: {", "case VB_CMD_BEGIN_CLIP: {")
    bad = [(ln, ins) for ln, ins in sass if ln is not None and re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\b", ins)
           and (fill[0] <= ln < fill[1] or interp[0] <= ln < interp[1])]
    assert not bad, f"local-memory instructions in fine's fill / colour path: {bad[:5]}"
    # the helpers inlined into CMD_COLOR (over, rg_scale) carry their own line numbers: no 128-bit local traffic anywhere
    # except the brushes' pixel copies and the blend stack (a bounded, known set)
    wide = [ins for _, ins in sass if re.match(r"(@!?U?P\d+\s+)?(LDL|STL)\.128\b", ins)]
    assert len(wide) <= 100, f"{len(wide)} 128-bit local loads/stores in k_fine<2>: rgba[] is probably back in local memory"


def test_fine_uses_bulk_copies_and_mbarriers(built, tmp_path_factory):
    ops = {re.sub(r"^(@!?U?P\d+\s+)", "", ins).split()[0].split(".")[0] for _, ins in _fine_sass_by_line(built, tmp_path_factory)}
    assert "UBLKCP" in ops, "no bulk copy (cp.async.bulk) in k_fine<2>"
    assert "SYNCS" in ops, "no mbarrier operation in k_fine<2>"


def test_kernels_do_not_spill(built):
    """Resource usage of every kernel: the stack is the blend stack / brush copies in fine, the dynamically indexed peer
    table (a by-value kernel argument) in the exchange kernels, and a few words elsewhere."""
    limits = {"k_fine": 512}
    for obj in sorted(os.listdir(built)):
        if not obj.startswith("k_") or not obj.endswith(".o"):
            continue
        res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, obj)], capture_output=True, text=True, check=True).stdout
        for fn, stack in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", res):
            lim = next((v for k, v in limits.items() if k in fn), 128 if obj == "k_exchange.o" else 64)
            assert int(stack) <= lim, f"{fn} in {obj}: {stack} bytes of stack"
