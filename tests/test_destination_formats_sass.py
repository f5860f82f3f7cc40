"""The stores of float and premultiplied destinations in the compiled k_fine (cuobjdump / nvdisasm on `build()`'s k_fine.o,
no GPU needed):

* the default instantiations (k_fine<AA>, k_fine<AA + FI_DMG>) store exactly as before destinations had formats: 32-bit and
  128-bit global stores, no other width and no surface store;
* the FI_DST instantiations store float texels with 128-bit global and surface stores (two RGBA16F texels or one RGBA32F
  texel each), beside the 64-bit per-texel ones of a partial tile or an odd column;
* store_float, which every FI_DST instantiation inlines, keeps the texels in registers: no local store and no wide local
  load. (Like the 8-bit store, it may reload a word or two of the tile loop's state that ptxas spilled.)"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FINE_SRC = os.path.join(ROOT, "vello_b200", "csrc", "k_fine.cu")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvdisasm") is None,
                                reason="CUDA binary utilities not installed")

FI_DMG, FI_DST = 16, 32
PRED = r"(@!?U?P\d+\s+)?"


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    """{mode: [(source line of k_fine.cu or None, instruction)]} of every k_fine<mode>."""
    import __graft_entry__ as g
    g.build()
    d = tmp_path_factory.mktemp("cubin")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(ROOT, "vello_b200", "csrc", "build", "k_fine.o")], cwd=d, check=True,
                   capture_output=True)
    cubin = next(f for f in os.listdir(d) if f.endswith(".cubin"))
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(d, cubin)], capture_output=True, text=True, check=True).stdout
    out, fn, cur = {}, None, None
    for ln in dis.splitlines():
        m = re.match(r"\s*\.text\._Z6k_fineILi(\d+)E\S*:", ln)
        if m:
            fn = out.setdefault(int(m.group(1)), [])
            continue
        if re.match(r"\s*\.text\.", ln):
            fn = None
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = int(m.group(2)) if m.group(1).endswith("k_fine.cu") else None
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
        if m and fn is not None:
            fn.append((cur, m.group(1).strip()))
    assert sorted(out) == sorted(aa + f for aa in (0, 1, 2) for f in (0, FI_DMG, FI_DST, FI_DST + FI_DMG)), sorted(out)
    return out


def stores(ins_list):
    """The store opcodes (STG / SUST with their modifiers) of a function, as a set."""
    ops = (re.sub("^" + PRED, "", ins).split()[0] for _, ins in ins_list)
    return {op for op in ops if op.startswith(("STG", "SUST"))}


@pytest.mark.parametrize("mode", [0, 1, 2, FI_DMG, 1 + FI_DMG, 2 + FI_DMG])
def test_default_stores_unchanged(sass, mode):
    assert stores(sass[mode]) == {"STG.E", "STG.E.128"}, f"k_fine<{mode}> stores {sorted(stores(sass[mode]))}"


@pytest.mark.parametrize("mode", [aa + f for aa in (0, 1, 2) for f in (FI_DST, FI_DST + FI_DMG)])
def test_destination_stores_are_wide(sass, mode):
    s = stores(sass[mode])
    assert "STG.E.128" in s and "STG.E.64" in s, f"k_fine<{mode}> global stores: {sorted(s)}"
    assert any(op.startswith("SUST") and ".128" in op for op in s), f"k_fine<{mode}> has no 128-bit surface store: {sorted(s)}"
    assert any(op.startswith("SUST") and ".64" in op for op in s), f"k_fine<{mode}> has no 64-bit surface store: {sorted(s)}"


def test_float_store_keeps_texels_in_registers(sass):
    src = open(FINE_SRC).read().splitlines()
    a = next(i for i, l in enumerate(src) if "__device__ __forceinline__ void store_float(" in l) + 1
    b = next(i for i, l in enumerate(src) if i + 1 > a and l.startswith("}")) + 1
    for mode, ins_list in sass.items():
        if not mode & FI_DST:
            continue
        lines = [ins for ln, ins in ins_list if ln is not None and a <= ln <= b]
        assert len(lines) > 20, f"k_fine<{mode}>: store_float not found at lines {a}..{b}"
        bad = [ins for ins in lines if re.match(PRED + r"(STL\b|LDL\.(64|128)\b)", ins)]
        assert not bad, f"k_fine<{mode}>: texels through local memory in store_float: {bad[:5]}"
