"""Backgrounds without a GPU: the compiled FI_BG instantiations of k_fine (cuobjdump / nvdisasm on `build()`'s k_fine_bg.o),
and Renderer.set_background's argument checks and the descriptor it passes to vb_set_background (a fake library).

* k_fine_bg.o holds exactly k_fine<AA + FI_DST + FI_BG> for the three AA modes, so k_fine.o keeps exactly its own twelve.
* They keep the guards tests/test_compiled_kernels.py applies to FI_DST: no local-memory instruction on the MSAA fill or the
  CMD_FILL / CMD_SOLID / CMD_COLOR cases, at most 100 128-bit local accesses, the 128-bit surface store, and no more stack than
  k_fine<AA + FI_DST>.
* The background is read with 128-bit global and surface loads, and never through the non-coherent path (LDG ... .CONSTANT):
  the background may be the destination the kernel writes."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from vello_b200.renderer import Renderer, _background_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
FINE_SRC = os.path.join(ROOT, "vello_b200", "csrc", "k_fine.cu")
FI_DST, FI_BG = 32, 64
BG_MODES = tuple(aa + FI_DST + FI_BG for aa in (0, 1, 2))
PRED = r"(@!?U?P\d+\s+)?"

needs_tools = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvdisasm") is None,
                                 reason="CUDA binary utilities not installed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


def _usage(obj):
    """{mode: (registers, stack, local)} of every k_fine<mode> in obj."""
    res = subprocess.run(["cuobjdump", "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    return {int(m): (int(reg), int(stack), int(local))
            for m, reg, stack, local in re.findall(r"Function _Z6k_fineILi(\d+)E\S*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)}


@pytest.fixture(scope="module")
def bg_sass(built, tmp_path_factory):
    """{mode: [(source line of k_fine.cu or None, instruction)]} of the k_fine<mode> in k_fine_bg.o."""
    d = tmp_path_factory.mktemp("cubin_bg")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(built, "k_fine_bg.o")], cwd=d, check=True, capture_output=True)
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
    return out


def _lines(start, end):
    """[first, end) source lines of k_fine.cu from the line holding `start` to the next one holding `end`."""
    src = open(FINE_SRC).read().splitlines()
    a = next(i for i, l in enumerate(src) if start in l) + 1
    return a, next(i for i, l in enumerate(src) if i + 1 > a and end in l) + 1


@needs_tools
def test_bg_object_holds_the_three_instantiations(built, bg_sass):
    assert sorted(bg_sass) == sorted(BG_MODES)
    assert sorted(_usage(os.path.join(built, "k_fine_bg.o"))) == sorted(BG_MODES)
    fine = _usage(os.path.join(built, "k_fine.o"))
    assert not any(m & FI_BG for m in fine), f"k_fine.o holds FI_BG instantiations: {sorted(fine)}"


@needs_tools
@pytest.mark.parametrize("mode", BG_MODES)
def test_bg_hot_path_has_no_local_memory(bg_sass, mode):
    sass = bg_sass[mode]
    assert len(sass) > 5000, f"k_fine<{mode}> not found in the disassembly"
    hot = [_lines("__device__ void fill_path_ms(", "// ---------------- blend.wgsl"), _lines("case VB_CMD_FILL: {", "case VB_CMD_BEGIN_CLIP: {")]
    bad = [(ln, ins) for ln, ins in sass if ln is not None and re.match(PRED + r"(LDL|STL)\b", ins) and any(a <= ln < b for a, b in hot)]
    assert not bad, f"local-memory instructions in k_fine<{mode}>'s fill / colour path: {bad[:5]}"
    wide = [ins for _, ins in sass if re.match(PRED + r"(LDL|STL)\.128\b", ins)]
    assert len(wide) <= 100, f"{len(wide)} 128-bit local loads/stores in k_fine<{mode}>: rgba[] is probably back in local memory"
    stores = [ins for _, ins in sass if re.match(PRED + r"SUST\b", ins)]
    assert any(".128" in ins for ins in stores), f"k_fine<{mode}>: the array store is not two 128-bit surface stores per lane"


@needs_tools
def test_bg_stack_matches_destination_counterpart(built):
    bg, fine = _usage(os.path.join(built, "k_fine_bg.o")), _usage(os.path.join(built, "k_fine.o"))
    for aa in (0, 1, 2):
        assert bg[aa + FI_DST + FI_BG][2] == 0, f"k_fine<{aa + FI_DST + FI_BG}> has local memory"
        assert bg[aa + FI_DST + FI_BG][1] <= fine[aa + FI_DST][1], \
            f"k_fine<{aa} + FI_DST + FI_BG>: {bg[aa + FI_DST + FI_BG][1]} bytes of stack, {fine[aa + FI_DST][1]} for k_fine<{aa} + FI_DST>"


@needs_tools
@pytest.mark.parametrize("mode", BG_MODES)
def test_bg_loads_are_wide_and_coherent(bg_sass, mode):
    """Nothing else in k_fine loads 128 bits from global memory (segments, tile lists and ramps are 64- or 32-bit __ldg loads),
    so the 128-bit global loads are the background's (__ldcg, inlined from the CUDA headers), and the 128-bit surface loads
    are in load_bg_texels."""
    ops = [re.sub("^" + PRED, "", ins).split()[0] for _, ins in bg_sass[mode]]
    wide = [op for op in ops if op.startswith("LDG") and ".128" in op]
    assert wide, f"k_fine<{mode}>: no 128-bit global load"
    assert not [op for op in wide if "CONSTANT" in op], f"k_fine<{mode}> reads the background through the non-coherent path: {sorted(set(wide))}"
    a, b = _lines("__device__ __forceinline__ void load_bg_texels(", "// The background's pixels as fine's")
    surf = [ins for ln, ins in bg_sass[mode] if ln is not None and a <= ln < b and re.match(PRED + r"SULD\S*\.128", ins)]
    assert surf, f"k_fine<{mode}>: no 128-bit surface load in load_bg_texels (lines {a}..{b})"


# ---- Renderer.set_background's arguments (no GPU: a fake library records the descriptor) ----
class FakeLib:
    def __init__(self):
        self.calls = []

    def vb_set_background(self, handle, d):
        self.calls.append(None if d is None else {f: getattr(d._obj, f) for f, _ in type(d._obj)._fields_})
        return 0


class Fake:
    def __init__(self, shape, strides=None, typestr="|u1", data=0x7000_0000):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (data, False), "strides": strides, "version": 3}


@pytest.fixture
def fake():
    r = Renderer._borrowed(FakeLib(), 1, owner=object())
    return r


def test_linear_descriptor(fake):
    fake.set_background(Fake((100, 64, 4)))
    d = fake.lib.calls[-1]
    assert (d["kind"], d["format"], d["ptr"], d["row_pitch_bytes"]) == (0, 0, 0x7000_0000, 256)
    fake.set_background(Fake((100, 64, 4), typestr="<f4"), format="rgba32f", alpha="premultiplied")
    d = fake.lib.calls[-1]
    assert (d["format"], d["row_pitch_bytes"]) == (3 | 0x100, 1024)
    fake.set_background(Fake((10, 8, 4), typestr="<f2"), format="rgba16f")
    assert fake.lib.calls[-1]["format"] == 2 and fake.lib.calls[-1]["row_pitch_bytes"] == 64
    fake.set_background(Fake((10, 8, 4)), format="bgra8")
    assert fake.lib.calls[-1]["format"] == 1


def test_batch_descriptor(fake):
    # [N, H, W, 4], contiguous and as a slice of wider rows (cells H row pitches apart)
    fake.set_background(Fake((5, 100, 64, 4)))
    d = fake.lib.calls[-1]
    assert (d["ptr"], d["row_pitch_bytes"]) == (0x7000_0000, 256)
    fake.set_background(Fake((5, 100, 64, 4), strides=(100 * 512, 512, 4, 1), data=0x7000_0040))
    d = fake.lib.calls[-1]
    assert (d["ptr"], d["row_pitch_bytes"]) == (0x7000_0040, 512)
    assert _background_image(Fake((1, 10, 8, 4), strides=(12345 * 4, 32, 4, 1)), "|u1") == (0x7000_0000, 32)


def test_array_descriptor_and_clear(fake):
    fake.set_background(array=0x1234, format="rgba16f", alpha="premultiplied", origin=(3, 7))
    d = fake.lib.calls[-1]
    assert (d["kind"], d["format"], d["array"], d["x"], d["y"]) == (1, 2 | 0x100, 0x1234, 3, 7)
    fake.set_background()
    assert fake.lib.calls[-1] is None and fake._background is None


@pytest.mark.parametrize("kwargs,exc,msg", [
    (dict(format="rgb8"), ValueError, "set_background: format is one of"),
    (dict(alpha="pre"), ValueError, "set_background: alpha is one of"),
    (dict(target=Fake((4, 4, 4)), array=1), ValueError, "set_background: give a target, an array or neither"),
    (dict(target=Fake((4, 4, 4), typestr="<f4")), ValueError, "a device image is (H, W, 4) uint8"),
    (dict(target=Fake((4, 4, 4)), format="rgba32f"), ValueError, "a device image is (H, W, 4) float32"),
    (dict(target=Fake((2, 4, 4, 4), strides=(4 * 64 + 16, 64, 4, 1))), ValueError, "set_background: the cells of an (N, H, W, 4)"),
    (dict(target=Fake((2, 4, 4, 3))), ValueError, "a device image is (H, W, 4)"),
    (dict(target=Fake((4, 4, 4), strides=(18, 4, 1))), ValueError, "row stride that is a multiple of 4"),
    (dict(target=object()), TypeError, "has no __cuda_array_interface__"),
])
def test_refused(fake, kwargs, exc, msg):
    with pytest.raises(exc, match=re.escape(msg)):
        fake.set_background(**kwargs)
    assert fake.lib.calls == []


@pytest.mark.parametrize("target,size,cells,ok", [
    (Fake((100, 64, 4)), (64, 100), 1, True),
    (Fake((100, 64, 4)), (64, 101), 1, False),   # a row short
    (Fake((100, 64, 4)), (65, 100), 1, False),   # a column short
    (Fake((100, 64, 4)), (64, 50), 2, True),     # a tall image holds two cells of 50 rows
    (Fake((100, 64, 4)), (64, 50), 3, False),
    (Fake((3, 50, 64, 4)), (64, 50), 3, True),
    (Fake((3, 50, 64, 4)), (64, 50), 4, False),  # a cell short
    (Fake((3, 60, 64, 4)), (64, 50), 3, False),  # cells 60 rows apart, read 50 rows apart
    (Fake((3, 60, 64, 4)), (64, 50), 1, True),
])
def test_background_shape_covers_the_frame(fake, target, size, cells, ok):
    from vello_b200.config import AA_MSAA16, RenderParams
    from vello_b200.encoding import BLACK
    fake.set_background(target)
    p = RenderParams(BLACK, size[0], size[1], AA_MSAA16)
    if ok:
        fake._check_background(p, cells)
    else:
        with pytest.raises(ValueError, match="set_background: a .* background cannot hold"):
            fake._check_background(p, cells)
    fake.set_background(array=5)
    fake._check_background(p, cells)  # an array's extent is the library's to check
