"""Static checks of the compiled sm_90a code: cuobjdump / nvdisasm on the objects `build()` produces, no GPU needed.

* Each kernel in BUDGETS keeps everything in registers (no stack, no local memory) and, where it has one, within its
  register and shared-memory budget. These kernels touch every tag word, transform, draw object or line of a frame; a local
  array or a spill would add a round trip through local memory for each of them.
* `k_fine` keeps the lane's pixels in registers: no local-memory instruction may be attributed to the MSAA fill
  (`fill_path_ms`) or to the interpreter's CMD_FILL / CMD_SOLID / CMD_COLOR cases. Four `#pragma unroll 1` brush loops once
  kept `rgba[]` / `area[]` in local memory, which made local traffic the kernel's top stall. The damage-tracking
  (FI_DMG) and registered-destination (FI_DST) instantiations keep the same guard, and FI_DST, which differs only at the
  store, uses no more stack than its counterpart.
* `k_fine` stages its mask LUT and command windows with bulk copies signalled on mbarriers (SASS UBLKCP / SYNCS), the
  Hopper (sm_90a) path DESIGN.md claims.
* No kernel of the pipeline spills more than a few registers."""
import fnmatch
import os
import re
import shutil
import subprocess
from collections import namedtuple

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vello_b200", "csrc", "build")
FINE_SRC = os.path.join(ROOT, "vello_b200", "csrc", "k_fine.cu")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")
needs_nvdisasm = pytest.mark.skipif(shutil.which("nvdisasm") is None, reason="nvdisasm not installed")

FI_DMG, FI_DST = 16, 32
HOT_MODES = (2, 2 + FI_DMG, 2 + FI_DST, 2 + FI_DST + FI_DMG)  # MSAA16: default, damage-tracked, destination, both
PRED = r"(@!?U?P\d+\s+)?"
REGS_PER_SM = 65536
SMEM_PER_SM = 228 * 1024  # sm_90: 228 KB of shared memory per SM (cuobjdump counts the 1 KB each CTA reserves)

Usage = namedtuple("Usage", "reg stack shared local")
# Each row: `obj` holds exactly `count` functions whose base name matches the pattern `kernel`, none of which uses stack or
# local memory. `regs` = (CTAs, threads): the registers let that many CTAs of that many threads share an SM. `smem` = CTAs:
# the shared memory lets that many CTAs share an SM.
Budget = namedtuple("Budget", "obj kernel count regs smem", defaults=(None, None))
BUDGETS = [
    Budget("k_pathtag.o", "k_pathtag_scan", 1),
    # the lean tag pass and the emit pass exist to run at a higher occupancy than the general k_flatten (128 registers):
    # FL_LEAN_MINB CTAs of FL_THREADS
    Budget("k_flatten.o", "k_flatten_lean", 1, regs=(4, 256)),
    Budget("k_flatten.o", "k_flatten_emit", 1, regs=(4, 256), smem=4),
    Budget("k_compose.o", "k_compose_streams", 1),
    Budget("k_compose.o", "k_instance_transforms", 1),
    # the bound draw data's per-frame pass and bind-time slot walk (k_colors.cu); the device resolve and the bound ramps
    Budget("k_colors.o", "k_draw_data", 1),
    Budget("k_colors.o", "k_draw_data_slots", 1),
    Budget("k_resolve.o", "k_resolve_finish", 1),
    Budget("k_resolve.o", "k_make_ramps", 1),
    Budget("k_resolve.o", "k_bound_ramps", 1),
    Budget("k_damage.o", "k_damage*", 5),
    Budget("k_recompose.o", "k_recompose_damage", 1),
    Budget("k_upload_diff.o", "k_upload_*", 3),
    Budget("k_coarse.o", "k_coarse", 2),  # <false> and <true> (damage-tracked)
]


def _key(mangled):
    """(base name, template arguments or None) of an Itanium-mangled function: `_Z6k_fineILi18EEv8VbConfig...` gives
    ("k_fine", "Li18E"). The name is read by its length prefix, so k_flatten never matches k_flatten_lean."""
    m = re.match(r"_Z(\d+)", mangled)
    i = m.end() + int(m.group(1))
    name, rest = mangled[m.end():i], mangled[i:]
    if not rest.startswith("I"):
        return name, None
    depth, j = 0, 0
    while True:
        if rest[j].isdigit():  # a length-prefixed name
            n = re.match(r"\d+", rest[j:]).group()
            j += len(n) + int(n)
        elif rest[j] == "L":  # a literal, L<type><value>E
            j = rest.index("E", j) + 1
        else:
            depth += (rest[j] in "IN") - (rest[j] == "E")
            j += 1
            if depth == 0:
                return name, rest[1:j - 1]


def _label(key):
    name, args = key
    return f"{name}<{args}>" if args else name


def _fine_mode(key):
    """MODE of k_fine<MODE> (AA + FI_DMG + FI_DST), None for any other function."""
    name, args = key
    return int(re.fullmatch(r"Li(\d+)E", args).group(1)) if name == "k_fine" else None


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return BUILD


@pytest.fixture(scope="module")
def usage(built):
    """{object: {(base name, template arguments): Usage}} of every k_*.o, from cuobjdump -res-usage."""
    out = {}
    for obj in sorted(f for f in os.listdir(built) if f.startswith("k_") and f.endswith(".o")):
        res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(built, obj)], capture_output=True, text=True, check=True).stdout
        fns = out[obj] = {}
        for fn, *vals in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res):
            assert _key(fn) not in fns, f"{fn} appears twice in {obj}"
            fns[_key(fn)] = Usage(*map(int, vals))
        assert len(fns) == res.count("Function "), f"unparsed resource usage in {obj}:\n{res}"
    return out


@pytest.fixture(scope="module")
def fine_sass(built, tmp_path_factory):
    """{mode: [(source line of k_fine.cu or None, instruction text)]} of k_fine<mode> for HOT_MODES, from nvdisasm's line
    info."""
    d = tmp_path_factory.mktemp("cubin")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(built, "k_fine.o")], cwd=d, check=True, capture_output=True)
    cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
    assert cubins, "no cubin in k_fine.o"
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(d, cubins[0])], capture_output=True, text=True, check=True).stdout
    out, cur, fn = {mode: [] for mode in HOT_MODES}, None, None
    for ln in dis.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", ln)
        if m:
            fn = out.get(_fine_mode(_key(m.group(1))))
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = int(m.group(2)) if m.group(1).endswith("k_fine.cu") else None
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
        if m and fn is not None:
            fn.append((cur, m.group(1).strip()))
    return out


@pytest.fixture(scope="module")
def hot_lines():
    """[first, end) source lines of k_fine.cu's MSAA fill and of the interpreter's CMD_FILL / CMD_SOLID / CMD_COLOR cases."""
    src = open(FINE_SRC).read().splitlines()

    def line_range(start, end):
        a = next(i for i, l in enumerate(src) if start in l) + 1
        return a, next(i for i, l in enumerate(src) if i + 1 > a and end in l) + 1
    return [line_range("__device__ void fill_path_ms(", "// ---------------- blend.wgsl"),
            line_range("case VB_CMD_FILL: {", "case VB_CMD_BEGIN_CLIP: {")]


@pytest.mark.parametrize("row", BUDGETS, ids=lambda row: row.kernel.rstrip("*_"))
def test_kernel_budget(usage, row):
    found = {key: u for key, u in usage[row.obj].items() if fnmatch.fnmatchcase(key[0], row.kernel)}
    assert len(found) == row.count, f"expected {row.count} {row.kernel} in {row.obj}, found {sorted(map(_label, found))}"
    for key, u in found.items():
        assert u.stack == 0 and u.local == 0, f"{_label(key)}: {u.stack} bytes of stack, {u.local} bytes of local memory"
        if row.regs:
            ctas, threads = row.regs
            assert u.reg * threads * ctas <= REGS_PER_SM, f"{_label(key)}: {u.reg} registers, fewer than {ctas} CTAs per SM"
        if row.smem:
            assert u.shared * row.smem <= SMEM_PER_SM, f"{_label(key)}: {u.shared} B of shared memory, fewer than {row.smem} CTAs per SM"


@needs_nvdisasm
@pytest.mark.parametrize("mode", HOT_MODES)
def test_fine_hot_path_has_no_local_memory(fine_sass, hot_lines, mode):
    sass = fine_sass[mode]
    assert len(sass) > 5000, f"k_fine<{mode}> not found in the disassembly"
    bad = [(ln, ins) for ln, ins in sass if ln is not None and re.match(PRED + r"(LDL|STL)\b", ins)
           and any(a <= ln < b for a, b in hot_lines)]
    assert not bad, f"local-memory instructions in k_fine<{mode}>'s fill / colour path: {bad[:5]}"
    # the helpers inlined into CMD_COLOR (over, rg_scale) carry their own line numbers: no 128-bit local traffic anywhere
    # except the brushes' pixel copies and the blend stack (a bounded, known set)
    wide = [ins for _, ins in sass if re.match(PRED + r"(LDL|STL)\.128\b", ins)]
    assert len(wide) <= 100, f"{len(wide)} 128-bit local loads/stores in k_fine<{mode}>: rgba[] is probably back in local memory"
    if mode & FI_DST:
        stores = [ins for _, ins in sass if re.match(PRED + r"SUST\b", ins)]
        assert any(".128" in ins for ins in stores), f"k_fine<{mode}>: the array store is not two 128-bit surface stores per lane"


@needs_nvdisasm
def test_fine_uses_bulk_copies_and_mbarriers(fine_sass):
    ops = {re.sub("^" + PRED, "", ins).split()[0].split(".")[0] for _, ins in fine_sass[2]}
    assert "UBLKCP" in ops, "no bulk copy (cp.async.bulk) in k_fine<2>"
    assert "SYNCS" in ops, "no mbarrier operation in k_fine<2>"


def test_destination_fine_stack_matches_counterpart(usage):
    stack = {_fine_mode(key): u.stack for key, u in usage["k_fine.o"].items()}
    for base in (0, 1, 2, FI_DMG, 1 + FI_DMG, 2 + FI_DMG):
        assert base in stack and base + FI_DST in stack, f"k_fine<{base}> or k_fine<{base} + FI_DST> missing from k_fine.o"
        assert stack[base + FI_DST] <= stack[base], f"k_fine<{base} + FI_DST>: {stack[base + FI_DST]} bytes of stack, {stack[base]} without"


def test_pathtag_scan_sass(usage, built):
    """The scan keeps each thread's tag words and monoids in registers and stages the partition's monoids in shared memory:
    the tag words arrive and the monoids leave as 128-bit global accesses, and nothing goes through local memory."""
    fns = sorted(map(_label, usage["k_pathtag.o"]))
    assert fns == ["k_pathtag_scan"], f"k_pathtag.o holds more than the scan: {fns}"
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(built, "k_pathtag.o")], capture_output=True, text=True, check=True).stdout
    assert not re.search(r"\b(LDL|STL)\b", sass), "k_pathtag_scan loads or stores local memory"
    assert re.search(r"\bSTG\.E\.128\b", sass), "no 128-bit global store in k_pathtag_scan"
    assert re.search(r"\bLDG\.E\.128", sass), "no 128-bit global load in k_pathtag_scan"


def test_kernels_do_not_spill(usage):
    """The stack is the blend stack / brush copies in fine, the dynamically indexed peer table (a by-value kernel argument) in
    the exchange kernels, and a few words elsewhere."""
    for obj, fns in usage.items():
        for key, u in fns.items():
            limit = 512 if key[0].startswith("k_fine") else 128 if obj == "k_exchange.o" else 64
            assert u.stack <= limit, f"{_label(key)} in {obj}: {u.stack} bytes of stack"
