"""coarse's emission walk (k_coarse.cu) at its edges: every tile's command stream must be the oracle's for a tile with 1 to
300 covered draws (more than one 256-draw chunk; about 40 draws fill a PTCL chunk, so the larger stacks jump to new chunks),
a zero-coverage clip opened before and closed after long runs of draws, and in the damage-tracked and batched
instantiations. Also pins the kernel's register and shared-memory budget in the compiled object (no GPU needed), so that
a change to the walk keeps four CTAs per SM and leaves room for k_path_tiling beside it."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_CLIP, Color, Scene, resolve
from vello_b200.shapes import Affine, BezPath, Circle, Rect

from . import parity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 16  # a run length the tests step around (W - 1, W, W + 1, 2 W, ...)
SIZE = 64  # 4x4 tiles; the stacks below cover tile (1, 1), pixels 16..32


def colour(k, a=90):
    return Color.from_rgba8((37 * k) % 256, (91 * k) % 256, (53 * k + 100) % 256, a)


def stack(s, n, k0=0):
    """n translucent draws that cover tile (1, 1) only, alternately with segments and as a full-tile solid."""
    for k in range(k0, k0 + n):
        shape = Circle(24.0 + (k % 3), 24.0 + (k % 5) * 0.5, 5.0) if k % 2 else Rect(16.0, 16.0, 32.0, 32.0)
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, colour(k), None, shape)


def stacked(n):
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(20, 40, 60, 255), None, Circle(30.0, 30.0, 28.0))  # under it all
    stack(s, n)
    return s


def zero_clip(before, inside, after):
    """`before` draws, then a clip whose path leaves tile (1, 1) uncovered though its box holds it (two small circles at
    opposite corners), `inside` draws under it (all skipped on that tile), the clip's end, then `after` draws."""
    s = Scene()
    stack(s, before)
    clip = BezPath()
    for cx, cy in ((6.0, 6.0), (58.0, 58.0)):
        clip.move_to(cx + 4.0, cy)
        clip.line_to(cx, cy + 4.0)
        clip.line_to(cx - 4.0, cy)
        clip.line_to(cx, cy - 4.0)
        clip.close_path()
    s.push_layer(FILL_EVEN_ODD, MIX_CLIP, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, clip)
    stack(s, inside, before)
    s.pop_layer()
    stack(s, after, before + inside)
    return s


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def check(renderer, oracle, scene, aa=AA_MSAA16, size=SIZE):
    packed = resolve(scene.encoding)
    img = renderer.render_to_texture(packed, RenderParams(BLACK, size, size, aa))
    ref = oracle.render(packed, size, size, BLACK.premul_rgba8_u32(), aa)
    parity.compare_all(renderer, oracle, packed.layout, size, size, check_ptcl_tiles=range((size // 16) ** 2))
    d = np.abs(img.astype(np.int32) - ref.astype(np.int32))
    assert d.max() <= (1 if aa == AA_AREA else 0), f"max diff {d.max()}"
    return img


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, W - 1, W, W + 1, 2 * W, 2 * W + 1, 255, 256, 257, 300])
def test_covered_run_lengths(renderer, oracle, n):
    """n covered draws on one tile (more than 256 spans two chunks); the larger stacks jump to new PTCL chunks."""
    check(renderer, oracle, stacked(n))


@pytest.mark.gpu
@pytest.mark.parametrize("before,inside,after", [(0, 2 * W, 3), (W - 1, W + 2, W), (W - 1, 300, 1), (3, 0, W)])
def test_zero_coverage_clip_over_long_runs(renderer, oracle, before, inside, after):
    check(renderer, oracle, zero_clip(before, inside, after))


@pytest.mark.gpu
def test_area_aa(renderer, oracle):
    check(renderer, oracle, stacked(2 * W + 1), aa=AA_AREA)


@pytest.mark.gpu
def test_batched_cells(renderer):
    """Each cell of a batch equals the scene rendered alone."""
    ss = [stacked(n) for n in (W, W + 1, 300)] + [zero_clip(W - 1, W + 2, W)]
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    frames = renderer.render_batch(ss, p)
    for i, s in enumerate(ss):
        assert np.array_equal(frames[i], renderer.render_to_texture(resolve(s.encoding), p)), f"cell {i}"


@pytest.mark.gpu
def test_damage_tracked_frame(renderer):
    """An incremental frame (k_coarse<true>) repaints the damaged tile exactly as a full frame does."""
    import torch
    packed = resolve(stacked(2 * W + 1).encoding)
    r = renderer
    r.upload(packed)
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    dst = torch.zeros((SIZE, SIZE, 4), dtype=torch.uint8, device="cuda")
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        full = dst.cpu().numpy()
        dst.fill_(7)
        torch.cuda.synchronize()
        r.add_damage([[16, 16, 32, 32]])
        r.render_resident(p, dst.data_ptr())
        img = dst.cpu().numpy()
        assert r.last_damage()[1, 1] and int(r.last_damage().sum()) == 1
        assert np.array_equal(img[16:32, 16:32], full[16:32, 16:32])
    finally:
        r.set_damage_tracking(False)


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")
def test_coarse_budget():
    """Both instantiations: no stack or local memory, at most 64 registers (four 256-thread CTAs per SM) and shared memory
    for four CTAs with room left for k_path_tiling, which runs beside it."""
    import __graft_entry__ as g
    g.build()
    obj = os.path.join(ROOT, "vello_b200", "csrc", "build", "k_coarse.o")
    res = subprocess.run(["cuobjdump", "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*k_coarse\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)
    assert len(found) == 2, res
    for fn, reg, stack_, shared, local in found:
        reg, stack_, shared, local = map(int, (reg, stack_, shared, local))
        assert stack_ == 0 and local == 0, f"{fn}: {stack_} B stack, {local} B local"
        assert reg <= 64, f"{fn}: {reg} registers"
        assert 4 * (shared + 1024) <= 160 * 1024, f"{fn}: {shared} B of shared memory"
