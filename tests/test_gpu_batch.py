"""Batched rendering (vb_set_cells / Renderer.render_batch): N scenes of one size in one pass into an [N, H, W, 4] buffer.
Every cell is compared with the same scene rendered alone at the same size (byte-equal in MSAA8/16, within assert_pixels'
tolerance in Area) and, for the mixed batch, with the oracle's single-scene frame."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (BLACK, COMPOSE_SRC_OVER, FILL_NON_ZERO, MIX_MULTIPLY, Color, Gradient, Scene, Stroke, batch,
                                 resolve)
from vello_b200.shapes import Affine, Circle, Rect

from . import parity
from .test_gpu_parity import assert_pixels

pytestmark = pytest.mark.gpu
BASE = Color.from_rgba8(20, 30, 40)


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


@pytest.fixture(scope="module")
def oracle():
    from oracle.vbo import Oracle
    return Oracle(threads=8)


def alone(r, s, p):
    """The scene rendered alone, with its open layers popped (a batch closes them behind each scene, as pop_layer does)."""
    c = Scene()
    c.append(s)
    for _ in range(s.encoding.n_open_clips):
        c.pop_layer()
    return r.render_to_texture(resolve(c.encoding), p)


def assert_cells(r, ss, p, frames, singles=None):
    assert frames.shape == (len(ss), p.height, p.width, 4)
    for i, s in enumerate(ss):
        ref = singles[i] if singles is not None else alone(r, s, p)
        if p.antialiasing_method == AA_AREA:
            assert_pixels(frames[i], ref, AA_AREA)
        else:
            assert np.array_equal(frames[i], ref), f"cell {i}: {int((frames[i] != ref).any(axis=2).sum())} pixels differ"


def mixed():
    out = [scenes.tiger(300, 220), scenes.brushes()[0], scenes.blend_grid()[0], scenes.many_clips()[0], scenes.deep_blend()[0],
           scenes.fill_types()[0], scenes.stroke_styles()[0], scenes.gradient_extend()[0], scenes.two_point_radial()[0],
           scenes.image_extend_modes()[0], scenes.funky_paths()[0], Scene()]
    return out


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_mixed_batch(renderer, oracle, aa):
    ss = mixed()
    p = RenderParams(BASE, 300, 220, aa)
    frames = renderer.render_batch(ss, p)
    assert_cells(renderer, ss, p, frames)
    for i, s in enumerate(ss):
        ref = oracle.render(resolve(s.encoding), 300, 220, BASE.premul_rgba8_u32(), aa)
        assert_pixels(frames[i], ref, aa)


def bleeder():
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 40, 40), None, Rect(-500, -500, 900, 900))
    s.stroke(Stroke(40.0), Affine.IDENTITY, Color.from_rgba8(40, 200, 40, 180), None, Circle(64.0, 48.0, 200.0))
    g = Gradient.linear((-300.0, -300.0), (400.0, 400.0), [(0.0, Color.from_rgba8(0, 0, 255)), (1.0, Color.from_rgba8(255, 255, 0))])
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, g, None, Rect(-300, 10, 700, 60))
    s.draw_blurred_rounded_rect(Affine.IDENTITY, Rect(-100, -100, 400, 300), Color.from_rgba8(255, 255, 255, 200), 20.0, 30.0)
    return s


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
def test_no_bleed(renderer, aa):
    p = RenderParams(BASE, 128, 96, aa)
    ss = [Scene(), Scene(), bleeder(), Scene(), Scene()]
    frames = renderer.render_batch(ss, p)
    base = np.array([20, 30, 40, 255], dtype=np.uint8)
    for i in (0, 1, 3, 4):
        assert (frames[i] == base).all(), f"cell {i} is not the base colour"
    assert_cells(renderer, ss[2:3], p, frames[2:3])


def open_layers(closed: bool):
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 100, 50), None, Rect(0, 0, 100, 80))
    s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Circle(50.0, 40.0, 35.0))
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.6, Affine.IDENTITY, Rect(10, 10, 90, 70))
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(30, 160, 220, 200), None, Rect(20, 0, 120, 60))
    if closed:
        s.pop_layer()
        s.pop_layer()
    return s


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
def test_open_layers_are_closed_per_cell(renderer, aa):
    """A scene that ends with open layers: its cell is the scene with those layers popped, and the cells after it are not
    inside them."""
    p = RenderParams(BASE, 100, 80, aa)
    ss = [open_layers(False), scenes.fill_types()[0], open_layers(False)]
    frames = renderer.render_batch(ss, p)
    assert_cells(renderer, [open_layers(True), ss[1], open_layers(True)], p, frames)


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16])
def test_one_cell_is_the_plain_frame(renderer, aa):
    s = scenes.tiger(256, 200)
    p = RenderParams(BLACK, 256, 200, aa)
    assert np.array_equal(renderer.render_batch([s], p)[0], alone(renderer, s, p))


@pytest.mark.parametrize("h", [16, 17, 256, 257])
def test_cell_heights(renderer, h):
    ss = [scenes.random_small(k)[0] for k in range(5)]
    p = RenderParams(BLACK, 200, h, AA_MSAA16)
    assert_cells(renderer, ss, p, renderer.render_batch(ss, p))


def test_thousands_of_tiny_cells(renderer):
    """3,000 cells of 32x24: one 256-draw partition spans many cells."""
    distinct = [scenes.random_small(k, n=12, size=40)[0] for k in range(30)]
    ss = [distinct[i % 30] for i in range(3000)]
    for aa in (AA_MSAA16, AA_AREA):
        p = RenderParams(BASE, 32, 24, aa)
        frames = renderer.render_batch(ss, p)
        singles = [alone(renderer, s, p) for s in distinct]
        assert_cells(renderer, ss, p, frames, [singles[i % 30] for i in range(3000)])


def test_big_cell_among_tiny(renderer):
    """One cell of 2,000 draws: a cell spans many partitions."""
    big = scenes.paris_like(2000, 96, seed=5)
    tiny = [scenes.random_small(k, n=5, size=64)[0] for k in range(6)]
    ss = tiny[:3] + [big] + tiny[3:]
    p = RenderParams(BLACK, 96, 64, AA_MSAA16)
    assert_cells(renderer, ss, p, renderer.render_batch(ss, p))


@pytest.mark.parametrize("arena", ["binning", "tiles", "ptcl"])
def test_grow_and_retry(arena):
    from vello_b200.renderer import Renderer
    ss = mixed()[:6]
    p = RenderParams(BASE, 300, 220, AA_MSAA16)
    r = Renderer()
    full = r.render_batch(ss, p)
    st = r.last_stats
    need = {"binning": st.binning, "tiles": st.tile, "ptcl": None}[arena]
    if arena == "ptcl":
        cfg = r.download("config", np.uint32)
        n_tiles = int(cfg[0]) * ((220 + 15) // 16) * len(ss)
        need = n_tiles * 64 + st.ptcl
    r.limit_arena(arena, need)  # exactly enough: no retry
    assert np.array_equal(r.render_batch(ss, p), full) and r.last_stats.retries == 0
    r.limit_arena(arena, need - 1)
    assert np.array_equal(r.render_batch(ss, p), full)
    assert r.last_stats.retries == 1
    r.close()


def test_invisible_switches(renderer):
    ss = [scenes.random_small(k)[0] for k in range(4)]
    p = RenderParams(BASE, 200, 150, AA_MSAA16)
    bs, offsets = batch(ss)
    packed = resolve(bs.encoding)
    renderer.upload(packed)
    renderer.set_cells(offsets)
    out = torch_out(len(ss), p)
    ptr = out.data_ptr()
    frames = []
    for _ in range(3):  # replayed graph
        renderer.render_resident(p, ptr)
        frames.append(out.cpu().numpy().copy())
    assert all(np.array_equal(f, frames[0]) for f in frames)
    assert_cells(renderer, ss, p, frames[0])
    renderer.upload(packed)  # a new upload is one cell again: every scene over each other
    renderer.set_cells([0, offsets[-1]])
    renderer.render_resident(p, ptr)
    whole = out[0].cpu().numpy()
    assert np.array_equal(whole, renderer.render_to_texture(packed, p))
    renderer.upload(packed)
    renderer.set_cells(offsets)  # cells change: captured again
    renderer.set_occlusion_cull(False)
    renderer.render_resident(p, ptr)
    renderer.set_occlusion_cull(True)
    assert np.array_equal(out.cpu().numpy(), frames[0])
    renderer.set_cuda_graph(False)
    renderer.render_resident(p, ptr)
    renderer.set_cuda_graph(True)
    assert np.array_equal(out.cpu().numpy(), frames[0])


def torch_out(n, p):
    torch = pytest.importorskip("torch")
    return torch.zeros((n, p.height, p.width, 4), dtype=torch.uint8, device="cuda")


def test_render_batch_into_cuda_tensor(renderer):
    ss = [scenes.random_small(k)[0] for k in range(3)]
    p = RenderParams(BASE, 120, 90, AA_AREA)
    out = torch_out(3, p)
    assert renderer.render_batch(ss, p, out=out) is out
    assert np.array_equal(out.cpu().numpy(), renderer.render_batch(ss, p))


def test_registered_texture_in_two_cells(renderer):
    torch = pytest.importorskip("torch")
    from vello_b200.scene_native import NativeScene
    px = (np.arange(40 * 30 * 4, dtype=np.uint32) * 53 % 251).astype(np.uint8).reshape(30, 40, 4)
    px[..., 3] = 255
    t = torch.from_numpy(px).cuda()
    im = renderer.register_texture(t)
    try:
        def cell(k):
            s = NativeScene()
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(10 * k, 90, 160), None, Rect(0, 0, 64, 48))
            s.draw_image(im, Affine.translate(3.0 + 5 * k, 4.0 + 2 * k))
            return s
        ss = [cell(0), cell(1), cell(2)]
        p = RenderParams(BASE, 64, 48, AA_MSAA16)
        frames = renderer.render_batch(ss, p)
        for k, s in enumerate(ss):
            s.upload_device(renderer)
            renderer.render_resident(p)
            assert np.array_equal(frames[k], renderer.download_target(p)), k
    finally:
        renderer.unregister_texture(im)


def test_rejections_leave_the_renderer_usable(renderer):
    from vello_b200.renderer import VelloB200Error
    s0, s1 = scenes.random_small(1)[0], open_layers(True)
    bs, offsets = batch([s0, s1])
    packed = resolve(bs.encoding)
    p = RenderParams(BASE, 100, 80, AA_MSAA16)
    good = renderer.render_batch([s0, s1], p)

    def ok():
        renderer.upload(packed)
        renderer.set_cells(offsets)
        out = torch_out(2, p)
        renderer.render_resident(p, out.data_ptr())
        assert np.array_equal(out.cpu().numpy(), good)

    n = offsets[-1]
    clip_cut = offsets[1] + 2  # inside s1's clip: BEGIN_CLIPs in one cell, their END_CLIPs in the next
    for bad in ([1, offsets[1], n], [0, offsets[1], n - 1], [0, n, offsets[1], n], [0, offsets[1], clip_cut, n]):
        renderer.upload(packed)
        with pytest.raises(VelloB200Error, match="vb_set_cells"):
            renderer.set_cells(bad)
        ok()
    renderer.upload(packed)
    renderer.set_cells(offsets)
    with pytest.raises(VelloB200Error, match="batch"):
        renderer.render_resident(p, 0, bin_rows=(0, 1))
    ok()
    with pytest.raises(VelloB200Error, match="batch"):
        renderer.render_resident(p, 0, tile_rows=(0, 2))
    ok()
    renderer.upload(packed)
    renderer.set_cells([0] * 40000 + [n])  # 40,000 cells (all but the last empty): more bin rows than the coarse grid indexes
    with pytest.raises(VelloB200Error, match="batch"):
        renderer.render_resident(p, 0)
    ok()


def test_stage_parity_of_a_batch(renderer, oracle):
    """The stages before binning and the path stages do not know about cells: the batch's encoding gives the same lines, path
    boxes, paths and tile backdrops as the oracle's single frame of that encoding at the cell's size."""
    ss = mixed()[:8]
    bs, offsets = batch(ss)
    packed = resolve(bs.encoding)
    p = RenderParams(BASE, 300, 220, AA_MSAA16)
    renderer.upload(packed)
    renderer.set_cells(offsets)
    renderer.render_resident(p)
    oracle.render(packed, 300, 220, BASE.premul_rgba8_u32(), AA_MSAA16)
    g = parity.gpu_buffers(renderer, ["lines", "path_bboxes", "paths", "tiles"])
    c = {n: oracle.buffer(n) for n in g}
    assert np.array_equal(g["path_bboxes"], c["path_bboxes"])
    lines_g = np.sort(np.ascontiguousarray(g["lines"]).view(np.uint32).reshape(len(g["lines"]), -1), axis=0)
    lines_c = np.sort(np.ascontiguousarray(c["lines"]).view(np.uint32).reshape(len(c["lines"]), -1), axis=0)
    assert np.array_equal(lines_g, lines_c)
    pg = np.ascontiguousarray(g["paths"]).view(np.uint32).reshape(len(g["paths"]), -1)
    pc = np.ascontiguousarray(c["paths"]).view(np.uint32).reshape(len(c["paths"]), -1)
    n = packed.layout.n_paths  # the oracle's buffer is padded past the last path
    assert len(pg) >= n and np.array_equal(pg[:n, :5], pc[:n, :5])
    tg = np.ascontiguousarray(g["tiles"]).view(np.int32).reshape(-1, 2)
    tc = np.ascontiguousarray(c["tiles"]).view(np.int32).reshape(-1, 2)
    nt = int(pg[n - 1, 4]) + (int(pg[n - 1, 2]) - int(pg[n - 1, 0])) * (int(pg[n - 1, 3]) - int(pg[n - 1, 1]))  # end of the last path's tiles
    assert len(tg) >= nt and len(tc) >= nt and np.array_equal(tg[:nt, 0], tc[:nt, 0])
