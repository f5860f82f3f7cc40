"""vb_hit_test / Renderer.hit_test on the GPU, held to the geometric statement in tests/hit_ref.py on the same frame's
downloaded buffers: every answer equals hit_ref's on every point that is not within a line's tolerance of a line the point
evaluates, and those ambiguous points stay under 1 %. Also: batches answer as their cells rendered alone, a viewed frame as
the host-mapped scene, a re-run frame as one that fitted at once, the device form as the host form; every state rule
returns its code; and hit tests leave the frame alone."""

import math

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Scene, batch, resolve, viewed
from vello_b200.shapes import Affine, Circle, Rect

from . import hit_ref

pytestmark = pytest.mark.gpu

VB_E_INVALID, VB_E_NO_SCENE = -1, -4


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def params(w, h, aa=AA_AREA):
    return RenderParams(base_color=BLACK, width=w, height=h, antialiasing_method=aa)


def frame(r, packed, w, h, aa=AA_AREA):
    r.upload(packed)
    r.render_resident(params(w, h, aa))


def points(w, h, seed=1, step=None, n_random=4000):
    """Pixel centres on a grid, random sub-pixel points, points on tile and bin edges, the frame's edges, and points that
    must answer -1 (negative, past the frame, NaN)."""
    rng = np.random.default_rng(seed)
    step = step or max(3, round(math.sqrt(w * h / 20000)))  # about 20,000 pixel centres
    m = max(250, w * h // 700)  # points per family of edge points
    gx, gy = np.meshgrid(np.arange(0, w, step) + 0.5, np.arange(0, h, step) + 0.5)
    grid = np.stack([gx.ravel(), gy.ravel()], 1)
    rand = rng.random((n_random, 2)) * (w, h)
    ex = np.unique(np.concatenate([np.arange(0, w, 16), np.arange(0, w, 256), [w - 2.0 ** -10]]))
    ey = np.unique(np.concatenate([np.arange(0, h, 16), np.arange(0, h, 256), [h - 2.0 ** -10]]))
    # on tile / bin edges: one coordinate on an edge, the other random (and both on edges, sampled)
    edge = np.concatenate([np.stack([rng.choice(ex, m), rng.random(m) * h], 1),
                           np.stack([rng.random(m) * w, rng.choice(ey, m)], 1),
                           np.stack([rng.choice(ex, m * 2 // 3), rng.choice(ey, m * 2 // 3)], 1),
                           [(0.0, 0.0), (w - 2.0 ** -10, 0.0), (0.0, h - 2.0 ** -10), (w - 2.0 ** -10, h - 2.0 ** -10)]])
    nan = float("nan")
    bad = [(-1.0, 5.0), (5.0, -1.0), (-2.0 ** -20, 3.0), (w, 3.0), (3.0, h), (w + 100.0, h + 5.0), (1e30, 1e30), (-1e30, 3.0),
           (nan, 3.0), (3.0, nan), (nan, nan), (float("inf"), 3.0), (3.0, -float("inf"))]
    return np.concatenate([grid, rand, edge, bad]).astype(np.float32), len(bad)


def check_against_ref(r, packed, w, h, pts, n_bad=0, max_ambiguous=0.01, min_hit=0.01):
    want, amb = hit_ref.hit_ref(hit_ref.frame_from_gpu(r, packed), pts, w, h)
    got = r.hit_test(pts)
    assert got.dtype == np.int32 and got.shape == (len(pts),)
    bad = (got != want) & ~amb
    if bad.any():
        k = np.nonzero(bad)[0]
        raise AssertionError(f"{len(k)} of {len(pts)} points differ from hit_ref, first at {pts[k[0]].tolist()}: "
                             f"{int(got[k[0]])} != {int(want[k[0]])}")
    if n_bad:
        assert (got[-n_bad:] == -1).all()
    share = float(amb.mean())
    print(f"ambiguous {100 * share:.3f} % of {len(pts)} points; {int((got >= 0).sum())} hit")
    assert share < max_ambiguous, share
    assert (got >= 0).mean() >= min_hit  # the answers are not all -1
    return got


def crowded_bin():
    """One 256 px bin whose draw list spans several 256-draw partitions, with clips among the draws."""
    rng = np.random.default_rng(7)
    s = Scene()
    for k in range(900):
        if k % 150 == 75:
            s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, Circle(float(rng.uniform(60, 200)), float(rng.uniform(60, 200)),
                                                                     float(rng.uniform(40, 120))))
        x, y = rng.uniform(0, 240, 2)
        c = Color.from_rgba8(*(int(v) for v in rng.integers(0, 256, 3)), int(rng.integers(0, 256)))
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Rect(float(x), float(y), float(x + rng.uniform(2, 60)), float(y + rng.uniform(2, 60))))
        if k % 150 == 140:
            s.pop_layer()
    return s


SCENES = {
    "tiger": lambda: (scenes.tiger(1024, 1024), 1024, 1024),
    "paris_like": lambda: (scenes.paris_like(2000, 1024), 1024, 1024),
    "beziers_clips": lambda: (scenes.beziers_clips(3000, 60, 1024), 1024, 1024),
    "many_clips": lambda: scenes.many_clips(),
    "crowded_bin": lambda: (crowded_bin(), 300, 300),
}


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16], ids=["area", "msaa16"])
@pytest.mark.parametrize("name", list(SCENES))
def test_answers_equal_the_geometric_reference(renderer, name, aa):
    s, w, h = SCENES[name]()
    packed = resolve(s.encoding)
    frame(renderer, packed, w, h, aa)
    pts, n_bad = points(w, h, seed=len(name))
    check_against_ref(renderer, packed, w, h, pts, n_bad)


def test_crowded_bin_spans_several_partitions(renderer):
    s = crowded_bin()
    packed = resolve(s.encoding)
    frame(renderer, packed, 300, 300)
    from oracle.vbo import DTYPES
    hdr = renderer.download("bin_headers", DTYPES["bin_headers"])
    n_parts = (packed.layout.n_draw_objects + 255) // 256
    assert n_parts >= 3
    counts = hdr["element_count"].reshape(n_parts, -1)[:, 0]  # bin 0 of every partition
    assert (counts > 0).sum() >= 3, counts


def test_batch_answers_are_the_cells_answers(renderer):
    w = h = 200
    cells = [scenes.random_small(seed, 60, 200)[0] for seed in range(6)] + [scenes.many_clips()[0], crowded_bin()]
    pts, _ = points(w, h, seed=3, step=5, n_random=1500)
    alone = []
    for s in cells:
        frame(renderer, resolve(s.encoding), w, h)
        alone.append(renderer.hit_test(pts))
    bs, offsets = batch(cells)
    renderer.upload(resolve(bs.encoding))
    renderer.set_cells(offsets)
    renderer.render_resident(params(w, h))
    tall = np.concatenate([pts + np.float32((0, c * h)) for c in range(len(cells))])
    got = renderer.hit_test(tall).reshape(len(cells), -1)
    for c in range(len(cells)):
        want = np.where(alone[c] >= 0, alone[c] + offsets[c], -1)
        inside = np.isfinite(pts).all(1) & (pts[:, 1] >= 0) & (pts[:, 1] < h)  # points off the cell's rows land in another cell
        assert (got[c][inside] == want[inside]).all(), c
    renderer.set_cells([0, offsets[-1]])


VIEWS = {
    "pan": Affine.translate(-137.25, 61.5),
    "zoom4": Affine.translate(-700.0, -300.0) * Affine.scale(4.0),
    "zoom16_rotated": Affine.translate(512.0, 512.0) * Affine.rotate(0.3) * Affine.scale(16.0) * Affine.translate(-420.0, -610.0),
}


@pytest.mark.parametrize("view", list(VIEWS))
def test_a_viewed_frame_answers_as_the_host_mapped_scene(view):
    from vello_b200.renderer import Renderer
    w = h = 1024
    packed = resolve(scenes.paris_like(2000, 1024).encoding)
    pts, _ = points(w, h, seed=11)
    a, b = Renderer(), Renderer()
    try:
        a.upload(packed)
        a.set_view(VIEWS[view])
        a.render_resident(params(w, h))
        got = a.hit_test(pts)
        mapped = viewed(packed, VIEWS[view])
        frame(b, mapped, w, h)
        want = b.hit_test(pts)
        assert (got == want).all(), int((got != want).sum())
        check_against_ref(b, mapped, w, h, pts, min_hit=0.0)
        # a new view changes nothing until the next frame
        a.set_view(Affine.IDENTITY)
        assert (a.hit_test(pts) == got).all()
    finally:
        a.close()
        b.close()


def test_grow_and_retry_answers_from_the_attempt_that_fitted():
    from vello_b200.renderer import Renderer
    w = h = 1024
    packed = resolve(scenes.paris_like(2000, 1024).encoding)
    pts, _ = points(w, h, seed=5)
    a, b = Renderer(), Renderer()
    try:
        frame(a, packed, w, h)
        want = a.hit_test(pts)
        b.upload(packed)
        b.render_resident(params(w, h))
        b.limit_arena("lines", int(b.last_stats.lines) // 2)
        b.limit_arena("segments", int(b.last_stats.segments) // 3)
        st = b.render_resident(params(w, h))
        assert st.retries >= 1
        assert (b.hit_test(pts) == want).all()
    finally:
        a.close()
        b.close()


def test_device_form_equals_host_form(renderer):
    torch = pytest.importorskip("torch")
    w = h = 1024
    frame(renderer, resolve(scenes.paris_like(2000, 1024).encoding), w, h)
    rng = np.random.default_rng(9)
    pts = (rng.random((1_000_000, 2)) * (w * 1.02, h * 1.02) - (w * 0.01, h * 0.01)).astype(np.float32)
    want = renderer.hit_test(pts)
    dev = torch.from_numpy(pts).cuda()
    out = torch.full((len(pts),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert renderer.hit_test(dev, out) is out
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == want).all()
    with pytest.raises(ValueError):
        renderer.hit_test(dev)  # no `out`
    with pytest.raises(ValueError):
        renderer.hit_test(dev, torch.empty(5, dtype=torch.int32, device="cuda"))


def _code(r, pts, out=None, on_device=0, n=None):
    pts = np.ascontiguousarray(pts, np.float32)
    out = np.zeros(len(pts), np.int32) if out is None else out
    return r.lib.vb_hit_test(r.handle, pts.ctypes.data, len(pts) if n is None else n, out.ctypes.data, on_device)


def test_state_rules():
    from vello_b200.renderer import Renderer
    r = Renderer()
    try:
        s, w, h = scenes.many_clips()
        packed = resolve(s.encoding)
        pts = np.array([[10.5, 10.5], [w / 2, h / 2]], np.float32)
        assert _code(r, pts) == VB_E_NO_SCENE  # nothing rendered yet
        assert _code(r, pts, n=0) == 0  # n = 0: nothing to do
        r.upload(packed)
        assert _code(r, pts) == VB_E_NO_SCENE
        r.render_resident(params(w, h))
        assert _code(r, pts) == 0
        ok = r.hit_test(pts)
        assert r.lib.vb_hit_test(r.handle, None, 2, np.zeros(2, np.int32).ctypes.data, 0) == VB_E_INVALID
        assert r.lib.vb_hit_test(r.handle, pts.ctypes.data, 2, None, 0) == VB_E_INVALID
        assert _code(r, pts, on_device=1) == VB_E_INVALID  # host memory is not device memory
        r.set_view(Affine.translate(3.0, 4.0))
        assert (r.hit_test(pts) == ok).all()  # the frame on screen is still the unviewed one
        r.set_view(None)
        # every call that rewrites what the answers read
        for undo in (lambda: r.set_cells([0, packed.layout.n_draw_objects]),
                     lambda: r.run_stages(params(w, h), "pathtag", "fine"),
                     lambda: r.upload_buffer("paths", r.download("paths", np.uint8)),
                     lambda: r.limit_arena("lines", r.NO_LIMIT),
                     lambda: r.upload(packed)):
            r.render_resident(params(w, h))
            assert _code(r, pts) == 0
            undo()
            assert _code(r, pts) == VB_E_NO_SCENE
        # a windowed frame
        r.render_resident(params(w, h), bin_rows=(0, 1))
        assert _code(r, pts) == VB_E_INVALID
        r.render_resident(params(w, h))
        # a frame in flight
        r.enqueue(params(w, h))
        assert _code(r, pts) == VB_E_INVALID
        r.finish()
        assert (r.hit_test(pts) == ok).all()
        stream = r.render_stream([packed] * 4, params(w, h))
        next(stream)  # three frames submitted, the first complete: the others are in flight
        assert _code(r, pts) == VB_E_INVALID
        list(stream)
        assert (r.hit_test(pts) == ok).all()
    finally:
        r.close()


def test_group_renderers_are_refused():
    from vello_b200.renderer import RendererGroup
    g = RendererGroup([0, 0])
    try:
        s, w, h = scenes.many_clips()
        g.render_to_texture(s, params(w, h))
        assert _code(g.renderer(0), np.array([[1.5, 1.5]], np.float32)) == VB_E_INVALID
    finally:
        g.close()


def test_hit_tests_leave_the_frame_alone():
    from vello_b200.renderer import Renderer
    w = h = 512
    packed = resolve(scenes.paris_like(1500, 512).encoding)
    p = params(w, h, AA_MSAA16)
    pts, _ = points(w, h, seed=2)
    a, b = Renderer(), Renderer()
    try:
        for r in (a, b):
            r.upload(packed)
            r.render_resident(p)
        launches, captures = a.last_stats.kernel_launches, a.debug_graph_captures()
        a.hit_test(pts)
        try:
            import torch
            out = torch.empty(len(pts), dtype=torch.int32, device="cuda")
            a.hit_test(torch.from_numpy(pts).cuda(), out)
            torch.cuda.synchronize()
        except ImportError:
            pass
        st_a = a.render_resident(p)
        st_b = b.render_resident(p)
        assert st_a.kernel_launches == launches == st_b.kernel_launches
        assert a.debug_graph_captures() == captures == b.debug_graph_captures()
        assert a.download_target(p).tobytes() == b.download_target(p).tobytes()
    finally:
        a.close()
        b.close()
