"""vb_hit_map / Renderer.hit_map: vb_hit_test's answer at every pixel centre of a rectangle of the last frame, one CTA per
16 x 16 tile. On the GPU, every map equals hit_test at the same centres with no pixel allowed to differ: whole frames and
sub-rectangles at tile, bin and frame edges of every scene hit tests are checked on, batches (and each cell against the cell
rendered alone), viewed frames, frames re-run after an overflow and damage-tracked incremental frames. Maps also equal the
geometric reference (tests/hit_ref.py), the host form equals the device form, pitched outputs change nothing outside the
rectangle, every state rule returns what vb_hit_test returns, and maps leave the frame alone. Without a GPU: k_hit_map
compiles to code with no stack and no local memory."""

import shutil

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA16
from vello_b200.encoding import FILL_NON_ZERO, Color, Scene, batch, resolve
from vello_b200.shapes import Affine, Rect

from . import hit_ref
from .test_compiled_kernels import built, usage  # noqa: F401 (the fixtures that read the compiled objects)
from .test_gpu_hit_test import SCENES, VB_E_INVALID, VB_E_NO_SCENE, VIEWS, _code, crowded_bin, frame, params

gpu = pytest.mark.gpu
GUARD = -123456


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def centres(x0, y0, w, h):
    """The pixel centres of the rectangle, row by row, as hit_test takes them."""
    gx, gy = np.meshgrid(np.arange(x0, x0 + w, dtype=np.float64) + 0.5, np.arange(y0, y0 + h, dtype=np.float64) + 0.5)
    return np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float32)


def check_equals_hit_test(r, rect=None, got=None):
    """The map of `rect` (None: the whole frame) equals hit_test at its centres, int for int."""
    if rect is None:
        rect = (0, 0) + tuple(r._hit_extent)
    x0, y0, w, h = rect
    got = r.hit_map(rect) if got is None else got
    assert got.dtype == np.int32 and got.shape == (h, w)
    want = r.hit_test(centres(*rect)).reshape(h, w)
    bad = np.argwhere(got != want)
    if len(bad):
        j, i = bad[0]
        raise AssertionError(f"{len(bad)} of {w * h} pixels of {rect} differ from hit_test, first at ({x0 + i}, {y0 + j}): "
                             f"{int(got[j, i])} != {int(want[j, i])}")
    return got


def sub_rects(w, h):
    """Rectangles at odd offsets across tile and bin edges, one pixel, one row, one column, and the frame's last corner (the
    last, partial tile when the size is not a multiple of 16)."""
    return [(13, min(250, h - 19), min(277, w - 13), 19), (min(250, w - 20), 7, 20, h - 7), (min(255, w - 1), min(256, h - 1), 1, 1),
            (0, h // 2 - 1, w, 1), (w // 2 + 5, 0, 1, h), (w - 33, h - 17, 33, 17), (w - 12, h - 12, 12, 12)]


@gpu
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA16], ids=["area", "msaa16"])
@pytest.mark.parametrize("name", list(SCENES))
def test_map_equals_hit_test(renderer, name, aa):
    s, w, h = SCENES[name]()
    frame(renderer, resolve(s.encoding), w, h, aa)
    whole = check_equals_hit_test(renderer)
    assert (whole >= 0).mean() >= 0.01
    for rect in sub_rects(w, h):
        x0, y0, rw, rh = rect
        sub = check_equals_hit_test(renderer, rect)
        assert (sub == whole[y0:y0 + rh, x0:x0 + rw]).all(), rect


@gpu
@pytest.mark.parametrize("name", ["tiger", "many_clips", "crowded_bin"])
def test_map_equals_the_geometric_reference(renderer, name):
    s, w, h = SCENES[name]()
    packed = resolve(s.encoding)
    frame(renderer, packed, w, h)
    got = renderer.hit_map()
    ys, xs = np.mgrid[0:h:3, 0:w:3]  # every ninth pixel centre: the reference is float64 numpy
    pts = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], 1).astype(np.float32)
    want, amb = hit_ref.hit_ref(hit_ref.frame_from_gpu(renderer, packed), pts, w, h)
    g = got[ys.ravel(), xs.ravel()]
    bad = (g != want) & ~amb
    assert not bad.any(), f"{int(bad.sum())} centres differ from hit_ref, first at {pts[np.argmax(bad)].tolist()}"
    assert amb.mean() < 0.01, amb.mean()
    assert (g >= 0).mean() >= 0.01


@gpu
def test_batch_map_is_the_cells_maps(renderer):
    w = h = 200  # not a multiple of 16: every cell ends in a partial tile row
    cells = [scenes.random_small(seed, 60, 200)[0] for seed in range(6)] + [scenes.many_clips()[0], crowded_bin()]
    alone = []
    for s in cells:
        frame(renderer, resolve(s.encoding), w, h)
        alone.append(renderer.hit_map())
    bs, offsets = batch(cells)
    renderer.upload(resolve(bs.encoding))
    renderer.set_cells(offsets)
    renderer.render_resident(params(w, h))
    try:
        tall = check_equals_hit_test(renderer)
        assert tall.shape == (len(cells) * h, w)
        for c, want in enumerate(alone):
            assert (tall.reshape(len(cells), h, w)[c] == np.where(want >= 0, want + offsets[c], -1)).all(), c
        for rect in [(3, h - 9, 150, 25), (0, 3 * h - 1, w, 2), (w - 7, h // 2, 7, 3 * h), (17, 5 * h + 3, 1, 1)]:
            x0, y0, rw, rh = rect
            assert (check_equals_hit_test(renderer, rect) == tall[y0:y0 + rh, x0:x0 + rw]).all(), rect
    finally:
        renderer.set_cells([0, offsets[-1]])


@gpu
@pytest.mark.parametrize("view", list(VIEWS))
def test_a_viewed_frame_maps_as_it_hit_tests(renderer, view):
    w = h = 1024
    renderer.upload(resolve(scenes.paris_like(2000, 1024).encoding))
    renderer.set_view(VIEWS[view])
    try:
        renderer.render_resident(params(w, h))
        check_equals_hit_test(renderer)
        check_equals_hit_test(renderer, (301, 77, 400, 333))
    finally:
        renderer.set_view(None)


@gpu
def test_a_rerun_frame_maps_from_the_attempt_that_fitted():
    from vello_b200.renderer import Renderer
    w = h = 1024
    packed = resolve(scenes.paris_like(2000, 1024).encoding)
    a, b = Renderer(), Renderer()
    try:
        frame(a, packed, w, h)
        want = a.hit_map()
        b.upload(packed)
        b.render_resident(params(w, h))
        b.limit_arena("lines", int(b.last_stats.lines) // 2)
        b.limit_arena("segments", int(b.last_stats.segments) // 3)
        st = b.render_resident(params(w, h))
        assert st.retries >= 1
        assert (check_equals_hit_test(b) == want).all()
    finally:
        a.close()
        b.close()


@gpu
def test_device_form_equals_host_form_and_pitched_outputs_keep_their_guards(renderer):
    torch = pytest.importorskip("torch")
    w = h = 1024
    frame(renderer, resolve(scenes.paris_like(2000, 1024).encoding), w, h)
    want = renderer.hit_map()
    out = torch.full((h, w), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert renderer.hit_map(out=out) is out
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == want).all()
    x0, y0, rw, rh = rect = (37, 250, 300, 45)
    sub = want[y0:y0 + rh, x0:x0 + rw]
    # a row slice of a wider device tensor, and a numpy view: only the rectangle's answers change
    big = torch.full((rh + 4, rw + 37), GUARD, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    view = big[2:2 + rh, 5:5 + rw]
    assert renderer.hit_map(rect, out=view) is view
    torch.cuda.synchronize()
    host_big = np.full((rh + 3, rw + 11), GUARD, np.int32)
    host_view = host_big[1:1 + rh, 6:6 + rw]
    assert renderer.hit_map(rect, out=host_view) is host_view
    for b, (r0, c0) in ((big.cpu().numpy(), (2, 5)), (host_big, (1, 6))):
        assert (b[r0:r0 + rh, c0:c0 + rw] == sub).all()
        guard = np.ones(b.shape, bool)
        guard[r0:r0 + rh, c0:c0 + rw] = False
        assert (b[guard] == GUARD).all()
    # one row of a device tensor: its pitch is never used
    row = torch.full((1, rw), GUARD, dtype=torch.int32, device="cuda")
    renderer.hit_map((x0, y0, rw, 1), out=row)
    torch.cuda.synchronize()
    assert (row.cpu().numpy()[0] == sub[0]).all()
    for bad in (torch.empty((rh, rw + 1), dtype=torch.int32, device="cuda"), torch.empty((rh, rw), dtype=torch.int64, device="cuda"),
                torch.empty((rh, 2 * rw), dtype=torch.int32, device="cuda")[:, ::2], np.empty((rh, rw), np.float32),
                np.empty((rh, 2 * rw), np.int32)[:, ::2], np.empty((rw, rh), np.int32).T):
        with pytest.raises(ValueError):
            renderer.hit_map(rect, out=bad)


def _map_code(r, rect, out=None, pitch=None, on_device=0):
    x0, y0, w, h = rect
    out = np.zeros((max(h, 1), max(w, 1)), np.int32) if out is None else out
    ptr = out.ctypes.data if isinstance(out, np.ndarray) else out
    return r.lib.vb_hit_map(r.handle, x0, y0, w, h, ptr, 4 * max(w, 1) if pitch is None else pitch, on_device)


@gpu
def test_state_rules():
    from vello_b200.renderer import Renderer
    r = Renderer()
    try:
        s, w, h = scenes.many_clips()
        packed = resolve(s.encoding)
        pts = np.array([[10.5, 10.5], [w / 2, h / 2]], np.float32)
        rect = (3, 5, 40, 30)

        def same(code):
            assert _code(r, pts) == code
            assert _map_code(r, rect) == code
        same(VB_E_NO_SCENE)  # nothing rendered yet
        assert _map_code(r, (0, 0, 0, 5)) == 0 and _map_code(r, (7, 7, 5, 0)) == 0  # empty: nothing to do
        r.upload(packed)
        same(VB_E_NO_SCENE)
        r.render_resident(params(w, h))
        same(0)
        ok = r.hit_map(rect)
        assert r.lib.vb_hit_map(r.handle, 0, 0, 2, 2, None, 8, 0) == VB_E_INVALID
        assert _map_code(r, rect, on_device=1) == VB_E_INVALID  # host memory is not device memory
        assert _code(r, pts, on_device=1) == VB_E_INVALID
        # rectangles that do not lie inside the frame, and pitches that are not whole rows
        for bad in [(w - 39, 0, 40, 1), (0, h - 9, 1, 10), (w, 0, 1, 1), (0, h, 1, 1), (2 ** 32 - 1, 0, 2, 1), (0, 2 ** 32 - 1, 1, 2)]:
            assert _map_code(r, bad) == VB_E_INVALID, bad
        assert _map_code(r, (0, 0, w, h)) == 0
        assert _map_code(r, rect, pitch=4 * 40 - 4) == VB_E_INVALID
        assert _map_code(r, rect, pitch=4 * 40 + 2) == VB_E_INVALID
        r.set_view(Affine.translate(3.0, 4.0))
        assert (r.hit_map(rect) == ok).all()  # the frame on screen is still the unviewed one
        r.set_view(None)
        # every call that rewrites what the answers read
        for undo in (lambda: r.set_cells([0, packed.layout.n_draw_objects]),
                     lambda: r.run_stages(params(w, h), "pathtag", "fine"),
                     lambda: r.upload_buffer("paths", r.download("paths", np.uint8)),
                     lambda: r.limit_arena("lines", r.NO_LIMIT),
                     lambda: r.upload(packed)):
            r.render_resident(params(w, h))
            same(0)
            undo()
            same(VB_E_NO_SCENE)
        # a windowed frame
        r.render_resident(params(w, h), bin_rows=(0, 1))
        same(VB_E_INVALID)
        r.render_resident(params(w, h))
        # a frame in flight
        r.enqueue(params(w, h))
        same(VB_E_INVALID)
        r.finish()
        assert (r.hit_map(rect) == ok).all()
        stream = r.render_stream([packed] * 4, params(w, h))
        next(stream)  # three frames submitted, the first complete: the others are in flight
        same(VB_E_INVALID)
        list(stream)
        assert (r.hit_map(rect) == ok).all()
        assert r.hit_map().shape == (h, w)
    finally:
        r.close()


@gpu
def test_group_renderers_are_refused():
    from vello_b200.renderer import RendererGroup
    g = RendererGroup([0, 0])
    try:
        s, w, h = scenes.many_clips()
        g.render_to_texture(s, params(w, h))
        r = g.renderer(0)
        assert _code(r, np.array([[1.5, 1.5]], np.float32)) == VB_E_INVALID
        assert _map_code(r, (1, 1, 1, 1)) == VB_E_INVALID
    finally:
        g.close()


@gpu
def test_maps_leave_the_frame_alone():
    torch = pytest.importorskip("torch")
    from vello_b200.renderer import Renderer
    w = h = 512
    packed = resolve(scenes.paris_like(1500, 512).encoding)
    p = params(w, h, AA_MSAA16)
    a, b = Renderer(), Renderer()
    try:
        for r in (a, b):
            r.upload(packed)
            r.render_resident(p)
        launches, captures = a.last_stats.kernel_launches, a.debug_graph_captures()
        a.hit_map()
        a.hit_map((5, 9, 300, 200))
        out = torch.empty((h, w), dtype=torch.int32, device="cuda")
        a.hit_map(out=out)
        torch.cuda.synchronize()
        st_a = a.render_resident(p)
        st_b = b.render_resident(p)
        assert st_a.kernel_launches == launches == st_b.kernel_launches
        assert a.debug_graph_captures() == captures == b.debug_graph_captures()
        assert a.download_target(p).tobytes() == b.download_target(p).tobytes()
    finally:
        a.close()
        b.close()


def _rects_scene(items):
    s = Scene()
    for x, y, rw, rh, rgba in items:
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(*rgba), None, Rect(x, y, x + rw, y + rh))
    return s


@gpu
def test_an_incremental_frame_maps_as_the_full_frame():
    torch = pytest.importorskip("torch")
    from vello_b200.renderer import Renderer
    w = h = 512
    g = np.random.default_rng(5)
    items = [(*(float(v) for v in g.uniform(0, 480, 2)), *(float(v) for v in g.uniform(4, 120, 2)),
              tuple(int(v) for v in g.integers(0, 256, 4))) for _ in range(300)]
    p0, p1 = resolve(_rects_scene(items).encoding), resolve(_rects_scene(items[:100] + items[110:]).encoding)
    a, b = Renderer(), Renderer()
    dst = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    try:
        a.set_damage_tracking(True)
        a.set_upload_diff(True)
        a.upload(p0)
        a.render_resident(params(w, h), dst.data_ptr())
        a.upload(p1)
        a.render_resident(params(w, h), dst.data_ptr())
        dmg = a.last_damage()
        assert dmg.any() and not dmg.all()  # incremental
        frame(b, p1, w, h)
        assert (check_equals_hit_test(a) == b.hit_map()).all()
    finally:
        a.close()
        b.close()


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA binary utilities not installed")
def test_hit_map_kernel_uses_no_stack_or_local_memory(usage):  # noqa: F811
    found = {key: u for key, u in usage["k_hit.o"].items() if key[0] == "k_hit_map"}
    assert len(found) == 1, sorted(usage["k_hit.o"])
    u = next(iter(found.values()))
    assert u.stack == 0 and u.local == 0, u

