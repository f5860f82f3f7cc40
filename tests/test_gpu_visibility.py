"""Bound visibility (Renderer.bind_draw_visibility, vb_bind_draw_visibility): every frame shows draw object k only while byte k
of a device array is nonzero, read when the frame runs. `r` binds; `ref` uploads the scene re-encoded without the hidden draw
objects (a hidden push_*_layer without its whole layer), and every frame of `r` must equal it: pixels, lines, hit tests and
hit maps. Run on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (COMPOSE_CLEAR, COMPOSE_COPY, COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_MULTIPLY, MIX_SCREEN,
                                 Color, Gradient, Image, Scene, Stroke, resolve)
from vello_b200.renderer import Renderer, RendererGroup
from vello_b200.shapes import Affine, Circle, Rect, RoundedRect

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_draw_colors import box_tiles
from .test_gpu_instance_transforms import aff, rand_rows
from .test_gpu_parity import assert_pixels
from .test_gpu_path_points import points
from .test_gpu_transforms import transforms

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1
IMG = np.random.default_rng(31).integers(0, 256, (18, 22, 4), dtype=np.uint8)
STOPS = [(0.0, Color(1.0, 0.2, 0.1, 1.0)), (0.6, Color(0.2, 0.9, 0.3, 0.8)), (1.0, Color(0.1, 0.3, 0.9, 0.6))]


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


# ---- scenes as lists of calls, each of which encodes exactly one draw object -----------------------------------------------
def mixed_ops(seed=0, dx=0.0):
    """Fills, strokes, blurred rectangles, a gradient, an image, and layers of every kind: a clip, MIX_MULTIPLY, a destructive
    compose (COMPOSE_CLEAR and COMPOSE_COPY), a luminance mask, and nested layers. Entry k is ("draw" | "push" | "pop", call);
    call k encodes draw object k."""
    g = np.random.default_rng(seed)

    def col():
        c = g.uniform(0, 1, 4)
        c[3] = g.choice([1.0, 0.75, 0.4])
        return Color(*map(float, c))

    ops = []

    def draw(f):
        ops.append(("draw", f))

    def push(f):
        ops.append(("push", f))

    def pop():
        ops.append(("pop", lambda s: s.pop_layer()))

    for i in range(6):
        c = col()
        draw(lambda s, i=i, c=c: s.fill(FILL_NON_ZERO, Affine.translate(dx + 20 + 45 * i, 15 + 9 * i), c, None, Rect(0, 0, 40, 30)))
    c = col()
    draw(lambda s: s.stroke(Stroke(5.0), Affine.IDENTITY, c, None, Circle(dx + 120, 120, 50)))
    c1 = col()
    draw(lambda s: s.draw_blurred_rounded_rect(Affine.translate(dx + 200, 60), Rect(0, 0, 70, 40), c1, 8.0, 5.0))
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((0, 0), (100, 0), STOPS), None, Rect(dx + 10, 180, 130, 240)))
    draw(lambda s: s.draw_image(Image(IMG), Affine.translate(dx + 150, 180) * Affine.scale(2.0)))
    # MIX_MULTIPLY holding a nested clip
    push(lambda s: s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, Affine.IDENTITY, Circle(dx + 190, 160, 90)))
    c2 = col()
    draw(lambda s: s.fill(FILL_EVEN_ODD, Affine.IDENTITY, c2, None, RoundedRect(dx + 110, 90, 290, 250, 14)))
    push(lambda s: s.push_clip_layer(FILL_NON_ZERO, Affine.rotate(0.1), Rect(dx + 130, 100, 260, 220)))
    c3, c4 = col(), col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c3, None, Circle(dx + 200, 170, 60)))
    draw(lambda s: s.draw_blurred_rounded_rect_in(Circle(dx + 210, 150, 40), Affine.IDENTITY, Rect(dx + 180, 120, 240, 180), c4, 6.0, 4.0))
    pop()
    pop()
    # destructive composes over what is below them
    push(lambda s: s.push_layer(FILL_NON_ZERO, 0, COMPOSE_CLEAR, 1.0, Affine.IDENTITY, Rect(dx + 30, 20, 90, 60)))
    c5 = col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c5, None, Circle(dx + 60, 40, 15)))
    pop()
    push(lambda s: s.push_layer(FILL_NON_ZERO, 0, COMPOSE_COPY, 0.9, Affine.IDENTITY, Circle(dx + 300, 90, 40)))
    c6 = col()
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c6, None, Rect(dx + 280, 60, 340, 120)))
    pop()
    # a luminance mask, and a screen layer
    push(lambda s: s.push_luminance_mask_layer(FILL_NON_ZERO, 1.0, Affine.IDENTITY, Rect(dx + 20, 250, 200, 310)))
    draw(lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((dx + 20, 0), (dx + 200, 0), STOPS), None, Rect(dx + 20, 250, 200, 310)))
    pop()
    push(lambda s: s.push_layer(FILL_NON_ZERO, MIX_SCREEN, COMPOSE_SRC_OVER, 1.0, Affine.IDENTITY, Rect(dx + 260, 200, 370, 300)))
    c7 = col()
    draw(lambda s: s.stroke(Stroke(3.0), Affine.IDENTITY, c7, None, Rect(dx + 270, 210, 350, 290)))
    pop()
    for i in range(8):
        c = col()
        draw(lambda s, i=i, c=c: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Circle(dx + 30 + 40 * i, 280, 14)))
    return ops


def build(ops, hidden=(), s=None):
    """The scene of `ops` without the draw objects in `hidden` (a hidden push without its whole layer; a pop is kept with its
    push), and `kept`: the draw object of the full scene that each draw object of the result is."""
    s = Scene() if s is None else s
    base = s.n_draw_objects
    hidden = set(int(k) for k in hidden)
    kept, skip = [], 0
    for k, (kind, f) in enumerate(ops):
        if skip:
            skip += {"push": 1, "pop": -1}.get(kind, 0)
            continue
        if k in hidden and kind == "push":
            skip = 1
            continue
        if k in hidden and kind == "draw":
            continue
        n0 = s.n_draw_objects
        f(s)
        assert s.n_draw_objects == n0 + 1, k
        kept.append(base + k)
    return s, kept


def closed(ops, hidden):
    """`hidden` with every draw object inside a hidden layer: the draws whose tags a frame does not flatten. A hidden layer's
    own draws are flattened unless they are hidden too; its empty clip then keeps them out of every pixel."""
    out, skip = set(hidden), 0
    for k, (kind, _) in enumerate(ops):
        if skip:
            out.add(k)
            skip += {"push": 1, "pop": -1}.get(kind, 0)
        elif kind == "push" and k in hidden:
            skip = 1
    return out


def layers(ops):
    return [k for k, (kind, _) in enumerate(ops) if kind == "push"]


def flags_of(n, hidden):
    f = np.ones(n, dtype=np.uint8)
    f[list(hidden)] = 0
    return f


def on_device(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def frame(r, aa=AA_MSAA16, w=W, h=H):
    p = RenderParams(BASE, w, h, aa)
    st = r.render_resident(p)
    return r.download_target(p), st


def same(img, want, aa):
    if aa == AA_AREA:
        assert_pixels(img, want, aa)
    else:
        assert (img == want).all()


def sorted_lines(r):
    """The frame's lines as sorted (x0, y0, x1, y1) bit patterns: the geometry flatten emitted, whatever its paths' indices."""
    a = r.download("lines", np.uint32).reshape(-1, 6)[:, 2:]
    return a[np.lexsort(a.T[::-1])]


def masks(ops, n):
    g = np.random.default_rng(5)
    L = layers(ops)
    out = [set(), set(range(n))]  # nothing hidden, everything hidden
    out += [{k} for k in L]  # each layer alone: clip, multiply, the nested clip, clear, copy, luminance mask, screen
    out += [set(np.nonzero(g.uniform(size=n) < q)[0].tolist()) for q in (0.2, 0.5, 0.8)]
    return out


# ---- 1. equality with removal ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_equals_the_scene_without_the_hidden_draws(rr, aa):
    r, ref = rr
    ops = mixed_ops()
    s, _ = build(ops)
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    for hidden in masks(ops, n):
        sub, _ = build(ops, hidden)
        ref.upload(resolve(sub.encoding))
        want, ref_st = frame(ref, aa)
        r.bind_draw_visibility(on_device(flags_of(n, hidden)))
        img, st = frame(r, aa)
        same(img, want, aa)
        assert st.lines >= ref_st.lines  # a hidden layer's own draws are still flattened
        # culling really happens: with a hidden layer's draws hidden too, flatten emits exactly the removal scene's lines
        r.bind_draw_visibility(on_device(flags_of(n, closed(ops, hidden))))
        img, st = frame(r, aa)
        same(img, want, aa)
        assert st.lines == ref_st.lines, sorted(hidden)
        assert np.array_equal(sorted_lines(r), sorted_lines(ref)), sorted(hidden)


def test_hit_tests_and_maps_never_return_a_hidden_draw(rr):
    r, ref = rr
    ops = mixed_ops(seed=2)
    s, _ = build(ops)
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    pts = np.random.default_rng(6).uniform(0, [W, H], (5000, 2)).astype(np.float32)
    for hidden in masks(ops, n)[2:]:
        r.bind_draw_visibility(on_device(flags_of(n, hidden)))
        frame(r, AA_AREA)
        sub, kept = build(ops, hidden)
        ref.upload(resolve(sub.encoding))
        frame(ref, AA_AREA)
        idx = np.array(kept + [-1], dtype=np.int32)  # removal index -> full index; -1 stays -1
        got, want = r.hit_test(pts), ref.hit_test(pts)
        assert (got == idx[want]).all(), sorted(hidden)
        assert not np.isin(got, list(hidden)).any()
        assert (r.hit_map() == idx[ref.hit_map()]).all(), sorted(hidden)


# ---- 2. rows: updates on the stream, strided and bool rows, a short array, re-runs -------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    ops = mixed_ops(seed=3)
    s, _ = build(ops)
    n = s.n_draw_objects
    packed = resolve(s.encoding)
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [flags_of(n, ms) for ms in masks(ops, n)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(n, dtype=torch.uint8, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_draw_visibility(t)
    caps = None
    for j, f in enumerate(seq):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        assert st.kernel_launches == unbound + 1
        ref.upload(resolve(build(ops, np.nonzero(f == 0)[0])[0].encoding))
        assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    # another pointer is another key: a new capture
    t2 = t.clone()
    torch.cuda.synchronize()
    r.bind_draw_visibility(t2)
    r.render_resident(p)
    assert r.debug_graph_captures() == caps + 1
    # unbound again: the launches, config and graph of a renderer that never bound
    r.bind_draw_visibility(None)
    ref.upload(packed)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)  # VbConfig's arena capacities only grow
    again[arenas] = cfg[arenas] = 0
    assert np.array_equal(again, cfg)


def test_strided_bool_and_short_rows_and_reruns(rr):
    r, ref = rr
    ops = mixed_ops(seed=4)
    s, _ = build(ops)
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    g = np.random.default_rng(7)
    f = (g.uniform(size=n) < 0.6).astype(np.uint8) * g.integers(1, 256, n).astype(np.uint8)  # any nonzero byte shows
    hidden = set(np.nonzero(f == 0)[0].tolist())
    ref.upload(resolve(build(ops, hidden)[0].encoding))
    want, _ = frame(ref)
    state = torch.zeros((n, 3), dtype=torch.uint8, device="cuda")
    state[:, 1] = torch.from_numpy(f).cuda()
    torch.cuda.synchronize()
    r.bind_draw_visibility(state[:, 1])  # a column: rows 3 bytes apart
    assert (frame(r)[0] == want).all()
    r.bind_draw_visibility(on_device(f != 0))  # bool
    assert (frame(r)[0] == want).all()
    # a row going from 1 to 2 changes nothing
    r.bind_draw_visibility(on_device(np.where(f != 0, 2, 0).astype(np.uint8)))
    assert (frame(r)[0] == want).all()
    # n below n_draw_objects: the rest are shown
    m = n - 9
    r.bind_draw_visibility(on_device(f[:m]))
    ref.upload(resolve(build(ops, {k for k in hidden if k < m})[0].encoding))
    want_m, _ = frame(ref)
    assert (frame(r)[0] == want_m).all()
    # a range that contains flatten reads the rows again
    p = RenderParams(BASE, W, H, AA_MSAA16)
    t = on_device(f)
    r.bind_draw_visibility(t)
    r.run_stages(p, "pathtag", "flatten")
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.run_stages(p, "draw", "fine", out.data_ptr())
    assert (out.cpu().numpy() == want).all()
    # a blocking frame re-run after an arena overflow reads them again
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    try:
        st = r.render_resident(p)
        assert st.retries == 1
        assert (r.download_target(p) == want).all()
    finally:
        r.limit_arena("lines", 0xFFFFFFFF)
    # an enqueued frame
    out.zero_()
    r.enqueue(p, out.data_ptr())
    r.finish()
    assert (out.cpu().numpy() == want).all()


# ---- 3. with other features ------------------------------------------------------------------------------------------------
def test_view_hides_tags_right_of_the_frame(rr):
    r, ref = rr
    ops = mixed_ops(seed=8)
    s, _ = build(ops)
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    # zoomed in on the left: most draws lie right of the frame, where a shown tag leaves only a box point
    view = Affine.translate(-10, -40) * Affine.scale(2.2)
    r.set_view(view)
    ref.set_view(view)
    try:
        for hidden in masks(ops, n)[2:]:
            r.bind_draw_visibility(on_device(flags_of(n, hidden)))
            img, st = frame(r)
            ref.upload(resolve(build(ops, hidden)[0].encoding))
            want, ref_st = frame(ref)
            assert (img == want).all(), sorted(hidden)
            assert st.lines >= ref_st.lines
            r.bind_draw_visibility(on_device(flags_of(n, closed(ops, hidden))))
            img, st = frame(r)
            assert (img == want).all() and st.lines == ref_st.lines, sorted(hidden)
            assert np.array_equal(r.download("draw_bboxes", np.float32).reshape(-1, 4)[build(ops, hidden)[1]],
                                  ref.download("draw_bboxes", np.float32).reshape(-1, 4)), sorted(hidden)
    finally:
        r.set_view(None)
        ref.set_view(None)


def test_batch_global_rows(rr):
    r, ref = rr
    cells = [mixed_ops(seed=k) for k in range(3)]
    whole, offs = Scene(), [0]
    for c in cells:
        build(c, s=whole)
        offs.append(whole.n_draw_objects)
    n = whole.n_draw_objects
    hidden = set(np.nonzero(np.random.default_rng(9).uniform(size=n) < 0.4)[0].tolist()) | {offs[1] + layers(cells[1])[0]}
    r.upload(resolve(whole.encoding))
    r.bind_draw_visibility(on_device(flags_of(n, hidden)))
    r.set_cells(offs)
    sub, new_offs = Scene(), [0]
    for c, o in zip(cells, offs):
        build(c, {k - o for k in hidden if o <= k < o + len(c)}, s=sub)
        new_offs.append(sub.n_draw_objects)
    ref.upload(resolve(sub.encoding))
    ref.set_cells(new_offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()


def test_composed_instances_with_bound_instance_transforms(rr):
    """The per-instance one-liner: flags from an instance mask repeated over the instances' draw counts."""
    r, ref = rr
    frag_ops = [mixed_ops(seed=10 + k) for k in range(3)]
    frags = [build(o)[0] for o in frag_ops]
    inst = [0, 1, 2, 1, 0]
    ids = [r.upload_fragment(f) for f in frags]
    _, offs = r.compose([(ids[i], None) for i in inst])
    xf = rand_rows(len(inst), 11, 60, 40) * np.float32([0.5, 0.5, 0.5, 0.5, 1, 1])
    r.bind_instance_transforms(on_device(xf.astype(np.float32)))
    shown = np.array([True, False, True, True, False])
    counts = torch.from_numpy(np.diff(np.asarray(offs, dtype=np.int64))).cuda()
    mask_inst = torch.from_numpy(shown).cuda()
    r.bind_draw_visibility(mask_inst.repeat_interleave(counts))
    host = Scene()
    for k, i in enumerate(inst):
        if shown[k]:
            host.append(build(frag_ops[i])[0], aff(xf[k]))
    ref.upload(resolve(host.encoding))
    assert (frame(r)[0] == frame(ref)[0]).all()
    # hidden draws inside instances, with global indices
    hidden = {int(offs[0]) + layers(frag_ops[0])[1], int(offs[2]) + 3, int(offs[3]) + 0}
    flags = np.repeat(shown, np.diff(offs)).astype(np.uint8)
    flags[list(hidden)] = 0
    r.bind_draw_visibility(on_device(flags))
    host = Scene()
    for k, i in enumerate(inst):
        if shown[k]:
            inner = {h - int(offs[k]) for h in hidden if offs[k] <= h < offs[k + 1]}
            host.append(build(frag_ops[i], inner)[0], aff(xf[k]))
    ref.upload(resolve(host.encoding))
    assert (frame(r)[0] == frame(ref)[0]).all()
    for f in ids:
        r.free_fragment(f)


def test_with_bound_colours_points_and_transforms(rr):
    """All bindings at once: colours (non-finite rows keep the encoded ones), points and transforms bound to their encoded
    values. A hidden path stays hidden while its points and transforms are read from rows."""
    r, ref = rr
    ops = mixed_ops(seed=12)
    s, _ = build(ops)
    n = s.n_draw_objects
    packed = resolve(s.encoding)
    r.upload(packed)
    cols = on_device(np.full((n, 4), np.nan, dtype=np.float32))
    pts = on_device(points(packed))
    trs = on_device(transforms(packed))
    r.bind_draw_colors(cols)
    r.bind_path_points(pts)
    r.bind_transforms(trs)
    for hidden in masks(ops, n)[2:]:
        r.bind_draw_visibility(on_device(flags_of(n, hidden)))
        img, st = frame(r)
        ref.upload(resolve(build(ops, hidden)[0].encoding))
        want, ref_st = frame(ref)
        assert (img == want).all(), sorted(hidden)
        r.bind_draw_visibility(on_device(flags_of(n, closed(ops, hidden))))
        img, st = frame(r)
        assert (img == want).all() and st.lines == ref_st.lines, sorted(hidden)
    r.bind_draw_colors(None)
    r.bind_path_points(None)
    r.bind_transforms(None)
    r.bind_draw_visibility(None)


# ---- 4. damage tracking ----------------------------------------------------------------------------------------------------
def damage_ops():
    """Neighbouring sprites, and a layer holding two of its own."""
    ops = []
    for k in range(6):
        x, y = 30 + 55 * k, 40 + 70 * (k % 2)
        c = Color(0.9, 0.15 * k, 0.2, 1.0)
        ops.append(("draw", lambda s, x=x, y=y, c=c: s.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, RoundedRect(x, y, x + 40, y + 40, 6))))
    ops.append(("push", lambda s: s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.9, Affine.IDENTITY, Circle(200, 240, 60))))
    ops.append(("draw", lambda s: s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.8, 0.3, 1.0), None, Rect(150, 200, 260, 260))))
    ops.append(("draw", lambda s: s.stroke(Stroke(4.0), Affine.IDENTITY, Color(0.1, 0.1, 0.9, 1.0), None, Circle(200, 240, 40))))
    ops.append(("pop", lambda s: s.pop_layer()))
    return ops


def test_damage_follows_the_visibility(rr):
    r, ref = rr
    ops = damage_ops()
    s, _ = build(ops)
    n = s.n_draw_objects
    r.upload(resolve(s.encoding))
    f = np.ones(n, dtype=np.uint8)
    t = on_device(f)
    r.bind_draw_visibility(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)

    def step(new=None):
        nonlocal f
        if new is not None:
            f = new.astype(np.uint8)
            t.copy_(torch.from_numpy(f))
            torch.cuda.synchronize()
        r.render_resident(p, dst.data_ptr())
        ref.upload(resolve(build(ops, np.nonzero(f == 0)[0])[0].encoding))
        assert (dst.cpu().numpy() == frame(ref)[0]).all()  # every incremental frame equals a full one
        return r.last_damage()

    try:
        assert step().sum() == n_tiles
        assert step().sum() == 0
        layer = layers(ops)[0]
        for k in [1, 2, layer, layer, 8, 1, 8]:
            before = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            new = f.copy()
            new[k] ^= 1
            got = step(new)
            after = r.download("draw_bboxes", np.float32).reshape(-1, 4)
            want = box_tiles(before[[k]], W, H) | box_tiles(after[[k]], W, H)
            assert want.any() and (got == want).all(), k
            if k == 1:  # only the toggled neighbour's box
                assert not (got & box_tiles(after[[0]], W, H) & ~box_tiles(before[[1]], W, H)).any()
        # a row going from 1 to 2 is no change
        assert step(np.where(f != 0, 2, 0)).sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_draw_visibility(None)


def test_upload_diff_after_a_bound_base_is_full(rr):
    r, ref = rr
    ops = damage_ops()
    s, _ = build(ops)
    packed = resolve(s.encoding)
    r.upload(packed)
    r.bind_draw_visibility(on_device(flags_of(s.n_draw_objects, {2})))
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        r.render_resident(p, dst.data_ptr())
        r.set_upload_diff(True)
        r.upload(packed)  # diffed against a base that hid a draw: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        ref.upload(packed)
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload(packed)  # an unbound base: the same upload damages nothing
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == 0
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 5. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_draw_visibility(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding_and_installations_unbind(rr):
    r, ref = rr
    ops = mixed_ops(seed=13)
    s, _ = build(ops)
    n = s.n_draw_objects
    packed = resolve(s.encoding)
    r.upload(packed)
    hidden = set(range(0, n, 3))
    t = on_device(flags_of(n, hidden))
    r.bind_draw_visibility(t)
    before, _ = frame(r)
    ref.upload(resolve(build(ops, hidden)[0].encoding))
    assert (before == frame(ref)[0]).all()

    def unchanged(what):
        assert r.lib.vb_last_error(r.handle), what
        assert (frame(r)[0] == before).all(), what

    ptr = t.data_ptr()
    host = np.zeros(n, dtype=np.uint8)
    for args in ((ptr, 0, 1), (ptr, n + 1, 1), (host.ctypes.data, n, 1), (ptr, n, 0), (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        unchanged(args)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    assert _bind_raw(r, ptr, n, 1) == VB_E_INVALID  # between enqueue and finish
    r.finish()
    assert (r.download_target(p) == before).all()
    x = Renderer()
    try:
        assert _bind_raw(x, ptr, 1, 1) == VB_E_INVALID and b"scene" in x.lib.vb_last_error(x.handle)
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        assert _bind_raw(x, ptr, n, 1) == VB_E_INVALID and b"exchange" in x.lib.vb_last_error(x.handle)
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        assert _bind_raw(g.renderer(0), ptr, 1, 1) == VB_E_INVALID
    finally:
        g.close()
    assert (frame(r)[0] == before).all()
    # every installation unbinds; None unbinds
    ref.upload(packed)
    encoded, _ = frame(ref)
    fid = r.upload_fragment(s)
    installs = [lambda: r.upload(packed), lambda: r.upload_scene(s), lambda: r.render_to_texture(packed, p),
                lambda: list(r.render_stream([packed], p)), lambda: r.recompose([(fid, None)]), lambda: r.compose([(fid, None)])]
    for install in installs:
        r.compose([(fid, None)])
        r.bind_draw_visibility(t)
        assert (frame(r)[0] == before).all()
        install()
        assert (frame(r)[0] == encoded).all()
    r.free_fragment(fid)
    r.upload(packed)
    r.bind_draw_visibility(t)
    r.bind_draw_visibility(None)
    assert (frame(r)[0] == encoded).all()
