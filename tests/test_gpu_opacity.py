"""Bound opacity (Renderer.bind_draw_opacity, vb_bind_draw_opacity): every frame draws layer or image k with the alpha in row k
of a device array, read when the frame runs. `r` binds; `ref` renders the host route on the same GPU: the scene re-encoded with
the rows applied (a clip layer whose row is below 1 as a Normal / SrcOver layer) and uploaded. Run on an H100 with
`pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import Packed, Scene, resolve
from vello_b200.renderer import Renderer, RendererGroup

from .test_gpu_compose import BASE, _render_cells
from .test_gpu_draw_colors import box_tiles
from .test_gpu_path_points import points
from .test_gpu_transforms import transforms
from .test_gpu_visibility import frame, on_device, same
from .test_opacity import build, opacity_ops, opacity_slots, patched, rand_rows
from .parity import tile_streams

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 384, 320
VB_E_INVALID = -1


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


@pytest.fixture
def fresh():
    """Two new renderers: the ptcl holds offsets that follow a renderer's arena history."""
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def raw(r, name):
    return r.download(name, np.uint32)


def commands(r):
    """Each tile's command list, as coarse wrote it: without the offsets that follow the order in which tiles took arena
    space (a list's continuation chunks, a FILL's segment slice and a deep layer's blend-spill slot)."""
    return tile_streams(raw(r, "ptcl"), None, ((W + 15) // 16) * ((H + 15) // 16))


def kinds_of(packed):
    return [s[1] if s else None for s in opacity_slots(packed)]


def host(ops, rows):
    return resolve(build(ops, rows).encoding)


# ---- 1. equality with the re-encoded scene -----------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_equals_the_reencoded_scene(fresh, aa):
    r, ref = fresh
    ops = opacity_ops(seed=1, full_clip=True)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    pts = np.random.default_rng(3).uniform(0, [W, H], (4000, 2)).astype(np.float32)
    for seed, rows in enumerate([rand_rows(n, 10), rand_rows(n, 11), np.full(n, 0.5, np.float32), np.zeros(n, np.float32),
                                 np.ones(n, np.float32)]):
        r.bind_draw_opacity(on_device(rows))
        want_scene = host(ops, rows)
        ref.upload(want_scene)
        img, _ = frame(r, aa)
        want, _ = frame(ref, aa)
        same(img, want, aa)
        assert np.array_equal(raw(r, "draw_data"), raw(ref, "draw_data")), seed
        assert np.array_equal(raw(r, "draw_bboxes"), raw(ref, "draw_bboxes")), seed
        assert commands(r) == commands(ref), seed
        assert (r.hit_test(pts) == ref.hit_test(pts)).all()
        assert (r.hit_map() == ref.hit_map()).all()
    r.bind_draw_opacity(None)


def test_streams_and_native_installations(rr):
    """Scenes installed from their streams, by either front end, bind as packed ones do."""
    from vello_b200.scene_native import NativeScene
    r, ref = rr
    ops = opacity_ops(seed=2)
    s = build(ops)
    ns = build(ops, s=NativeScene())
    rows = rand_rows(s.n_draw_objects, 4)
    ref.upload(host(ops, rows))
    want, _ = frame(ref)
    r.upload_scene(s)
    r.bind_draw_opacity(on_device(rows))
    assert (frame(r)[0] == want).all()
    ns.upload_device(r)
    r.bind_draw_opacity(on_device(rows))
    assert (frame(r)[0] == want).all()
    r.bind_draw_opacity(None)


def test_full_cover_clip_layer_fades_its_interior(fresh):
    """A clip layer covering the whole frame emits nothing in its interior tiles; at row 0.5 it becomes a blend layer and its
    interior fades. At row 1 the ptcl is the unbound frame's."""
    r, ref = fresh
    ops = opacity_ops(seed=5, full_clip=True)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    assert kinds_of(packed)[0] == "clip"
    r.upload(packed)
    ref.upload(packed)
    unbound, _ = frame(ref)
    ptcl0 = commands(ref)
    rows = np.full(n, np.nan, np.float32)
    rows[0] = 1.0
    r.bind_draw_opacity(on_device(rows))
    img, _ = frame(r)
    assert (img == unbound).all() and commands(r) == ptcl0
    rows[0] = 0.5
    r.bind_draw_opacity(on_device(rows))
    img, _ = frame(r)
    ref.upload(host(ops, rows))
    assert (img == frame(ref)[0]).all()
    # every tile lies inside the clip: where a fill covers one, it fades over the base colour
    assert (img[35:50, 90:130] != unbound[35:50, 90:130]).any(2).mean() > 0.9
    assert commands(r) != ptcl0


# ---- 2. rows -----------------------------------------------------------------------------------------------------------------
def test_row_rules(rr):
    r, ref = rr
    ops = opacity_ops(seed=6)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    ref.upload(packed)
    encoded, _ = frame(ref)
    kinds = kinds_of(packed)
    bound = [k for k, x in enumerate(kinds) if x]
    rows = rand_rows(n, 7)
    # NaN and +-inf keep the encoded words
    for j, bad in enumerate((np.nan, np.inf, -np.inf)):
        rows[bound[j::3]] = bad
    r.bind_draw_opacity(on_device(rows))
    ref.upload(host(ops, rows))
    assert (frame(r)[0] == frame(ref)[0]).all()
    assert np.array_equal(raw(r, "draw_data"), patched(packed, rows).scene[packed.layout.draw_data_base:packed.layout.transform_base])
    # rows of colour, gradient and blur draws, END_CLIPs and pops change nothing
    other = np.array([np.nan if x else 0.3 for x in kinds], dtype=np.float32)
    r.bind_draw_opacity(on_device(other))
    assert (frame(r)[0] == encoded).all()
    # a partial n, and a tail of one row: draw objects from n on keep their encoded values
    for m in (n // 2, 1, n):
        r.bind_draw_opacity(on_device(rows[:m]))
        ref.upload(host(ops, rows[:m]))
        assert (frame(r)[0] == frame(ref)[0]).all(), m
    # strided columns, (n, 1) and 1-D tensors
    ref.upload(host(ops, rows))
    want, _ = frame(ref)
    state = torch.zeros((n, 7), dtype=torch.float32, device="cuda")
    state[:, 5] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    for t in (state[:, 5], state[:, 5:6], on_device(rows[:, None]), on_device(rows)):
        r.bind_draw_opacity(t)
        assert (frame(r)[0] == want).all()
    r.bind_draw_opacity(None)


def test_updates_on_the_stream_replay_the_graph_in_one_pass(rr):
    r, ref = rr
    ops = opacity_ops(seed=8)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    unbound = r.render_resident(p).kernel_launches
    cfg = r.download("config", np.uint32)
    seq = [rand_rows(n, 100 + j) for j in range(20)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty(n, dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_draw_opacity(t)
    # a first pass lets the arenas grow to what every row set needs (a clip layer drawn as a blend layer writes more commands)
    for j in range(len(seq)):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        r.render_resident(p)
    caps = r.debug_graph_captures()
    for j, rows in enumerate(seq):
        with torch.cuda.stream(torch.cuda.ExternalStream(r.stream)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        # one pass writes the frame's draw data: the scene's words with the bound opacity words (k_draw_data)
        assert st.kernel_launches == unbound + 1
        if j % 4 == 0:
            ref.upload(host(ops, rows))
            assert (r.download_target(p) == frame(ref)[0]).all(), f"frame {j}"
    bound_cfg = r.download("config", np.uint32)
    t2 = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    t2[:, 1] = t
    torch.cuda.synchronize()
    r.bind_draw_opacity(t2[:, 1])  # another pointer and pitch is another key
    r.render_resident(p)
    assert r.debug_graph_captures() == caps + 1
    r.bind_draw_opacity(None)  # unbound again: what a renderer that never bound launches and configures
    st = r.render_resident(p)
    assert st.kernel_launches == unbound
    again = r.download("config", np.uint32)
    arenas = slice(15, 22)
    again[arenas] = cfg[arenas] = bound_cfg[arenas] = 0
    assert np.array_equal(again, cfg)
    assert not np.array_equal(bound_cfg, cfg)  # bound frames read the draw data from the region past the scene


def test_reruns_split_ranges_views_and_enqueued_frames(rr):
    r, ref = rr
    ops = opacity_ops(seed=9)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    rows = rand_rows(n, 10)
    ref.upload(host(ops, rows))
    want, ref_st = frame(ref)
    r.bind_draw_opacity(on_device(rows))
    st = r.render_resident(p)
    assert (r.download_target(p) == want).all()
    # a blocking frame re-run after an arena overflow
    r.limit_arena("lines", int(st.lines) - 1)
    try:
        st = r.render_resident(p)
        assert st.retries >= 1
        assert (r.download_target(p) == want).all()
    finally:
        r.limit_arena("lines", 0xFFFFFFFF)
    # ranges that start at draw write the draw data again
    for a, b in [("pathtag", "flatten"), ("pathtag", "pathtag")]:
        r.run_stages(p, a, b)
        if b == "pathtag":
            r.run_stages(p, "flatten", "flatten")
        out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        r.run_stages(p, "draw", "fine", out.data_ptr())
        assert (out.cpu().numpy() == want).all(), (a, b)
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    r.enqueue(p, out.data_ptr())
    r.finish()
    assert (out.cpu().numpy() == want).all()
    # a view
    from vello_b200.shapes import Affine
    v = Affine.translate(-40, -25) * Affine.scale(1.6)
    r.set_view(v)
    ref.set_view(v)
    try:
        assert (frame(r)[0] == frame(ref)[0]).all()
    finally:
        r.set_view(None)
        ref.set_view(None)
    r.bind_draw_opacity(None)


# ---- 3. with other features ------------------------------------------------------------------------------------------------
def test_with_every_other_binding(rr):
    """Colours, stops, visibility, transforms, points and widths bound at once (at their encoded values, or moving the
    transforms and points, which the host route patches too) with opacity."""
    r, ref = rr
    ops = opacity_ops(seed=13)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    L = packed.layout
    r.upload_scene(build(ops))  # from its streams: gradient stops can be bound
    rows = rand_rows(n, 14)
    tr = transforms(packed)
    tr[:, 4:] += np.float32(5.0)
    pts = points(packed) + np.float32(1.25)
    r.bind_draw_colors(on_device(np.full((n, 4), np.nan, dtype=np.float32)))
    r.bind_gradient_stops(on_device(np.full((1, 5), np.nan, dtype=np.float32)))
    r.bind_draw_visibility(on_device(np.ones(n, dtype=np.uint8)))
    r.bind_transforms(on_device(tr))
    r.bind_path_points(on_device(pts))
    r.bind_stroke_widths(on_device(np.full(n, np.nan, dtype=np.float32)))
    r.bind_draw_opacity(on_device(rows))
    want = host(ops, rows)
    sc = np.array(want.scene, dtype=np.uint32)
    sc[L.transform_base:L.style_base] = tr.reshape(-1).view(np.uint32)
    sc[L.path_data_base:L.path_data_base + pts.size] = pts.reshape(-1).view(np.uint32)
    ref.upload(Packed(sc, L, want.ramps, want.atlas))
    assert (frame(r)[0] == frame(ref)[0]).all()
    # a bound colour and opacity on the same frame: the colour row of a fill applies, its opacity row does not
    cols = np.full((n, 4), np.nan, dtype=np.float32)
    k = next(i for i, (kind, _, _) in enumerate(ops) if kind == "draw")
    cols[k] = [0.1, 0.9, 0.2, 0.6]
    r.bind_draw_colors(on_device(cols))
    ref.bind_draw_colors(on_device(cols))
    assert (frame(r)[0] == frame(ref)[0]).all()
    ref.bind_draw_colors(None)
    for b in ("bind_draw_colors", "bind_gradient_stops", "bind_draw_visibility", "bind_transforms", "bind_path_points",
              "bind_stroke_widths", "bind_draw_opacity"):
        getattr(r, b)(None)


def test_composed_instances_and_batches_use_global_rows(rr):
    r, ref = rr
    frag_ops = [opacity_ops(seed=20 + k) for k in range(2)]
    inst = [0, 1, 0]
    ids = [r.upload_fragment(build(o)) for o in frag_ops]
    _, offs = r.compose([(ids[i], None) for i in inst])
    n = int(offs[-1])
    rows = rand_rows(n, 22)
    r.bind_draw_opacity(on_device(rows))
    whole = Scene()
    for k, i in enumerate(inst):
        whole.append(build(frag_ops[i], rows[int(offs[k]):int(offs[k + 1])]))
    ref.upload(resolve(whole.encoding))
    assert (frame(r)[0] == frame(ref)[0]).all()
    r.bind_draw_opacity(None)
    for f in ids:
        r.free_fragment(f)
    # a batch: rows are global, in cell order
    cells = [opacity_ops(seed=30 + k) for k in range(3)]
    whole, cell_offs = Scene(), [0]
    for c in cells:
        build(c, s=whole)
        cell_offs.append(whole.n_draw_objects)
    rows = rand_rows(whole.n_draw_objects, 31)
    r.upload(resolve(whole.encoding))
    r.bind_draw_opacity(on_device(rows))
    r.set_cells(cell_offs)
    want = Scene()
    for j, c in enumerate(cells):
        build(c, rows[cell_offs[j]:cell_offs[j + 1]], s=want)
    ref.upload(resolve(want.encoding))
    ref.set_cells(cell_offs)
    assert (_render_cells(r, 3, W, H, AA_MSAA16) == _render_cells(ref, 3, W, H, AA_MSAA16)).all()
    r.bind_draw_opacity(None)


def test_hit_tests_and_maps_do_not_change(rr):
    r, ref = rr
    ops = opacity_ops(seed=40, full_clip=True)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    ref.upload(packed)
    frame(ref)
    pts = np.random.default_rng(41).uniform(0, [W, H], (3000, 2)).astype(np.float32)
    want, want_map = ref.hit_test(pts), ref.hit_map()
    for v in (0.0, 1.0):
        r.bind_draw_opacity(on_device(np.full(n, v, np.float32)))
        frame(r)
        assert (r.hit_test(pts) == want).all(), v
        assert (r.hit_map() == want_map).all(), v
    r.bind_draw_opacity(None)


# ---- 4. damage tracking ----------------------------------------------------------------------------------------------------
def test_damage_is_the_boxes_of_changed_layers_and_images(rr):
    r, ref = rr
    ops = opacity_ops(seed=50, full_clip=False)
    packed = host(ops, ())
    n = packed.layout.n_draw_objects
    r.upload(packed)
    kinds = kinds_of(packed)
    rows = np.full(n, np.nan, dtype=np.float32)
    t = on_device(rows)
    r.bind_draw_opacity(t)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)

    def step(new):
        t.copy_(torch.from_numpy(new))
        torch.cuda.synchronize()
        r.render_resident(p, dst.data_ptr())
        ref.upload(host(ops, new))
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        return r.last_damage(), r.download("draw_bboxes", np.float32).reshape(-1, 4)

    try:
        assert step(rows)[0].sum() == n_tiles
        assert step(rows)[0].sum() == 0
        layers = [k for k, x in enumerate(kinds) if x == "layer"]
        clips = [k for k, x in enumerate(kinds) if x == "clip"]
        images = [k for k, x in enumerate(kinds) if x == "image"]
        cur = rows.copy()
        for ch, v in (([layers[0]], 0.4), ([images[1]], 0.3), ([clips[0]], 0.5), ([layers[2], images[0]], 0.0), ([clips[0]], 1.0)):
            new = cur.copy()
            new[ch] = np.float32(v)
            got, boxes = step(new)
            want = box_tiles(boxes[ch], W, H)
            assert want.any() and (got == want).all(), ch
            cur = new
        # unchanged words: a row converting to the same byte, a NaN over an encoded value, ignored rows
        new = cur.copy()
        new[images[1]] = np.float32(0.3) + np.float32(1e-4)  # the same byte as 0.3
        assert step(new)[0].sum() == 0
        cur = new
        new = cur.copy()
        new[clips[0]] = np.nan  # back to the encoded clip layer, which row 1 left as encoded
        new[[k for k, x in enumerate(kinds) if x is None]] = 0.2
        assert step(new)[0].sum() == 0
    finally:
        r.set_damage_tracking(False)
        r.bind_draw_opacity(None)


def test_upload_diff_and_recompose_after_a_bound_base_are_full(rr):
    r, ref = rr
    ops = opacity_ops(seed=51)
    s = build(ops)
    packed = resolve(s.encoding)
    n = packed.layout.n_draw_objects
    r.upload(packed)
    r.bind_draw_opacity(on_device(rand_rows(n, 52)))
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    n_tiles = ((W + 15) // 16) * ((H + 15) // 16)
    r.set_damage_tracking(True)
    try:
        r.render_resident(p, dst.data_ptr())
        r.render_resident(p, dst.data_ptr())
        r.set_upload_diff(True)
        r.upload(packed)  # diffed against a base with bound opacity: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        ref.upload(packed)
        assert (dst.cpu().numpy() == frame(ref)[0]).all()
        r.upload(packed)  # an unbound base: nothing
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == 0
        r.set_upload_diff(False)
        fid = r.upload_fragment(s)
        r.compose([(fid, None)])
        r.render_resident(p, dst.data_ptr())
        r.bind_draw_opacity(on_device(rand_rows(n, 53)))
        r.render_resident(p, dst.data_ptr())
        r.recompose([(fid, None)])  # a bound base: full
        r.render_resident(p, dst.data_ptr())
        assert r.last_damage().sum() == n_tiles
        r.free_fragment(fid)
    finally:
        r.set_upload_diff(False)
        r.set_damage_tracking(False)


# ---- 5. errors, installations and unbinding --------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_draw_opacity(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding_and_installations_unbind(rr):
    r, ref = rr
    ops = opacity_ops(seed=60)
    s = build(ops)
    packed = resolve(s.encoding)
    n = packed.layout.n_draw_objects
    r.upload(packed)
    rows = rand_rows(n, 61)
    t = on_device(rows)
    r.bind_draw_opacity(t)
    before, _ = frame(r)
    ref.upload(host(ops, rows))
    assert (before == frame(ref)[0]).all()

    def refused(x, args, word):
        assert _bind_raw(x, *args) == VB_E_INVALID, args
        msg = x.lib.vb_last_error(x.handle)
        assert msg.startswith(b"vb_bind_draw_opacity: ") and word in msg, (args, msg)

    ptr = t.data_ptr()
    hostmem = np.zeros(n, dtype=np.float32)
    for args, word in (((ptr, 0, 4), b"rows"), ((ptr, n + 1, 4), b"rows"), ((hostmem.ctypes.data, n, 4), b"device"),
                       ((ptr + 2, n - 1, 4), b"aligned"), ((ptr, n, 0), b"pitch"), ((ptr, n, 2), b"pitch"), ((ptr, n, 6), b"pitch"),
                       ((ptr, n, 1 << 32), b"pitch")):
        refused(r, args, word)
        assert (frame(r)[0] == before).all(), args
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    refused(r, (ptr, n, 4), b"enqueued")
    r.finish()
    assert (r.download_target(p) == before).all()
    x = Renderer()
    try:
        refused(x, (ptr, 1, 4), b"scene")
        x.upload(packed)
        nbytes, arena = C.c_size_t(0), C.c_void_p()
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, C.byref(arena), C.byref(nbytes)) == 0
        refused(x, (ptr, n, 4), b"exchange")
    finally:
        x.close()
    g = RendererGroup([0, 0])
    try:
        refused(g.renderer(0), (ptr, 1, 4), b"vb_group")
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
        r.bind_draw_opacity(t)
        assert (frame(r)[0] == before).all()
        install()
        assert (frame(r)[0] == encoded).all()
    r.free_fragment(fid)
    r.upload(packed)
    r.bind_draw_opacity(t)
    r.bind_draw_opacity(None)
    assert (frame(r)[0] == encoded).all()
