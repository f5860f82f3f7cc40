"""Bound instance transforms (Renderer.bind_instance_transforms, vb_bind_instance_transforms): after a compose, every frame
renders instance k under row k of a device array, read when the frame runs. `r` binds; `ref` takes the compose route, composing
the same fragments with `Affine(row)` for every instance, and every frame of `r` must equal it. Run on an H100 with
`pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import Color, FILL_NON_ZERO, Scene
from vello_b200.renderer import Renderer, RendererGroup, VelloB200Error
from vello_b200.shapes import Affine, Rect

from .test_gpu_compose import BASE, _render_cells, frame, host_packed, mixed_fragments, mixed_instances, upload_all
from .test_gpu_parity import assert_pixels

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 512, 384
VB_E_INVALID = -1


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


def rand_rows(n, seed, w=W, h=H):
    """n random f32 affines: rotation, shear, reflection, scale and translation."""
    g = np.random.default_rng(seed)
    th, sh = g.uniform(-np.pi, np.pi, n), g.uniform(-0.4, 0.4, n)
    sx, sy = g.uniform(0.5, 1.5, n) * g.choice([-1.0, 1.0], n), g.uniform(0.5, 1.5, n)
    c, s = np.cos(th), np.sin(th)  # rotate(th) * shear(sh) * scale(sx, sy)
    rows = np.stack([c * sx, s * sx, (c * sh - s) * sy, (s * sh + c) * sy, g.uniform(0, w, n), g.uniform(0, h, n)], 1)
    return rows.astype(np.float32)


def aff(row):
    return Affine(tuple(float(v) for v in row))


def on_device(rows):
    t = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    torch.cuda.synchronize()
    return t


def stream_of(r):
    return torch.cuda.ExternalStream(r.stream)


class Setup:
    """The mixed fragments uploaded to both renderers; `r` composed with mixed_instances."""

    def __init__(self, r, ref, frags=None, inst=None):
        self.r, self.ref = r, ref
        self.frags = frags if frags is not None else mixed_fragments()
        self.inst = inst if inst is not None else mixed_instances(len(self.frags))
        self.ids, self.rids = upload_all(r, self.frags), upload_all(ref, self.frags)
        self.lay, self.offs = r.compose([(self.ids[i], t) for i, t in self.inst])

    def compose_ref(self, rows, keep=()):
        """The compose route: instance k as Affine(rows[k]), or as composed for k in `keep`."""
        return self.ref.compose([(self.rids[i], t if k in keep else aff(rows[k])) for k, (i, t) in enumerate(self.inst)])

    def free(self):
        for i in self.ids:
            self.r.free_fragment(i)
        for i in self.rids:
            self.ref.free_fragment(i)


def same_frame(img, want, aa):
    if aa == AA_AREA:
        assert_pixels(img, want, aa)
    else:
        assert (img == want).all()


# ---- 1. equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16, AA_AREA])
def test_bound_equals_compose_route(rr, aa):
    r, ref = rr
    s = Setup(r, ref)
    rows = rand_rows(len(s.inst), 1)
    r.bind_instance_transforms(on_device(rows))
    img = frame(r, W, H, aa)
    s.compose_ref(rows)
    want = frame(ref, W, H, aa)
    got_tr = r.download("transforms", np.uint32)
    assert got_tr.size > 0 and np.array_equal(got_tr, ref.download("transforms", np.uint32))
    packed, _ = host_packed(s.frags, [(i, aff(rows[k])) for k, (i, _) in enumerate(s.inst)])
    assert np.array_equal(got_tr, packed.scene[packed.layout.transform_base:packed.layout.style_base])
    for name in ("path_bboxes", "draw_bboxes", "draw_monoids"):
        assert np.array_equal(r.download(name, np.uint32), ref.download(name, np.uint32)), name
    same_frame(img, want, aa)
    s.free()


# ---- 2. updates without calls ----------------------------------------------------------------------------------------------
def test_updates_on_the_stream_replay_the_graph(rr):
    r, ref = rr
    s = Setup(r, ref)
    n = len(s.inst)
    p = RenderParams(BASE, W, H, AA_MSAA16)
    seq = [rand_rows(n, 100 + j) for j in range(20)]
    all_rows = on_device(np.stack(seq))
    t = torch.empty((n, 6), dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_instance_transforms(t)
    caps = None
    for j in range(20):
        with torch.cuda.stream(stream_of(r)):
            t.copy_(all_rows[j])
        st = r.render_resident(p)
        img = r.download_target(p)
        if caps is None:
            caps = r.debug_graph_captures()
        assert r.debug_graph_captures() == caps, f"frame {j} captured a graph"
        s.compose_ref(seq[j])
        ref_st = ref.render_resident(p)
        assert st.kernel_launches == ref_st.kernel_launches + 1
        assert (img == ref.download_target(p)).all(), f"frame {j}"
    for j in range(5):  # enqueue / finish, ordered only by the stream
        with torch.cuda.stream(stream_of(r)):
            t.copy_(all_rows[19 - j])
        r.enqueue(p)
        r.finish()
        s.compose_ref(seq[19 - j])
        assert (r.download_target(p) == frame(ref, W, H, AA_MSAA16)).all(), f"enqueued frame {j}"
    s.free()


# ---- 3. a view on top ------------------------------------------------------------------------------------------------------
def test_view_on_top(rr):
    r, ref = rr
    s = Setup(r, ref)
    rows = rand_rows(len(s.inst), 2)
    r.bind_instance_transforms(on_device(rows))
    s.compose_ref(rows)
    view = Affine.translate(-40, 25) * Affine.scale(1.4) * Affine.rotate(0.1)
    r.set_view(view)
    ref.set_view(view)
    try:
        img, want = frame(r, W, H, AA_MSAA16), frame(ref, W, H, AA_MSAA16)
        assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
        assert r.download("bump", np.uint32)[7] == ref.download("bump", np.uint32)[7], "culled lines differ"
        assert (img == want).all()
    finally:
        r.set_view(None)
        ref.set_view(None)
    assert (frame(r, W, H, AA_MSAA16) == frame(ref, W, H, AA_MSAA16)).all(), "the binding survives the view"
    s.free()


# ---- 4. cells and hit testing ----------------------------------------------------------------------------------------------
def test_hit_test_and_cells(rr):
    r, ref = rr
    frags = mixed_fragments()
    open_clips = 10  # cells must balance their clips: leave out the fragment with open clips
    s = Setup(r, ref, frags, [(i, t) for i, t in mixed_instances(len(frags)) if i != open_clips])
    rows = rand_rows(len(s.inst), 3, 200, 160)
    r.bind_instance_transforms(on_device(rows))
    _, ref_offs = s.compose_ref(rows)
    assert ref_offs == s.offs
    frame(r, W, H, AA_AREA)
    frame(ref, W, H, AA_AREA)
    pts = np.random.default_rng(4).uniform(0, [W, H], (6000, 2)).astype(np.float32)
    got = r.hit_test(pts)
    assert (got >= 0).sum() > 100 and (got == ref.hit_test(pts)).all()
    r.set_cells(s.offs)
    ref.set_cells(ref_offs)
    n = len(s.offs) - 1
    assert (_render_cells(r, n, 200, 160, AA_MSAA16) == _render_cells(ref, n, 200, 160, AA_MSAA16)).all()
    s.free()


# ---- 5. a blocking frame re-run after an overflow --------------------------------------------------------------------------
def test_rerun_reads_the_same_rows(rr):
    r, ref = rr
    s = Setup(r, ref)
    rows = rand_rows(len(s.inst), 5)
    r.bind_instance_transforms(on_device(rows))
    p = RenderParams(BASE, W, H, AA_MSAA16)
    st0 = r.render_resident(p)
    r.limit_arena("lines", int(st0.lines) - 1)
    st = r.render_resident(p)
    assert st.retries == 1 and st.lines == st0.lines
    s.compose_ref(rows)
    assert (r.download_target(p) == frame(ref, W, H, AA_MSAA16)).all()
    s.free()


# ---- 6. rows that are not finite -------------------------------------------------------------------------------------------
def test_non_finite_rows_keep_the_composed_transform(rr):
    r, ref = rr
    s = Setup(r, ref)
    assert s.inst[0][1] is None and s.inst[6][1] is None and s.inst[2][1] is not None and s.inst[4][1] is not None
    rows = rand_rows(len(s.inst), 6)
    bad = {0: (4, np.nan), 6: (0, np.inf), 2: (3, -np.inf), 4: (1, np.nan), 3: (5, np.inf)}  # instance: (coefficient, value)
    for k, (c, v) in bad.items():
        rows[k, c] = v
    r.bind_instance_transforms(on_device(rows))
    s.compose_ref(rows, keep=set(bad))
    for aa in (AA_MSAA16, AA_AREA):
        img, want = frame(r, W, H, aa), frame(ref, W, H, aa)
        assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
        same_frame(img, want, aa)
    s.free()


# ---- 7. strided rows -------------------------------------------------------------------------------------------------------
def test_column_slice_of_a_state_tensor(rr):
    r, ref = rr
    s = Setup(r, ref)
    rows = rand_rows(len(s.inst), 7)
    state = torch.zeros((len(s.inst), 8), dtype=torch.float32, device="cuda")
    state[:, 2:8] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    r.bind_instance_transforms(state[:, 2:8])
    img = frame(r, W, H, AA_MSAA16)
    r.bind_instance_transforms(on_device(rows))
    assert (img == frame(r, W, H, AA_MSAA16)).all()
    s.compose_ref(rows)
    assert (img == frame(ref, W, H, AA_MSAA16)).all()
    s.free()


# ---- 8. lifetime and clearing ----------------------------------------------------------------------------------------------
def test_free_unbind_and_new_scenes(rr):
    r, ref = rr
    s = Setup(r, ref)
    rows = rand_rows(len(s.inst), 8)
    r.bind_instance_transforms(on_device(rows))
    bound = frame(r, W, H, AA_MSAA16)
    for i in s.ids:
        r.free_fragment(i)
    assert (frame(r, W, H, AA_MSAA16) == bound).all(), "freeing the fragments changed a bound frame"
    # unbound: the composed scene, with the launches, config and graphs of a renderer that was never bound
    r.bind_instance_transforms(None)
    ref.compose([(s.rids[i], t) for i, t in s.inst])
    p = RenderParams(BASE, W, H, AA_MSAA16)
    st, ref_st = r.render_resident(p), ref.render_resident(p)
    assert (r.download_target(p) == ref.download_target(p)).all()
    assert st.kernel_launches == ref_st.kernel_launches
    assert np.array_equal(r.download("config", np.uint32), ref.download("config", np.uint32))
    caps = r.debug_graph_captures()
    r.render_resident(p)
    assert r.debug_graph_captures() == caps
    # a compose and an upload each unbind
    s.ids = upload_all(r, s.frags)
    r.compose([(s.ids[i], t) for i, t in s.inst])
    r.bind_instance_transforms(on_device(rows))
    moved = [(i, Affine.translate(3, 2)) for i, _ in s.inst]
    r.compose([(s.ids[i], t) for i, t in moved])
    ref.compose([(s.rids[i], t) for i, t in moved])
    assert (frame(r, W, H, AA_MSAA16) == frame(ref, W, H, AA_MSAA16)).all()
    r.compose([(s.ids[i], t) for i, t in s.inst])
    r.bind_instance_transforms(on_device(rows))
    packed, _ = host_packed(s.frags, moved)
    r.upload(packed)
    ref.upload(packed)
    assert (frame(r, W, H, AA_MSAA16) == frame(ref, W, H, AA_MSAA16)).all()
    s.free()


# ---- 9. errors -------------------------------------------------------------------------------------------------------------
def _bind_raw(r, ptr, n, pitch):
    return r.lib.vb_bind_instance_transforms(r.handle, C.c_void_p(ptr), n, pitch)


def test_errors_leave_the_binding(rr):
    r, ref = rr
    s = Setup(r, ref)
    n = len(s.inst)
    rows = rand_rows(n, 9)
    t = on_device(rows)
    r.bind_instance_transforms(t)
    before = frame(r, W, H, AA_MSAA16)

    def check(call):
        with pytest.raises(VelloB200Error, match="invalid"):
            call()
        assert (frame(r, W, H, AA_MSAA16) == before).all()

    check(lambda: r.bind_instance_transforms(on_device(rand_rows(n + 1, 10))))  # n is not the instance count
    ptr = t.data_ptr()
    host = np.zeros((n, 6), dtype=np.float32)
    for args in ((ptr, 0, 24), (host.ctypes.data, n, 24), (ptr + 2, n, 24), (ptr, n, 20), (ptr, n, 26), (ptr, n, 1 << 32)):
        assert _bind_raw(r, *args) == VB_E_INVALID, args
        assert r.lib.vb_last_error(r.handle)
        assert (frame(r, W, H, AA_MSAA16) == before).all(), args
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.enqueue(p)
    with pytest.raises(VelloB200Error, match="invalid"):  # between enqueue and finish
        r.bind_instance_transforms(t)
    r.finish()
    assert (r.download_target(p) == before).all()
    # a fragment of the compose freed before the bind
    extra = r.upload_fragment(s.frags[0])
    r.compose([(s.ids[i], tr) for i, tr in s.inst] + [(extra, None)])
    r.bind_instance_transforms(on_device(rand_rows(n + 1, 11)))  # binds
    composed = [(s.ids[i], tr) for i, tr in s.inst] + [(extra, None)]
    r.compose(composed)
    r.free_fragment(extra)
    unbound = frame(r, W, H, AA_MSAA16)
    with pytest.raises(VelloB200Error, match="freed"):
        r.bind_instance_transforms(on_device(rand_rows(n + 1, 12)))
    assert (frame(r, W, H, AA_MSAA16) == unbound).all()
    # a scene that was not composed
    packed, _ = host_packed(s.frags, s.inst)
    r.upload(packed)
    uploaded = frame(r, W, H, AA_MSAA16)
    with pytest.raises(VelloB200Error, match="vb_compose"):
        r.bind_instance_transforms(t)
    assert (frame(r, W, H, AA_MSAA16) == uploaded).all()
    with pytest.raises(ValueError):  # not (n, 6) float32 with 4-byte columns
        r.bind_instance_transforms(torch.zeros((n, 6), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        r.bind_instance_transforms(torch.zeros((6, n), dtype=torch.float32, device="cuda").t())
    # a renderer of a vb_group, and one with the exchange enabled
    g = RendererGroup([0, 0])
    try:
        with pytest.raises(VelloB200Error, match="invalid"):
            g.renderer(0).bind_instance_transforms(t)
    finally:
        g.close()
    x = Renderer()
    try:
        fid = x.upload_fragment(s.frags[0])
        x.compose([(fid, None)])
        assert x.lib.vb_exchange_configure(x.handle, 0, 1, None, None) == 0 and x.lib.vb_exchange_enable(x.handle, 1) == 0
        assert _bind_raw(x, t.data_ptr(), 1, 24) == VB_E_INVALID
        assert b"exchange" in x.lib.vb_last_error(x.handle)
        x.lib.vb_exchange_enable(x.handle, 0)
        x.free_fragment(fid)
    finally:
        x.close()
    s.free()


# ---- 10. scale -------------------------------------------------------------------------------------------------------------
def test_large_fragment_among_100k_instances(rr):
    r, ref = rr
    big = scenes.paris_like(2500, 1024, seed=5)
    tiny = []
    for k in range(4):
        sc = Scene()
        sc.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(60 * k, 200 - 40 * k, 90, 255), None, Rect(0, 0, 5 + k, 4))
        tiny.append(sc)
    frags = tiny + [big]
    n = 100_000
    inst = [(k % 4, Affine.translate(k % 400 * 5, k // 400 * 8) if k % 7 else None) for k in range(n)]
    inst.insert(n // 2, (4, Affine.scale(1.5)))
    s = Setup(r, ref, frags, inst)
    g = np.random.default_rng(13)
    rows = np.zeros((n + 1, 6), dtype=np.float32)
    th = g.uniform(-0.3, 0.3, n + 1)
    rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3] = np.cos(th), np.sin(th), -np.sin(th), np.cos(th)
    rows[:, 4], rows[:, 5] = g.uniform(0, 2040, n + 1), g.uniform(0, 2040, n + 1)
    rows[n // 2] = (1.8, 0.1, -0.1, 1.8, 40.0, 60.0)
    r.bind_instance_transforms(on_device(rows))
    s.compose_ref(rows)
    img, want = frame(r, 2048, 2048, AA_MSAA16), frame(ref, 2048, 2048, AA_MSAA16)
    assert np.array_equal(r.download("transforms", np.uint32), ref.download("transforms", np.uint32))
    assert (img == want).all()
    s.free()
