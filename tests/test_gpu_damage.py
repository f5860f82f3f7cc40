"""Damage tracking (Renderer.set_damage_tracking / add_damage / last_damage, vb_set_damage_tracking / vb_add_damage /
vb_last_damage): a frame into the destination of the last successful frame repaints only its damaged tiles and writes no other
pixel. `r` tracks; `ref` renders the same composition with the same bound rows and tracking off, always in full, and every
frame of `r` must equal it byte for byte. Run on an H100 with `pytest -m gpu`."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import Color, FILL_NON_ZERO, resolve
from vello_b200.renderer import Renderer, RendererGroup, VelloB200Error
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Rect

from .test_gpu_compose import BASE, mixed_fragments, mixed_instances, upload_all
from .test_gpu_instance_transforms import rand_rows

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 512, 384
SENTINEL = 0x5A


@pytest.fixture(scope="module")
def rr():
    r, ref = Renderer(), Renderer()
    yield r, ref
    r.close()
    ref.close()


class Pair:
    """The same fragments composed on `r` (tracking on, rendering into the device array `dst`) and on `ref` (tracking off),
    each bound to its own device copy of the same rows."""

    def __init__(self, r, ref, frags=None, inst=None, w=W, h=H, aa=AA_MSAA16, seed=1):
        self.r, self.ref, self.w, self.h = r, ref, w, h
        self.frags = frags if frags is not None else mixed_fragments()
        self.inst = inst if inst is not None else mixed_instances(len(self.frags))
        self.ids, self.rids = upload_all(r, self.frags), upload_all(ref, self.frags)
        lay, self.offs = r.compose([(self.ids[i], t) for i, t in self.inst])
        self.n_draw = lay.n_draw_objects
        ref.compose([(self.rids[i], t) for i, t in self.inst])
        self.rows = rand_rows(len(self.inst), seed, w, h)
        self.t = torch.from_numpy(self.rows.copy()).cuda()
        self.t_ref = torch.from_numpy(self.rows.copy()).cuda()
        torch.cuda.synchronize()
        r.bind_instance_transforms(self.t)
        ref.bind_instance_transforms(self.t_ref)
        self.dst = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        self.p = RenderParams(BASE, w, h, aa)
        r.set_damage_tracking(True)

    def set_rows(self, rows):
        self.rows = rows.astype(np.float32)
        self.t.copy_(torch.from_numpy(self.rows))
        self.t_ref.copy_(torch.from_numpy(self.rows))
        torch.cuda.synchronize()

    def step(self, p=None):
        """One frame of each: (tracked destination, reference frame)."""
        p = p or self.p
        self.r.render_resident(p, self.dst.data_ptr())
        self.ref.render_resident(p)
        return self.dst.cpu().numpy(), self.ref.download_target(p)

    def free(self):
        self.r.set_damage_tracking(False)
        for i in self.ids:
            self.r.free_fragment(i)
        for i in self.rids:
            self.ref.free_fragment(i)


def pixel_mask(tiles, w, h):
    return np.kron(tiles.astype(np.uint8), np.ones((16, 16), dtype=np.uint8)).astype(bool)[:h, :w]


def changed_tiles(a, b):
    """Tiles in which two frames differ."""
    d = (a != b).any(axis=2)
    th, tw = (d.shape[0] + 15) // 16, (d.shape[1] + 15) // 16
    pad = np.zeros((th * 16, tw * 16), dtype=bool)
    pad[:d.shape[0], :d.shape[1]] = d
    return pad.reshape(th, 16, tw, 16).any(axis=(1, 3))


def moved(rows, ks, g, nonfinite=False):
    rows = rows.copy()
    for k in ks:
        if nonfinite:
            rows[k, g.integers(0, 6)] = np.nan
        else:
            rows[k, 4:] += g.uniform(-20, 20, 2).astype(np.float32)
            rows[k, :4] *= np.float32(g.uniform(0.9, 1.1))
    return rows


# ---- 1, 2, 9. exactness, soundness of the mask, clips and layers across instances ---------------------------------------------
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_incremental_frames_equal_full_frames(rr, aa):
    r, ref = rr
    s = Pair(r, ref, aa=aa)
    n = len(s.inst)
    img, want = s.step()
    assert (img == want).all() and r.last_damage().all()
    g = np.random.default_rng(5)
    layers = [k for k, (i, _) in enumerate(s.inst) if i in (9, 10)]  # the fragments with layers, masks and open clips
    plan = [[], [0], list(g.choice(n, 3, replace=False)), list(range(n)), layers, [layers[-1]], "nan", []]
    plan += [list(g.choice(n, int(g.integers(0, 6)), replace=False)) for _ in range(30 - len(plan))]
    prev = want
    for j, ks in enumerate(plan):
        rows = moved(s.rows, g.choice(n, 2, replace=False), g, nonfinite=True) if ks == "nan" else moved(s.rows, ks, g)
        s.set_rows(rows)
        img, want = s.step()
        assert (img == want).all(), f"step {j} ({ks}): {int((img != want).any(axis=2).sum())} pixels differ from the full frame"
        dmg = r.last_damage()
        missing = changed_tiles(prev, want) & ~dmg
        assert not missing.any(), f"step {j}: tiles {np.argwhere(missing)[:4].tolist()} changed but are not damaged"
        if isinstance(ks, list) and not ks:
            assert not dmg.any(), f"step {j}: nothing moved, yet {int(dmg.sum())} tiles are damaged"
        prev = want
    s.free()


def translations(n, seed, w, h):
    rows = np.zeros((n, 6), np.float32)
    rows[:, 0] = rows[:, 3] = 1.0
    rows[:, 4:] = np.random.default_rng(seed).uniform([0, 0], [w, h], (n, 2))
    return rows


def test_one_moving_instance_damages_few_tiles(rr):
    r, ref = rr
    frags = [NativeScene()]
    frags[0].fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 1.0), None, Rect(0, 0, 20, 14))
    inst = [(0, None)] * 200
    s = Pair(r, ref, frags=frags, inst=inst, w=1024, h=768)
    s.set_rows(translations(200, 3, 1000, 750))
    s.step()
    rows = s.rows.copy()
    rows[17, 4:] += 33
    s.set_rows(rows)
    img, want = s.step()
    assert (img == want).all()
    dmg = r.last_damage()
    assert 0 < dmg.sum() <= 0.01 * dmg.size, f"{int(dmg.sum())} of {dmg.size} tiles damaged for one 20 x 14 instance"
    s.free()


# ---- 3. nothing else is written ----------------------------------------------------------------------------------------------
def test_clean_tiles_are_not_written(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    before = s.dst.cpu().numpy()
    s.dst.fill_(SENTINEL)  # poison every pixel; a frame without damage must leave all of them
    torch.cuda.synchronize()
    img, want = s.step()
    assert not r.last_damage().any() and (img == SENTINEL).all()
    s.dst.copy_(torch.from_numpy(before).cuda())
    g = np.random.default_rng(9)
    s.set_rows(moved(s.rows, [3, 20], g))
    s.dst.fill_(SENTINEL)
    torch.cuda.synchronize()
    img, want = s.step()
    m = pixel_mask(r.last_damage(), W, H)
    assert m.any() and not m.all()
    assert (img[m] == want[m]).all() and (img[~m] == SENTINEL).all()
    s.free()


# ---- 4. caller rectangles on an uploaded scene -------------------------------------------------------------------------------
def test_rectangles_on_an_uploaded_scene(rr):
    r, _ = rr
    packed = resolve(scenes.tiger(W, H).encoding)
    r.upload(packed)
    r.set_damage_tracking(True)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.render_resident(p, dst.data_ptr())
    full = dst.cpu().numpy()
    assert r.last_damage().all()
    dst.fill_(SENTINEL)
    torch.cuda.synchronize()
    r.add_damage([[100, 50, 140, 90], [W - 5, H - 5, W + 100, H + 100]])  # the second one is clamped to the frame
    r.render_resident(p, dst.data_ptr())
    img = dst.cpu().numpy()
    tiles = r.last_damage()
    want = np.zeros_like(tiles)
    want[50 // 16:(90 + 15) // 16, 100 // 16:(140 + 15) // 16] = True
    want[-1, -1] = True
    assert (tiles == want).all()
    m = pixel_mask(tiles, W, H)
    assert (img[m] == full[m]).all() and (img[~m] == SENTINEL).all()
    r.set_damage_tracking(False)


# ---- 5. full-frame triggers --------------------------------------------------------------------------------------------------
def test_full_frame_triggers(rr):
    """Each trigger follows an incremental frame into the same destination pointer and changes nothing else, so each one alone
    must make the frame full; the frame after it, with the same parameters, is incremental again."""
    r, ref = rr
    s = Pair(r, ref)
    g = np.random.default_rng(11)
    s.step()

    def pair(p, dst):
        r.render_resident(p, dst.data_ptr())
        ref.render_resident(p)
        n = p.width * p.height * 4  # a smaller frame fills the front of the destination, rows p.width pixels apart
        return dst.view(-1)[:n].view(p.height, p.width, 4).cpu().numpy(), ref.download_target(p)

    def check(what, p, dst=None):
        dst = s.dst if dst is None else dst
        img, want = pair(p, dst)
        assert r.last_damage().all(), f"{what}: expected a full frame"
        assert (img == want).all(), f"{what}: pixels differ from the full frame"
        s.set_rows(moved(s.rows, [1], g))
        img, want = pair(p, dst)
        assert not r.last_damage().all(), f"{what}: the frame after it should be incremental"
        assert (img == want).all(), f"{what}: the incremental frame after it differs from the full frame"

    p = s.p
    s.set_rows(moved(s.rows, [2], g))
    img, want = pair(p, s.dst)  # the base: incremental, in s.dst
    assert not r.last_damage().all() and (img == want).all()
    r.set_damage_tracking(True)  # on again
    check("tracking switched on again", p)
    r.bind_instance_transforms(s.t)  # the same rows bound again
    check("bind", p)
    p = RenderParams(BASE, W, H, AA_MSAA8)
    check("AA", p)
    p = RenderParams(Color.from_rgba8(90, 10, 10), W, H, AA_MSAA8)
    check("base colour", p)
    p = RenderParams(Color.from_rgba8(90, 10, 10), W - 24, H - 40, AA_MSAA8)
    check("size", p)  # same destination pointer, smaller frame
    r.set_cells([0, s.n_draw])  # one cell: no batch, but a new split
    check("set_cells", p)
    view = Affine.translate(-10, 6) * Affine.scale(1.1)
    r.set_view(view)
    ref.set_view(view)
    check("view", p)
    r.set_view(None)
    ref.set_view(None)
    check("view cleared", p)
    check("destination", p, torch.zeros_like(s.dst))
    r.bind_instance_transforms(None)  # unbind: both render the scene as composed
    ref.bind_instance_transforms(None)
    img, want = pair(p, s.dst)
    assert r.last_damage().all() and (img == want).all()
    s.free()


def test_full_frame_after_reupload(rr):
    r, _ = rr
    packed = resolve(scenes.tiger(W, H).encoding)
    r.upload(packed)
    r.set_damage_tracking(True)
    dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    p = RenderParams(BASE, W, H, AA_MSAA16)
    r.render_resident(p, dst.data_ptr())
    full = dst.cpu().numpy()
    r.render_resident(p, dst.data_ptr())
    assert not r.last_damage().any()
    dst.fill_(SENTINEL)
    torch.cuda.synchronize()
    r.upload(packed)  # the same bytes again: still a new installation
    r.render_resident(p, dst.data_ptr())
    assert r.last_damage().all() and (dst.cpu().numpy() == full).all()
    # a streamed frame rewrites the mask without the tracker following it: the last report is gone, not stale
    r.add_damage([[0, 0, 16, 16]])
    r.render_resident(p, dst.data_ptr())
    assert r.last_damage().sum() == 1
    list(r.render_stream([packed], p))
    with pytest.raises(VelloB200Error):
        r.last_damage()
    r.set_damage_tracking(False)


def _override_pair(r, ref, t):
    """The same two-instance composition on r and ref, each drawing the device pixels `t` through its own registered texture."""
    out = []
    for x in (r, ref):
        tex = x.register_texture(t)
        s = NativeScene()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.4, 0.8, 1.0), None, Rect(0, 0, 120, 80))
        s.draw_image(tex, Affine.translate(40, 30))
        fid = x.upload_fragment(s)
        x.compose([(fid, None), (fid, Affine.translate(200, 150))])
        out.append((tex, fid))
    return out


def test_dirty_override(rr):
    r, ref = rr
    t = torch.randint(0, 256, (16, 24, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    made = _override_pair(r, ref, t)
    try:
        r.set_damage_tracking(True)
        dst = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        p = RenderParams(BASE, W, H, AA_MSAA16)

        def pair():
            r.render_resident(p, dst.data_ptr())
            ref.render_resident(p)
            return dst.cpu().numpy(), ref.download_target(p)

        pair()
        img, want = pair()
        assert not r.last_damage().any() and (img == want).all()

        def new_pixels():
            t.copy_(torch.randint(0, 256, (16, 24, 4), dtype=torch.uint8, device="cuda"))
            torch.cuda.synchronize()
            for x, (tex, _) in zip((r, ref), made):
                x.mark_override_image_dirty(tex)

        new_pixels()  # dirty, no rectangles: the frame is full
        img, want = pair()
        assert r.last_damage().all() and (img == want).all()
        img, want = pair()
        assert not r.last_damage().any() and (img == want).all()
        new_pixels()  # dirty, with rectangles over both places of the image: incremental
        r.add_damage([[32, 24, 72, 56], [232, 174, 272, 206]])
        img, want = pair()
        dmg = r.last_damage()
        assert dmg.any() and not dmg.all()
        assert (img == want).all(), f"{int((img != want).any(axis=2).sum())} pixels differ from the full frame"
    finally:
        r.set_damage_tracking(False)
        for x, (tex, fid) in zip((r, ref), made):
            x.free_fragment(fid)
            x.unregister_texture(tex)


def test_full_frame_after_recompose(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    r.compose([(s.ids[i], t) for i, t in s.inst])  # the same scene again: still a new installation
    ref.compose([(s.rids[i], t) for i, t in s.inst])
    img, want = s.step()
    assert r.last_damage().all() and (img == want).all()
    s.free()


# ---- 6. arena overflow re-runs -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arena", ["ptcl", "segments"])
def test_overflow_rerun_keeps_the_damage(rr, arena):
    r, ref = rr
    s = Pair(r, ref)
    g = np.random.default_rng(13)
    s.step()
    s.set_rows(moved(s.rows, list(range(len(s.inst))), g))  # every instance: damaged tiles all over the frame
    # segments are written for every tile, damaged or not; ptcl down to its static area: every dynamic chunk overflows
    r.limit_arena(arena, 1 if arena == "segments" else (W // 16) * (H // 16) * 64)
    img, want = s.step()
    assert r.last_stats.retries >= 1 and (img == want).all()
    s.set_rows(moved(s.rows, [7], g))
    img, want = s.step()
    assert (img == want).all() and not r.last_damage().all()
    s.free()


# ---- 7. graph replay ---------------------------------------------------------------------------------------------------------
def test_moving_rows_replays_the_graph(rr):
    r, ref = rr
    s = Pair(r, ref)
    g = np.random.default_rng(17)
    s.step()
    s.set_rows(moved(s.rows, [2], g))
    s.step()
    caps = r.debug_graph_captures()
    for _ in range(8):
        s.set_rows(moved(s.rows, list(g.choice(len(s.inst), 3, replace=False)), g))
        img, want = s.step()
        assert (img == want).all()
    assert r.debug_graph_captures() == caps
    s.free()


# ---- 8. hit tests ------------------------------------------------------------------------------------------------------------
def test_hit_tests_on_incremental_frames(rr):
    r, ref = rr
    s = Pair(r, ref)
    g = np.random.default_rng(19)
    s.step()
    s.set_rows(moved(s.rows, [0, 4, 11], g))
    s.step()
    assert not r.last_damage().all()
    pts = np.random.default_rng(2).uniform([0, 0], [W, H], (4000, 2)).astype(np.float32)
    assert (r.hit_test(pts) == ref.hit_test(pts)).all()
    s.free()


# ---- 10. scale ---------------------------------------------------------------------------------------------------------------
def test_ten_thousand_instances_one_moving(rr):
    r, ref = rr
    frags = [NativeScene()]
    frags[0].fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.2, 0.7, 0.4, 0.8), None, Rect(0, 0, 18, 12))
    frags[0].fill(FILL_NON_ZERO, Affine.translate(4, 3), Color(0.9, 0.9, 0.2, 1.0), None, Rect(0, 0, 6, 6))
    inst = [(0, None)] * 10000
    s = Pair(r, ref, frags=frags, inst=inst, w=2048, h=2048, seed=23)
    s.set_rows(translations(10000, 23, 2030, 2036))
    s.step()
    rows = s.rows.copy()
    rows[4321, 4:] += 17
    s.set_rows(rows)
    img, want = s.step()
    assert (img == want).all()
    dmg = r.last_damage()
    assert 0 < dmg.sum() < 0.01 * dmg.size
    s.free()


# ---- 11. errors --------------------------------------------------------------------------------------------------------------
def test_errors():
    r = Renderer()
    try:
        with pytest.raises(VelloB200Error):
            r._check(r.lib.vb_add_damage(r.handle, None, 1), "vb_add_damage")
        r.add_damage(np.zeros((0, 4), np.uint32))  # nothing to add: fine
        with pytest.raises(VelloB200Error):
            r.last_damage()  # no frame yet
        r.upload(resolve(scenes.tiger(64, 64).encoding))
        r.set_damage_tracking(True)
        r.enqueue(RenderParams(BASE, 64, 64, AA_MSAA16))
        with pytest.raises(VelloB200Error):
            r.add_damage([[0, 0, 8, 8]])  # meant for the frame after the one in flight
        r.finish()
        r.add_damage([[0, 0, 8, 8]])
        r.set_damage_tracking(False)
        arena, nbytes = C.c_void_p(), C.c_size_t()
        r._check(r.lib.vb_exchange_configure(r.handle, 0, 1, C.byref(arena), C.byref(nbytes)), "vb_exchange_configure")
        with pytest.raises(VelloB200Error):
            r.set_damage_tracking(True)
    finally:
        r.close()
    g = RendererGroup([0])
    try:
        with pytest.raises(VelloB200Error):
            g.renderer(0).set_damage_tracking(True)
    finally:
        g.close()
