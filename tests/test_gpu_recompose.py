"""Recompose with damage tracking (Renderer.recompose, vb_recompose): after a recompose, the next frame into the destination of
the base frame repaints only the tiles of the instances added, removed or changed. `r` tracks and recomposes into one device
destination; `ref` composes the same lists with tracking off and always renders in full. Every frame of `r` must equal `ref`'s
byte for byte, and the composed scenes must be identical. Run on an H100 with `pytest -m gpu`."""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import Color, FILL_NON_ZERO, Image
from vello_b200.renderer import Renderer, VelloB200Error
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Circle, Rect

from .test_gpu_compose import BASE, mixed_fragments, mixed_instances, upload_all

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
    """The same fragments on `r` (tracking on, recomposing, rendering into the device array `dst`) and on `ref` (tracking off,
    composing, rendering into its own target). Instances are (fragment index, Affine or None)."""

    def __init__(self, r, ref, frags=None, inst=None, w=W, h=H, aa=AA_MSAA16):
        self.r, self.ref, self.w, self.h = r, ref, w, h
        self.frags = frags if frags is not None else mixed_fragments()
        self.ids, self.rids = upload_all(r, self.frags), upload_all(ref, self.frags)
        self.dst = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        self.p = RenderParams(BASE, w, h, aa)
        r.set_damage_tracking(True)
        self.set(inst if inst is not None else mixed_instances(len(self.frags)), how="compose")

    def set(self, inst, how="recompose"):
        """Give both renderers the instance list: `r` through `how` ("recompose" or "compose"), `ref` through compose."""
        self.inst = list(inst)
        lay, self.offs = getattr(self.r, how)([(self.ids[i], t) for i, t in self.inst])
        rlay, roffs = self.ref.compose([(self.rids[i], t) for i, t in self.inst])
        assert (lay.as_array() == rlay.as_array()).all() and self.offs == roffs
        self.n_draw = lay.n_draw_objects

    def step(self, p=None, dst=None):
        """One frame of each: (tracked destination, reference frame)."""
        p = p or self.p
        dst = self.dst if dst is None else dst
        self.r.render_resident(p, dst.data_ptr())
        self.ref.render_resident(p)
        return dst.cpu().numpy(), self.ref.download_target(p)

    def boxes(self):
        return self.r.download("draw_bboxes", np.float32).reshape(-1, 4)[:self.n_draw].copy()

    def free(self):
        self.r.set_damage_tracking(False)
        for i in self.ids:
            self.r.free_fragment(i)
        for i in self.rids:
            self.ref.free_fragment(i)


def same_scene(r, ref):
    for name, dt in (("scene", np.uint32), ("ramps", np.uint32), ("atlas", np.uint8)):
        a, b = r.download(name, dt), ref.download(name, dt)
        assert a.size == b.size and (a == b).all(), f"recompose and compose made different {name}"


def changed_tiles(a, b):
    d = (a != b).any(axis=2)
    th, tw = (d.shape[0] + 15) // 16, (d.shape[1] + 15) // 16
    pad = np.zeros((th * 16, tw * 16), dtype=bool)
    pad[:d.shape[0], :d.shape[1]] = d
    return pad.reshape(th, 16, tw, 16).any(axis=(1, 3))


def pixel_mask(tiles, w, h):
    return np.kron(tiles.astype(np.uint8), np.ones((16, 16), dtype=np.uint8)).astype(bool)[:h, :w]


def box_tiles(boxes, w, h):
    """The tiles of clipped draw boxes, rounded out as tile_alloc rounds them."""
    wt, ht = (w + 15) // 16, (h + 15) // 16
    m = np.zeros((ht, wt), dtype=bool)
    for x0, y0, x1, y1 in boxes:
        if not (x0 < x1 and y0 < y1):
            continue
        tx0, tx1 = int(np.clip(np.floor(x0 / 16), 0, wt)), int(np.clip(np.ceil(x1 / 16), 0, wt))
        ty0, ty1 = int(np.clip(np.floor(y0 / 16), 0, ht)), int(np.clip(np.ceil(y1 / 16), 0, ht))
        m[ty0:ty1, tx0:tx1] = True
    return m


# ---- exactness and soundness over random edits -------------------------------------------------------------------------------
def random_edit(g, inst, n_frags, step):
    """One edit of a UI's instance list, and its name."""
    inst = list(inst)
    n = len(inst)
    k = int(g.integers(0, n))
    ops = ["replace", "insert", "delete", "front", "back", "transform", "none", "layers", "image_early", "gradient_early"]
    op = ops[step % len(ops)] if step < 2 * len(ops) else ops[int(g.integers(0, len(ops)))]
    t = Affine.translate(float(g.uniform(-40, 300)), float(g.uniform(-40, 250)))
    if op == "replace":
        inst[k] = (int(g.integers(0, n_frags)), inst[k][1])
    elif op == "insert":
        inst.insert(k, (int(g.integers(0, n_frags)), t))
    elif op == "delete" and n > 1:
        del inst[k]
    elif op == "front":
        inst.insert(0, inst.pop(k))
    elif op == "back":
        inst.append(inst.pop(k))
    elif op == "transform":
        inst[k] = (inst[k][0], t)
    elif op == "layers":  # the fragments with layers, masks and open clips: add one, or remove one
        have = [j for j, (i, _) in enumerate(inst) if i in (9, 10)]
        if have and g.random() < 0.5:
            del inst[have[int(g.integers(0, len(have)))]]
        else:
            inst.insert(k, (int(g.choice([9, 10])), t))
    elif op == "image_early":  # later images move in the atlas
        inst.insert(int(g.integers(0, 3)), (int(g.choice([6, 7, 8])), t))
    elif op == "gradient_early":  # later ramps move to other rows
        inst.insert(int(g.integers(0, 3)), (int(g.choice([4, 5])), t))
    return inst, op


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_recomposed_frames_equal_full_frames(rr, aa):
    r, ref = rr
    s = Pair(r, ref, aa=aa)
    img, want = s.step()
    assert (img == want).all() and r.last_damage().all()
    g = np.random.default_rng(31 + aa)
    prev = want
    incremental = 0
    for j in range(32):
        inst, op = random_edit(g, s.inst, len(s.frags), j)
        s.set(inst)
        same_scene(r, ref)
        img, want = s.step()
        assert (img == want).all(), f"step {j} ({op}): {int((img != want).any(axis=2).sum())} pixels differ from the full frame"
        dmg = r.last_damage()
        missing = changed_tiles(prev, want) & ~dmg
        assert not missing.any(), f"step {j} ({op}): tiles {np.argwhere(missing)[:4].tolist()} changed but are not damaged"
        if op == "none":
            assert not dmg.any(), f"step {j}: nothing changed, yet {int(dmg.sum())} tiles are damaged"
        incremental += not dmg.all()
        prev = want
    assert incremental >= 20, f"only {incremental} of 32 recomposes gave an incremental frame"
    s.free()


def new_boxes(s, ks):
    b = s.boxes()
    return [x for k in ks for x in b[s.offs[k]:s.offs[k + 1]]]


def test_ramp_rows_do_not_damage_but_atlas_places_do(rr):
    """An instance whose ramps move to other rows is not damaged: a row holds the same bytes wherever it is. An instance whose
    images move in the atlas is: fine samples in atlas coordinates."""
    r, ref = rr
    frags = mixed_fragments()
    extra = NativeScene()  # an image of its own, placed first in the atlas when inserted in front
    px = np.random.default_rng(5).integers(0, 256, (12, 10, 4), dtype=np.uint8)
    extra.draw_image(Image(px, key=px.ctypes.data), Affine.translate(2, 3))
    frags.append(extra)
    inst = [(4, Affine.translate(300, 200)), (0, Affine.translate(20, 20)), (6, Affine.translate(200, 30))]
    s = Pair(r, ref, frags=frags, inst=inst)
    s.step()
    # fragment 9 draws a gradient with other stops: the ramps of fragment 4 move from row 0 to row 1
    s.set([(9, Affine.translate(10, 250))] + inst)
    img, want = s.step()
    assert (img == want).all()
    assert (r.last_damage() == box_tiles(new_boxes(s, [0]), W, H)).all(), "moved ramp rows must not damage"
    old = s.boxes()
    old_offs = s.offs
    s.set([(len(frags) - 1, None)] + s.inst)  # fragment 6's images now follow the new image in the atlas
    img, want = s.step()
    assert (img == want).all()
    k6 = len(s.inst) - 1
    expect = box_tiles(new_boxes(s, [0, k6]), W, H) | box_tiles(old[old_offs[k6 - 1]:old_offs[k6]], W, H)
    assert (r.last_damage() == expect).all(), "an instance whose images moved in the atlas must be damaged, and nothing else"
    s.free()


# ---- smallness -----------------------------------------------------------------------------------------------------------------
def test_no_change_damages_nothing_and_compose_everything(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    s.set(s.inst)
    img, want = s.step()
    assert (img == want).all() and not r.last_damage().any()
    s.set(s.inst, how="compose")
    img, want = s.step()
    assert (img == want).all() and r.last_damage().all()
    s.free()


def small_fragments():
    frags = []
    for k in range(16):
        f = NativeScene()
        c = Color.from_rgba8(40 + 13 * k, 200 - 9 * k, 60 + 11 * k, 255 if k % 3 else 200)
        if k % 2:
            f.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Rect(0, 0, 8 + k, 6 + k // 2))
        else:
            f.fill(FILL_NON_ZERO, Affine.IDENTITY, c, None, Circle(6, 6, 3 + k / 4))
        frags.append(f)
    return frags


def grid_instances(n, seed, w, h):
    g = np.random.default_rng(seed)
    return [(int(g.integers(0, 16)), Affine.translate(float(g.uniform(0, w - 30)), float(g.uniform(0, h - 30)))) for _ in range(n)]


def test_one_edit_among_ten_thousand_damages_only_its_boxes(rr):
    r, ref = rr
    w = h = 2048
    s = Pair(r, ref, frags=small_fragments(), inst=grid_instances(10_000, 41, w, h), w=w, h=h)
    s.step()
    g = np.random.default_rng(43)
    for op in ["replace", "insert", "delete", "raise", "insert_front"]:
        old_boxes, old_offs, inst = s.boxes(), s.offs, list(s.inst)
        k = int(g.integers(100, 9_900))
        if op == "replace":
            inst[k] = ((inst[k][0] + 1) % 16, inst[k][1])
            gone, new = [k], [k]
        elif op == "insert":
            inst.insert(k, (3, Affine.translate(1000.5, 700.25)))
            gone, new = [], [k]
        elif op == "insert_front":
            inst.insert(0, (5, Affine.translate(10.5, 1900.25)))
            gone, new = [], [0]
        elif op == "delete":
            del inst[k]
            gone, new = [k], []
        else:  # raise: to the top of the z-order
            inst.append(inst.pop(k))
            gone, new = [k], [len(inst) - 1]
        s.set(inst)
        img, want = s.step()
        assert (img == want).all(), f"{op}: pixels differ from the full frame"
        boxes = s.boxes()
        expect = np.zeros_like(r.last_damage())
        for i in gone:
            expect |= box_tiles(old_boxes[old_offs[i]:old_offs[i + 1]], w, h)
        for i in new:
            expect |= box_tiles(boxes[s.offs[i]:s.offs[i + 1]], w, h)
        dmg = r.last_damage()
        assert expect.any() and (dmg == expect).all(), f"{op}: {int(dmg.sum())} tiles damaged, the instance's boxes cover {int(expect.sum())}"
    s.free()


def test_clean_tiles_are_not_written(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    s.dst.fill_(SENTINEL)
    torch.cuda.synchronize()
    inst = list(s.inst)
    inst[3] = (2, inst[3][1])
    del inst[20]
    s.set(inst)
    img, want = s.step()
    m = pixel_mask(r.last_damage(), W, H)
    assert m.any() and not m.all()
    assert (img[m] == want[m]).all() and (img[~m] == SENTINEL).all()
    s.free()


# ---- every fallback on its own is a full, exact frame ------------------------------------------------------------------------
def edited(inst):
    inst = list(inst)
    inst[1] = (3, inst[1][1])
    return inst


def test_fallbacks(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()

    def edit():
        s.set(edited(s.inst) if s.inst[1][0] != 3 else mixed_instances(len(s.frags)))

    def full(what, **kw):
        img, want = s.step(**kw)
        assert r.last_damage().all(), f"{what}: expected a full frame"
        assert (img == want).all(), f"{what}: pixels differ from the full frame"
        edit()  # the next recompose is followed again
        img, want = s.step(**kw)
        assert not r.last_damage().all() and (img == want).all(), f"{what}: the recompose after it should be incremental"

    r.set_damage_tracking(False)
    edit()
    img, want = s.step()
    assert (img == want).all() and r.last_damage().all(), "tracking off"
    r.set_damage_tracking(True)  # on again: no base
    edit()
    full("no base")
    rows = np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), (len(s.inst), 1))
    t, t_ref = torch.from_numpy(rows).cuda(), torch.from_numpy(rows.copy()).cuda()
    r.bind_instance_transforms(t)  # a bound base: its transforms came from device memory
    ref.bind_instance_transforms(t_ref)
    s.step()
    edit()
    full("bound base")
    edit()
    edit()  # two recomposes without a frame between them
    full("two recomposes")
    r.run_stages(s.p, "pathtag", "binning")
    edit()
    full("run_stages since the base")
    s.step()
    r.limit_arena("segments", 1)
    r.enqueue(s.p, s.dst.data_ptr())
    with pytest.raises(VelloB200Error):
        r.finish()  # an enqueued frame is not re-run: it failed for good
    r.limit_arena("segments", Renderer.NO_LIMIT)
    edit()
    full("a failed frame since the base")
    view = Affine.translate(-10, 6) * Affine.scale(1.1)
    r.set_view(view)
    ref.set_view(view)
    edit()
    full("view")  # with the view kept, recomposes are followed
    r.set_view(None)
    ref.set_view(None)
    edit()
    full("view cleared")
    r.set_cells([0, s.n_draw])
    edit()
    full("cells")
    edit()
    img, want = s.step(dst=torch.zeros_like(s.dst))
    assert r.last_damage().all() and (img == want).all(), "another destination: expected a full frame"
    s.free()


def test_past_the_edit_bound_is_exact(rr):
    """Reversing 5,000 instances needs far more than VB_RECOMPOSE_MAX_EDITS edits: the middle is matched by position."""
    r, ref = rr
    s = Pair(r, ref, frags=small_fragments(), inst=grid_instances(5_000, 47, 1024, 768), w=1024, h=768)
    _, prev = s.step()
    s.set(s.inst[::-1])
    img, want = s.step()
    assert (img == want).all()
    assert not (changed_tiles(prev, want) & ~r.last_damage()).any()
    s.free()


# ---- frame machinery -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arena", ["ptcl", "segments"])
def test_overflow_rerun_keeps_the_damage(rr, arena):
    """A frame re-run after an arena overflow damages what the same recompose damages without one."""
    r, ref = rr
    # a stack of 150 instances in front of the open clips of mixed_instances, and the bottom one replaced: its tiles need more
    # commands than ptcl's static area holds
    a = [(1, Affine.translate(200 + 0.25 * k, 150)) for k in range(150)] + mixed_instances(12)
    s = Pair(r, ref, inst=a)
    s.step()
    b = list(a)
    b[0] = (2, b[0][1])
    s.set(b)
    s.step()
    expect = r.last_damage()
    s.set(a)
    s.step()
    s.set(b)
    # segments are written for every tile, damaged or not; ptcl down to its static area: every dynamic chunk overflows
    r.limit_arena(arena, 1 if arena == "segments" else (W // 16) * (H // 16) * 64)
    img, want = s.step()
    assert r.last_stats.retries >= 1 and (img == want).all()
    assert (r.last_damage() == expect).all() and not expect.all()
    s.free()


def test_enqueue_finish_graph_replay_and_hit_tests(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    s.step()
    s.set(edited(s.inst))
    r.enqueue(s.p, s.dst.data_ptr())
    r.finish()
    launches = r.last_stats.kernel_launches
    ref.render_resident(s.p)
    want = ref.download_target(s.p)
    assert not r.last_damage().all() and (s.dst.cpu().numpy() == want).all()
    pts = np.random.default_rng(2).uniform([0, 0], [W, H], (4000, 2)).astype(np.float32)
    assert (r.hit_test(pts) == ref.hit_test(pts)).all()
    s.step()  # the first steady frame after it
    caps = r.debug_graph_captures()
    for _ in range(4):
        img, want = s.step()
        assert (img == want).all() and not r.last_damage().any()
    assert r.debug_graph_captures() == caps, "steady frames after a recompose must replay their graph"
    assert r.last_stats.kernel_launches + 1 == launches, "the frame after the recompose runs k_recompose_damage once"
    s.free()


# ---- errors leave the scene and the damage --------------------------------------------------------------------------------
def test_errors_leave_the_scene_and_the_damage(rr):
    r, ref = rr
    s = Pair(r, ref)
    s.step()
    before = r.download("scene", np.uint32)
    bad = [(s.ids[0], None), (123_456_789, None)]
    with pytest.raises(VelloB200Error):
        r.recompose(bad)
    with pytest.raises(VelloB200Error):
        r.recompose([(s.ids[0], Affine((float("inf"), 0.0, 0.0, 1.0, 0.0, 0.0)))])
    assert (r.download("scene", np.uint32) == before).all()
    img, want = s.step()  # still tracked against the same base: nothing changed
    assert (img == want).all() and not r.last_damage().any()
    s.set(edited(s.inst))  # an armed recompose, then a failing one: the armed damage stays
    with pytest.raises(VelloB200Error):
        r.recompose(bad)
    img, want = s.step()
    dmg = r.last_damage()
    assert (img == want).all() and dmg.any() and not dmg.all()
    s.free()
