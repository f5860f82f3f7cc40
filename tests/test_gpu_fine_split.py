"""fine's split queue (k_coarse.cu CO_FLAGGED, k_fine.cu FI_LISTS_*): coarse puts every tile of the window into a simple list
(only FILL / SOLID / COLOR / JUMP from its occlusion start), painted by the lean k_fine_solid, or into a flagged list, painted
by the full k_fine after it. Scenes here mix simple tiles with tiles flagged by clips, blend layers, gradients, images and
blurred rectangles, and with tiles whose complex commands sit below an opaque cover (simple again from the occlusion start).

In area AA, MSAA8 and MSAA16: the frame equals the oracle's fine replayed on the GPU's own buffers byte for byte and
`compare_all` passes; every tile of the window is in exactly one list, and both kinds of list are non-empty; the same holds
with occlusion culling off (one k_fine over every list), in tile-row stripes and in a batch of cells."""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import (BLACK, COMPOSE_SRC_OVER, FILL_EVEN_ODD, FILL_NON_ZERO, MIX_MULTIPLY, Color, Gradient, Image, Scene,
                                 resolve)
from vello_b200.shapes import Affine, Circle, Rect

from . import parity

pytestmark = pytest.mark.gpu

AAS = [AA_AREA, AA_MSAA8, AA_MSAA16]
FINE_LISTS = 16  # vb_types.h VB_FINE_LISTS
W, H = 512, 384


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def mixed_scene(seed):
    """Translucent and opaque circles over the frame (simple tiles), a clip layer, a multiply layer, a gradient, an image and a
    blurred rectangle (flagged tiles), and a gradient and an image under an opaque full-tile cover (simple from the cover on).
    Returns the scene and {name: (tile x, tile y)} of a tile of each kind."""
    rng = np.random.default_rng(seed)
    s = Scene()
    I = Affine.translate(0.0, 0.0)
    for _ in range(120):
        x, y, r = rng.uniform(0, W), rng.uniform(0, H), rng.uniform(4, 40)
        a = 255 if rng.random() < 0.7 else int(rng.integers(40, 220))
        col = Color.from_rgba8(*(int(v) for v in rng.integers(0, 256, 3)), a)
        s.fill(FILL_EVEN_ODD if rng.random() < 0.2 else FILL_NON_ZERO, I, col, None, Circle(x, y, r))
    stops = [(0.0, Color.from_rgba8(255, 0, 0, 255)), (1.0, Color.from_rgba8(0, 0, 255, 128))]
    img = Image(rng.integers(0, 256, size=(24, 24, 4), dtype=np.uint8))
    # under a cover: tiles (1..2, 1..2) run a gradient and an image, then an opaque rectangle over both tiles
    s.fill(FILL_NON_ZERO, I, Gradient.linear((16, 16), (48, 48), stops), None, Rect(16, 16, 48, 48))
    s.fill(FILL_NON_ZERO, Affine.translate(20.0, 20.0), img, None, Rect(0, 0, 24, 24))
    s.fill(FILL_NON_ZERO, I, Color.from_rgba8(10, 200, 30, 255), None, Rect(16, 16, 48, 48))
    # flagged: a gradient, an image, a blurred rectangle, a clip layer and a multiply layer, each in tiles of its own (the clip
    # only on its edge: a tile the clip covers whole emits no clip commands)
    s.fill(FILL_NON_ZERO, I, Gradient.linear((96, 96), (150, 140), stops), None, Rect(96, 96, 150, 140))
    s.fill(FILL_NON_ZERO, Affine.translate(200.0, 100.0), img, None, Rect(0, 0, 24, 24))
    s.draw_blurred_rounded_rect(I, Rect(300, 60, 360, 110), Color.from_rgba8(40, 40, 220, 200), 6.0, 4.0)
    s.push_clip_layer(FILL_NON_ZERO, I, Circle(100, 300, 40))
    s.fill(FILL_NON_ZERO, I, Color.from_rgba8(250, 200, 0, 255), None, Rect(50, 250, 150, 350))
    s.pop_layer()
    s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY, COMPOSE_SRC_OVER, 0.8, I, Rect(380, 250, 470, 330))
    s.fill(FILL_NON_ZERO, I, Color.from_rgba8(0, 180, 250, 200), None, Circle(420, 290, 50))
    s.pop_layer()
    return s, {"covered": (1, 1), "gradient": (7, 7), "image": (13, 7), "blur": (20, 5), "clip": (3, 18), "layer": (26, 18)}


def lists_of(r, n_tiles, stride):
    """{tile of the window: (list, occlusion start)} from coarse's lists of the last frame, asserting each tile is in exactly
    one of them."""
    counts = r.download("fine_lists", np.uint32).astype(np.int64)
    assert counts.shape == (FINE_LISTS,)
    cls = r.download("cls_list", np.uint32).reshape(-1, 2)
    seen = {}
    for lst in range(FINE_LISTS):
        for t, start in cls[lst * stride:lst * stride + counts[lst]]:
            assert int(t) not in seen, f"tile {int(t)} in lists {seen[int(t)][0]} and {lst}"
            seen[int(t)] = (lst, int(start))
    assert sorted(seen) == list(range(n_tiles)), f"{n_tiles - len(seen)} tiles of the window in no list"
    return seen


def render_checked(r, oracle, packed, aa):
    img = r.render_to_texture(packed, RenderParams(BLACK, W, H, aa))
    parity.assert_replay(r, oracle, packed, img, W, H, aa, BLACK)
    return img


@pytest.mark.parametrize("aa", AAS)
def test_split_frame_matches_replay(renderer, oracle, aa):
    scene, where = mixed_scene(7)
    packed = resolve(scene.encoding)
    img = renderer.render_to_texture(packed, RenderParams(BLACK, W, H, aa))
    oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), aa)
    parity.compare_all(renderer, oracle, packed.layout, W, H)
    parity.assert_replay(renderer, oracle, packed, img, W, H, aa, BLACK)
    wt, ht = (W + 15) // 16, (H + 15) // 16
    seen = lists_of(renderer, wt * ht, wt * ht)
    flagged = {t for t, (lst, _) in seen.items() if lst & 1}
    assert flagged and len(flagged) < wt * ht, f"{len(flagged)} of {wt * ht} tiles flagged"
    for name, (tx, ty) in where.items():
        assert ((ty * wt + tx) in flagged) == (name != "covered"), f"the {name} tile ({tx}, {ty})"
    # occlusion culling off: one k_fine over every list, the same pixels
    renderer.set_occlusion_cull(False)
    try:
        off = render_checked(renderer, oracle, packed, aa)
    finally:
        renderer.set_occlusion_cull(True)
    assert np.array_equal(off, img)


@pytest.mark.parametrize("aa", AAS)
def test_split_stripes(renderer, oracle, aa):
    """Two tile-row stripes cut through flagged tiles: each stripe's lists hold exactly its own tiles, and the stripes equal
    the matching rows of the full frame."""
    packed = resolve(mixed_scene(11)[0].encoding)
    full = renderer.render_to_texture(packed, RenderParams(BLACK, W, H, aa))
    wt, ht, cut = (W + 15) // 16, (H + 15) // 16, 7
    parts = []
    for rows in ((0, cut), (cut, ht)):
        parts.append(renderer.render_to_texture(packed, RenderParams(BLACK, W, H, aa), tile_rows=rows))
        seen = lists_of(renderer, wt * (rows[1] - rows[0]), wt * ht)
        assert any(lst & 1 for lst, _ in seen.values()) and any(lst & 1 == 0 for lst, _ in seen.values())
    assert np.array_equal(np.concatenate(parts, axis=0), full)


@pytest.mark.parametrize("aa", AAS)
def test_split_batch(renderer, aa):
    """A batch of three cells, one of them without any flagged tile, equals each scene rendered alone."""
    scenes = [mixed_scene(3)[0], mixed_scene(5)[0], Scene()]
    rng = np.random.default_rng(1)
    for _ in range(40):
        scenes[2].fill(FILL_NON_ZERO, Affine.translate(0.0, 0.0), Color.from_rgba8(*(int(v) for v in rng.integers(0, 256, 4))), None,
                       Circle(rng.uniform(0, W), rng.uniform(0, H), rng.uniform(5, 60)))
    p = RenderParams(BLACK, W, H, aa)
    frames = renderer.render_batch(scenes, p)
    wt, ht = (W + 15) // 16, (H + 15) // 16
    seen = lists_of(renderer, wt * ht * 3, wt * ht * 3)
    assert not any(lst & 1 for t, (lst, _) in seen.items() if t >= 2 * wt * ht), "a tile of the plain cell is flagged"
    assert any(lst & 1 for lst, _ in seen.values())
    for i, s in enumerate(scenes):
        alone = renderer.render_to_texture(resolve(s.encoding), p)
        assert np.array_equal(frames[i], alone), f"cell {i}"
