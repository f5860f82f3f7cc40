"""The statement of hit testing (tests/hit_ref.py) held to known answers on the oracle's buffers, and the draw-object
counters (`Scene.n_draw_objects`, `vb_scene_n_draw_objects`) that name the answers. CPU only.

tests/test_gpu_hit_test.py holds vb_hit_test to hit_ref on the GPU's own buffers."""
import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_MSAA16
from vello_b200.encoding import BLACK, FILL_EVEN_ODD, FILL_NON_ZERO, Color, Image, Scene, resolve
from vello_b200.shapes import Affine, BezPath, Rect

from . import hit_ref
from .test_scene_native import RECIPES, MirrorScene

I = Affine.IDENTITY
W = H = 128
RED, GREEN, BLUE = Color.from_rgba8(220, 40, 40), Color.from_rgba8(40, 200, 60), Color.from_rgba8(40, 60, 220)
CLEAR = Color.from_rgba8(255, 255, 255, 0)


def fill(s, shape, color=RED, rule=FILL_NON_ZERO):
    """Fill and return the draw-object index the fill received."""
    ix = s.n_draw_objects
    s.fill(rule, I, color, None, shape)
    assert s.n_draw_objects == ix + 1
    return ix


def clip(s, shape, rule=FILL_NON_ZERO):
    ix = s.n_draw_objects
    s.push_clip_layer(rule, I, shape)
    return ix


def ring(outer, inner):
    """Two squares in the same direction: a ring under even-odd, a filled square under nonzero."""
    p = BezPath()
    for a, b in (outer, inner):
        p.move_to(a, a)
        p.line_to(b, a)
        p.line_to(b, b)
        p.line_to(a, b)
        p.close_path()
    return p


def answers(oracle, s, points, w=W, h=H):
    packed = resolve(s.encoding)
    oracle.bind(packed, w, h, BLACK.premul_rgba8_u32(), AA_MSAA16)
    oracle.run("pathtag", "path_tiling")
    got, amb = hit_ref.hit_ref(hit_ref.frame_from_oracle(oracle, packed), np.asarray(points, np.float32), w, h)
    assert not amb.any(), f"points {np.asarray(points)[amb].tolist()} lie on a line"
    return got.tolist()


def test_a_stack_of_overlapping_rects(oracle):
    s = Scene()
    a = fill(s, Rect(10, 10, 90, 90))
    b = fill(s, Rect(40, 40, 120, 120), GREEN)
    c = fill(s, Rect(60, 20, 80, 100), BLUE)
    pts = [(20, 20), (50, 50), (70, 50), (100, 100), (70, 95), (5, 5), (125.5, 125.5), (-1, 5), (5, -0.25), (128, 5), (5, 128),
           (300, 20), (float("nan"), 20), (20, float("nan")), (127.999, 127.999), (0, 0)]
    assert answers(oracle, s, pts) == [a, b, c, b, c, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1]


def test_an_even_odd_ring_and_its_hole(oracle):
    s = Scene()
    below = fill(s, Rect(50, 50, 70, 70), GREEN)
    eo = fill(s, ring((10, 110), (40, 80)), rule=FILL_EVEN_ODD)
    nz = fill(s, ring((112, 126), (116, 122)))  # the same figure under nonzero: no hole
    assert answers(oracle, s, [(20, 20), (60, 60), (45, 45), (105, 60), (119, 119), (113, 113)]) == [eo, below, -1, eo, nz, nz]


def test_a_draw_in_a_clip_that_excludes_the_point_and_the_draw_below(oracle):
    s = Scene()
    bg = fill(s, Rect(0, 0, 128, 128))
    clip(s, Rect(0, 0, 64, 128))
    inner = fill(s, Rect(32, 32, 96, 96), GREEN)
    s.pop_layer()
    assert answers(oracle, s, [(40, 40), (80, 40), (10, 10), (63.5, 50), (64.5, 50)]) == [inner, bg, bg, inner, bg]


def test_nested_clips_three_deep(oracle):
    s = Scene()
    bg = fill(s, Rect(0, 0, 128, 128))
    clip(s, Rect(0, 0, 100, 128))
    clip(s, Rect(20, 0, 128, 128))
    clip(s, ring((0, 128), (50, 70)), FILL_EVEN_ODD)  # a frame-sized square with a hole
    deep = fill(s, Rect(0, 0, 128, 128), GREEN)
    s.pop_layer()
    mid = fill(s, Rect(0, 100, 128, 128), BLUE)
    s.pop_layer()
    s.pop_layer()
    top = fill(s, Rect(0, 120, 10, 128))
    pts = [(30, 30), (60, 60), (110, 30), (10, 30), (50, 110), (10, 110), (110, 110), (5, 124), (60, 124)]
    assert answers(oracle, s, pts) == [deep, bg, bg, bg, mid, bg, bg, top, mid]


def test_a_transparent_fill_is_hit(oracle):
    s = Scene()
    fill(s, Rect(0, 0, 100, 100))
    glass = fill(s, Rect(20, 20, 60, 60), CLEAR)
    assert answers(oracle, s, [(30, 30), (70, 70)]) == [glass, 0]


def test_a_blurred_rect_and_an_image_in_their_rectangles(oracle):
    s = Scene()
    blur = s.n_draw_objects
    s.draw_blurred_rounded_rect(I, Rect(40, 40, 80, 80), BLUE, 5.0, 4.0)  # drawn in the rect inflated by 2.5 sigma = 10
    img = s.n_draw_objects
    pixels = np.zeros((12, 16, 4), np.uint8)  # fully transparent: still hit
    s.draw_image(Image(pixels), Affine.translate(90.0, 10.0))
    assert (blur, img) == (0, 1) and s.n_draw_objects == 2
    pts = [(32, 32), (60, 60), (89, 89), (28, 28), (91, 60), (95, 15), (105.5, 21.5), (95, 23), (89, 15)]
    assert answers(oracle, s, pts) == [blur, blur, blur, -1, -1, img, img, -1, -1]


def test_an_empty_shape_encodes_no_draw():
    s = Scene()
    s.fill(FILL_NON_ZERO, I, RED, None, BezPath())
    assert s.n_draw_objects == 0
    s.fill(FILL_NON_ZERO, I, RED, None, Rect(0, 0, 1, 1))
    s.push_clip_layer(FILL_NON_ZERO, I, Rect(0, 0, 1, 1))
    assert s.n_draw_objects == 2
    s.pop_layer()
    assert s.n_draw_objects == 3 == resolve(s.encoding).layout.n_draw_objects


class CountingMirror(MirrorScene):
    """A MirrorScene that checks, after every call, that both front ends count the same draw objects."""


for _name in ("fill", "stroke", "push_layer", "push_luminance_mask_layer", "push_clip_layer", "pop_layer", "draw_image",
              "draw_blurred_rounded_rect", "draw_blurred_rounded_rect_in"):
    def _wrap(name):
        base = getattr(MirrorScene, name)

        def call(self, *a):
            base(self, *a)
            if not getattr(self, "_quiet", False):
                assert self.n_draw_objects == self.native.n_draw_objects == len(self.encoding.draw_tags), name
        return call
    setattr(CountingMirror, _name, _wrap(_name))


@pytest.mark.parametrize("name", RECIPES + ["tricky_strokes", "image_extend_modes"])
def test_native_counts_the_same_draw_objects(monkeypatch, name):
    monkeypatch.setattr(scenes, "Scene", CountingMirror)
    s = getattr(scenes, name)()[0]
    assert isinstance(s, CountingMirror)
    layout = resolve(s.encoding).layout
    assert s.n_draw_objects == s.native.n_draw_objects
    if s.encoding.n_open_clips == 0:
        assert layout.n_draw_objects == s.n_draw_objects
