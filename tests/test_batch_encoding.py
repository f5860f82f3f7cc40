"""Batches of scenes (vb_scene_batch / encoding.batch): the native batch of mirrored scenes resolves to the same bytes as the
Python statement, offsets included, and each scene's open layers are closed right behind it. CPU only."""
import numpy as np
import pytest

from vello_b200 import encoding, scenes
from vello_b200.encoding import DRAWTAG_BEGIN_CLIP, DRAWTAG_END_CLIP, resolve
from vello_b200.scene_native import NativeScene
from vello_b200.shapes import Affine, Circle, Rect

from .test_scene_native import MirrorScene, assert_same


@pytest.fixture()
def mirror(monkeypatch):
    monkeypatch.setattr(scenes, "Scene", MirrorScene)
    return None


def open_layers():
    s = MirrorScene()
    s.fill(encoding.FILL_NON_ZERO, Affine.IDENTITY, encoding.RED, None, Rect(0, 0, 40, 40))
    s.push_clip_layer(encoding.FILL_NON_ZERO, Affine.IDENTITY, Circle(30.0, 30.0, 25.0))
    s.push_layer(encoding.FILL_NON_ZERO, encoding.MIX_MULTIPLY, encoding.COMPOSE_SRC_OVER, 0.5, Affine.IDENTITY, Rect(5, 5, 50, 50))
    s.fill(encoding.FILL_NON_ZERO, Affine.IDENTITY, encoding.Color(0.2, 0.4, 0.6, 0.8), None, Rect(10, 10, 60, 60))
    return s


def native_batch(ss):
    bs, offsets = encoding.batch(ss)
    b = MirrorScene()
    b.encoding = bs.encoding
    n_offsets = b.native.batch([s.native for s in ss])
    return b, offsets, n_offsets


def draw_tags(packed):
    L = packed.layout
    return packed.scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects]


def test_batch_bytes_and_offsets_identical(mirror):
    ss = [scenes.fill_types()[0], open_layers(), MirrorScene(), scenes.brushes()[0], scenes.many_clips()[0], open_layers(),
          scenes.random_small(3)[0]]
    b, offsets, n_offsets = native_batch(ss)
    assert offsets == n_offsets
    assert_same(b)
    packed = resolve(b.encoding)
    assert offsets[0] == 0 and offsets[-1] == packed.layout.n_draw_objects
    assert all(a <= c for a, c in zip(offsets, offsets[1:]))
    tags = draw_tags(packed)
    for c in range(len(ss)):  # every cell balances its clips by itself
        t = tags[offsets[c]:offsets[c + 1]]
        assert int((t == DRAWTAG_BEGIN_CLIP).sum()) == int((t == DRAWTAG_END_CLIP).sum()), c
    # a cell holds the draw tags its scene resolves to alone, the trailing END_CLIPs of its open layers included
    for c, s in enumerate(ss):
        p = resolve(s.encoding)
        L = p.layout
        alone = p.scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects + s.encoding.n_open_clips]
        assert np.array_equal(tags[offsets[c]:offsets[c + 1]], alone), c


def test_closing_tags_are_pop_layers(mirror):
    """The tags that close a scene's open layers are those of pop_layer: the batch of one open scene is the scene popped."""
    s, popped = open_layers(), open_layers()
    popped.pop_layer()
    popped.pop_layer()
    b, offsets, _ = native_batch([s])
    assert offsets == [0, popped.encoding.n_paths]
    assert resolve(b.encoding).scene.tobytes() == resolve(popped.encoding).scene.tobytes()


def test_empty_batch_and_bad_arguments():
    b, offsets = encoding.batch([])
    assert offsets == [0] and resolve(b.encoding).layout.n_draw_objects == 0
    n = NativeScene()
    assert n.batch([]) == [0]
    with pytest.raises(Exception):
        n.batch([n])  # a scene cannot be a part of its own batch
