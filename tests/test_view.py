"""Views of a resident scene on the host side: `encoding.viewed`, the transform mapping that `Renderer.set_view` performs on the
device, is `Scene().append(scene, view)` byte for byte, and the view API rejects what it must (no GPU needed)."""
import math

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.encoding import Scene, resolve, viewed
from vello_b200.shapes import Affine


def appended(scene: Scene, view: Affine) -> Scene:
    out = Scene()
    out.append(scene, view)
    return out


def random_affines(seed: int, n: int):
    """Rotations, mirrors, skews and non-uniform scales from 1e-3 to 1e3, with fractional translations."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        sx, sy = 10.0 ** rng.uniform(-3, 3, 2)
        if rng.random() < 0.3:
            sx = -sx  # mirror
        t = Affine.rotate(float(rng.uniform(-math.pi, math.pi))) * Affine.scale(float(sx), float(sy))
        if rng.random() < 0.5:
            t = Affine((1.0, 0.0, float(rng.uniform(-2, 2)), 1.0, 0.0, 0.0)) * t  # skew
        out.append(Affine.translate(float(rng.uniform(-5000, 5000)), float(rng.uniform(-5000, 5000))) * t)
    return out


SCENES = {
    "tiger": lambda: scenes.tiger(256, 256),
    "stroke_styles": lambda: scenes.stroke_styles()[0],
    "brushes": lambda: scenes.brushes()[0],
    "many_clips": lambda: scenes.many_clips()[0],
    "paris_like": lambda: scenes.paris_like(300, 512, seed=3),
}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_viewed_equals_append(name):
    scene = SCENES[name]()
    packed = resolve(scene.encoding)
    views = [Affine(), Affine.translate(7.0, -3.0), Affine.translate(0.37, 12.625), Affine.scale(-1.0, 1.0)] + random_affines(len(name), 12)
    for v in views:
        want = resolve(appended(scene, v).encoding)
        got = viewed(packed, v)
        assert got.layout == want.layout
        assert got.scene.tobytes() == want.scene.tobytes(), v.coeffs
        assert np.array_equal(got.ramps, want.ramps) and np.array_equal(got.atlas, want.atlas)


def test_viewed_leaves_the_scene_alone():
    packed = resolve(scenes.tiger(128, 128).encoding)
    before = packed.scene.copy()
    viewed(packed, Affine.scale(3.0, 0.5))
    assert np.array_equal(packed.scene, before)


def test_view_product_is_unfused_f32():
    """The association and rounding of math.rs:51-73 that the device kernel restates: each product and sum rounded to f32,
    translation ((a*e' + c*f') + e)."""
    s = Scene()
    s.append(scenes.stroke_styles()[0], None)
    packed = resolve(s.encoding)
    v = Affine((1.0000001, 3e-8, -2.5e-8, 0.9999999, 1234.567, -0.001))
    t = packed.scene[packed.layout.transform_base:packed.layout.style_base].view(np.float32).reshape(-1, 6).astype(np.float64)
    got = viewed(packed, v).scene[packed.layout.transform_base:packed.layout.style_base].view(np.float32).reshape(-1, 6)
    a = [np.float32(x) for x in v.coeffs]
    f = np.float32
    for row, g in zip(t, got):
        b = [f(x) for x in row]
        e = f(f(a[0] * b[4]) + f(a[2] * b[5]))
        assert g[4] == f(e + a[4])
        assert g[0] == f(f(a[0] * b[0]) + f(a[2] * b[1]))
