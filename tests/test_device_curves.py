"""Curved fragments from device arrays, without a GPU: the `point_kinds` checks of `Renderer.upload_device_paths`, which raise
before the library is called; the worst-case stream lengths against the host encoder on random curved rings; and the
parallel decision rule of k_device_paths.cu (tests/device_curves_ref.py) against the PathEncoder on thousands of random
degenerate rings, with the walk flag set exactly where the rule needs the encoders' order."""
import numpy as np
import pytest

from vello_b200.encoding import Encoding
from vello_b200.shapes import Arc, Circle, Ellipse, RoundedRect, path_elements

from . import device_curves_ref as ref
from .test_device_paths import Dev, Lib, worst_case


@pytest.fixture
def r():
    from vello_b200.renderer import Renderer
    r = Renderer.__new__(Renderer)
    r.lib, r.handle = Lib(), None
    return r


PTS, ROFF, COLS = Dev((4, 2), "<f4"), Dev((2,), "<i4"), Dev((1, 4), "<f4")


@pytest.mark.parametrize("kinds, match", [
    (Dev((4,), "<i4"), "uint8 or bool"),
    (Dev((4,), "<f4"), "uint8 or bool"),
    (Dev((4, 1), "|u1"), "1-D"),
    (Dev((3,), "|u1"), "3 entries for 4 points"),
    (Dev((5,), "|b1"), "5 entries for 4 points"),
    (Dev((4,), "|u1", strides=(2,)), "contiguous"),
    (np.zeros(4, np.uint8), "__cuda_array_interface__"),
])
def test_point_kinds_checks(r, kinds, match):
    with pytest.raises((ValueError, TypeError), match=match):
        r.upload_device_paths(PTS, ROFF, COLS, point_kinds=kinds)


def random_curved(rng, n_paths, pool, max_rings=3, max_segments=5):
    """Random paths of rings with random L / Q / C segments over a small pool of coordinate values."""
    pts, kinds, roff, poff = [], [], [0], [0]
    for _ in range(n_paths):
        for _ in range(int(rng.integers(0, max_rings + 1))):
            if rng.random() < 0.1:
                roff.append(len(pts))  # an empty ring
                continue
            pts.append((rng.choice(pool), rng.choice(pool)))
            kinds.append(0)
            for _ in range(int(rng.integers(0, max_segments + 1))):
                deg = int(rng.integers(1, 4))
                for k in range(deg):
                    pts.append((rng.choice(pool), rng.choice(pool)))
                    kinds.append(0 if k == deg - 1 else 1)
            if rng.random() < 0.3:  # a curved closing segment onto a repeat of the first point
                pts.append((rng.choice(pool), rng.choice(pool)))
                kinds.append(1)
                pts.append(pts[roff[-1]])
                kinds.append(0)
            roff.append(len(pts))
        poff.append(len(roff) - 1)
    return np.array(pts, np.float32).reshape(-1, 2), np.array(kinds, np.uint8), roff, poff


def host_encoded(pts, kinds, roff, poff, stroke, closed):
    """(tag bytes, path-data words) of the PathEncoder over each path's element list."""
    e = Encoding()
    closes = closed or not stroke
    for i in range(len(poff) - 1):
        els = []
        for k in range(poff[i], poff[i + 1]):
            if roff[k] < roff[k + 1]:
                els += ref.elements(pts, kinds, roff[k], roff[k + 1]) + ([("Z",)] if closes else [])
        e.encode_path_elements(els, not stroke)
    return list(e.path_tags), np.array(e.path_data, np.float32)


POOL = [0.0, -0.0, 1.0, 5.0, 2e-12, 7.5]
EPS_POOL = [0.0, -0.0, 4e-13, 8e-13, -8e-13, 1e-12, 2e-12, -2e-12, 3e-12, 1.0]


@pytest.mark.parametrize("seed", range(12))
def test_worst_case_bounds_the_encoder(seed):
    """The allocation vb_fragment_from_device_curves makes (the polyline worst case of the counts) holds every curved
    encoding: a kept segment's points write two words each and its one tag belongs to its end point."""
    rng = np.random.default_rng(seed)
    pts, kinds, roff, poff = random_curved(rng, int(rng.integers(0, 12)), POOL)
    for stroke in (False, True):
        for closed in (False, True):
            tags, data = host_encoded(pts, kinds, roff, poff, stroke, closed)
            n_paths = len(poff) - 1
            got = (len(tags) + (2 if n_paths else 0), len(data), tags.count(ref.TAG_PATH))
            bound = worst_case(len(pts), len(roff) - 1, n_paths)
            assert got[0] <= bound[0] and got[1] <= bound[1] and got[2] <= bound[2], (got, bound)
            # the packed block scan: at most 4 tags and 6 words a point, 256 points a partition, within 11 bits each
            assert 4 * 256 < 1 << 11 and 6 * 256 < 1 << 11


@pytest.mark.parametrize("pool", [POOL, EPS_POOL], ids=["values", "eps"])
@pytest.mark.parametrize("seed", range(4))
def test_parallel_rule_is_the_encoder(pool, seed):
    """The rule of the kernels, point for point against the PathEncoder, on random degenerate curved rings: the first kept
    segment by the tangent test, later ones by the span against their own start, and the walk where that is not exact."""
    rng = np.random.default_rng(100 + seed)
    walked = unwalked = 0
    for _ in range(250):
        pts, kinds, roff, poff = random_curved(rng, int(rng.integers(1, 5)), pool)
        for stroke, closed in ((False, True), (True, False), (True, True)):
            want_tags, want_data = host_encoded(pts, kinds, roff, poff, stroke, closed)
            tags, data, w = ref.encode(pts, kinds, roff, poff, stroke, closed)
            assert tags == want_tags, (pts.tolist(), kinds.tolist(), roff, poff, stroke, closed)
            assert data.view(np.uint32).tolist() == want_data.view(np.uint32).tolist()
            walked += len(w)
            unwalked += len(roff) - 1 - len(w)
    assert unwalked > 0
    if pool is EPS_POOL:
        assert walked > 0, "the pool makes rings that need the walk"


def test_walk_flag_is_needed():
    """Without the walk, the rule differs from the encoder on a ring that drops an EPS-close segment ending unequal to its
    start: the flag is not merely conservative there."""
    e = 6e-13
    P = np.array([(0, 0), (2e-12, 0), (2e-12 + e, 0), (2e-12 + 2 * e, 0)], np.float32)
    keep, first, last, deg, walk = ref.ring_rule(P, [0, 0, 0, 0])
    assert walk and first == 1 and keep == {1: True, 2: False, 3: True}


def test_tangent_is_not_the_span():
    """A quad whose span exceeds EPS while neither point is EPS-far from p0 is dropped in the MoveTo state."""
    P = np.array([(0, 0), (8e-13, 0), (-8e-13, 0), (5, 5)], np.float32)
    keep, first, last, deg, walk = ref.ring_rule(P, [0, 1, 0, 0])
    assert first == 3 and not keep[2]
    e = Encoding()
    e.encode_path_elements(ref.elements(P, [0, 1, 0, 0], 0, 4) + [("Z",)], True)
    assert e.path_tags[0] == ref.TAG_LINE


@pytest.mark.parametrize("shape", [Circle(50, 60, 20), Circle(0, 0, 5000), Ellipse(40, 40, 30, 10, 0.4),
                                   RoundedRect(10, 10, 90, 60, 12), Arc(50, 50, 30, 20, 0.3, 4.0)],
                         ids=["circle", "circle_n8", "ellipse", "rounded_rect", "arc"])
def test_kurbo_shapes_round_trip(shape):
    """Points and kinds of a shape's elements give back the shape's encoding under the rule."""
    els = list(path_elements(shape, 0.1))
    pts, kinds, roff = ref.points_of(els)
    closes = els[-1][0] == "Z"
    for stroke in (False, True):
        e = Encoding()
        e.encode_path_elements(els, not stroke)
        tags, data, _ = ref.encode(pts, kinds, roff, [0, len(roff) - 1], stroke, closes)
        assert tags == list(e.path_tags) and (data.view(np.uint32) == np.array(e.path_data, np.float32).view(np.uint32)).all()
