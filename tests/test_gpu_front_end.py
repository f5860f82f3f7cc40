"""The front end of a frame: the path tag scan at its partition edges, and draw / clip's links running beside flatten.

`k_pathtag_scan` scans PT_PART tag words per CTA, loads them as 16-byte vectors (scalar loads for a tag stream that does not
start on a 16-byte boundary, and for a partition's last words) and stores the partition's monoids as 16-byte words staged
in shared memory. Its `tag_monoids` must equal the oracle's at tag-word counts on both sides of the partition size and its
multiples. It also writes the path table draw reads (`path_draw`: a path's style and transform index), which must give
the fields flatten stores in `path_bboxes`.

Whole frames launch draw and clip's depth scan and links on a second stream beside flatten; with per-stage timing on they
run serially. Both must give the oracle's draw and clip buffers and the same pixels, with the same kernel launches.
"""
import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, Packed, resolve
from oracle.vbo import DTYPES

from . import parity

pytestmark = pytest.mark.gpu

PT_PART = 2048  # tag words per CTA of k_pathtag_scan (k_pathtag.cu)
STYLE_FLAGS_FILL = 0x40000000  # a style word's fill-rule bit
COUNTS = [1, 3, 4, 5, PT_PART - 1, PT_PART, PT_PART + 1, 2 * PT_PART - 1, 2 * PT_PART + 1, 3 * PT_PART, 7 * PT_PART - 1,
          7 * PT_PART + 1, 40 * PT_PART + 3]


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def with_tag_stream(packed: Packed, words: np.ndarray, lead: int) -> Packed:
    """`packed` with its tag stream replaced by `words`, starting `lead` words into the scene."""
    lay = packed.layout
    old = lay.path_data_base - lay.path_tag_base
    scene = np.concatenate([np.zeros(lead, np.uint32), words.astype(np.uint32), packed.scene[lay.path_data_base:]])
    shift = lead + words.size - old
    layout = type(lay)(**vars(lay))
    layout.path_tag_base = lead
    for f in ("path_data_base", "draw_tag_base", "draw_data_base", "transform_base", "style_base"):
        setattr(layout, f, getattr(lay, f) + shift)
    return Packed(scene, layout, packed.ramps, packed.atlas)


@pytest.mark.parametrize("lead", [0, 1, 2])
@pytest.mark.parametrize("n_words", COUNTS)
def test_tag_monoids_at_partition_edges(renderer, oracle, n_words, lead):
    """Random tag words: every field of the monoid grows, across CTAs and inside the last, partial one. A lead of 1 or 2
    words puts the stream off the 16-byte grid (the scalar loads)."""
    s, w, h = scenes.filled_square()
    rng = np.random.default_rng(n_words * 3 + lead)
    packed = with_tag_stream(resolve(s.encoding), rng.integers(0, 1 << 32, n_words, dtype=np.uint64).astype(np.uint32), lead)
    p = RenderParams(BLACK, w, h, AA_AREA)
    renderer.upload(packed)
    renderer.run_stages(p, "pathtag", "pathtag")
    oracle.bind(packed, w, h)
    oracle.run("pathtag", "pathtag")
    g, c = renderer.download("tag_monoids", DTYPES["tag_monoids"]), oracle.buffer("tag_monoids")
    assert g.shape == c.shape == (n_words,)
    bad = np.nonzero(g.view(np.uint32).reshape(-1, 5) != c.view(np.uint32).reshape(-1, 5))[0]
    assert bad.size == 0, f"{np.unique(bad).size} tag monoids differ, first at word {int(bad[0])}"


def headline():
    return resolve(scenes.paris_like(30000, 4096, 30000).encoding), 4096, 4096


def clips():
    return resolve(scenes.beziers_clips(20000, 1000, 2048, seed=7).encoding), 2048, 2048


@pytest.mark.parametrize("make", [headline, clips], ids=["paris-30k", "beziers-clips"])
def test_draw_and_clip_beside_flatten(renderer, oracle, make):
    """A whole frame (draw and clip's links forked beside flatten): the front end's buffers equal the oracle's, and the path
    table equals what flatten stored in the path boxes."""
    packed, w, h = make()
    renderer.render_to_texture(packed, RenderParams(BLACK, w, h, AA_MSAA16))
    assert renderer.last_stats.failed == 0
    oracle.bind(packed, w, h, BLACK.premul_rgba8_u32(), AA_MSAA16)
    oracle.run("pathtag", "clip")
    parity.compare_all(renderer, oracle, packed.layout, w, h, before="binning")
    pd = renderer.download("path_draw", np.uint32).reshape(-1, 2)
    bb = oracle.buffer("path_bboxes")
    assert pd.shape[0] == packed.layout.n_paths
    styles = packed.scene[packed.layout.style_base + pd[:, 0]]
    assert np.array_equal((styles & STYLE_FLAGS_FILL) != 0, bb["draw_flags"] != 0), "draw flags"
    assert np.array_equal(pd[:, 1], bb["trans_ix"]), "transform indices"


@pytest.mark.parametrize("make", [headline, clips], ids=["paris-30k", "beziers-clips"])
def test_forked_and_serial_frames_are_identical(make):
    """Frames with the fork (no timing) and serial frames (per-stage timing) give the same pixels and launch the same kernels.
    MSAA pixels are integer sample counts, so they are the same bytes however the kernels overlap; area AA sums a tile's
    segments in the order path_tiling's atomics gave them, which differs from frame to frame by a last bit anyway.
    Launches are compared between frames launched kernel by kernel (a replayed graph counts a host destination's bands
    differently), which per-stage timing always is."""
    from vello_b200.renderer import Renderer, RendererOptions
    packed, w, h = make()
    out = {}
    for timing in (False, True):
        r = Renderer(RendererOptions(timing=timing))
        try:
            for aa in (AA_MSAA8, AA_MSAA16):
                p = RenderParams(BLACK, w, h, aa)
                r.set_cuda_graph(True)
                img = r.render_to_texture(packed, p)
                again = r.render_to_texture(packed, p)  # without timing: the second frame replays a graph
                r.set_cuda_graph(False)
                direct = r.render_to_texture(packed, p)
                assert np.array_equal(img, again) and np.array_equal(img, direct)
                out[timing, aa] = (img, r.last_stats.kernel_launches)
        finally:
            r.close()
    for aa in (AA_MSAA8, AA_MSAA16):
        (a, la), (b, lb) = out[False, aa], out[True, aa]
        assert la == lb, f"aa={aa}: {la} launches with the fork, {lb} serial"
        assert np.array_equal(a, b), f"aa={aa}: {int((a != b).any(axis=2).sum())} pixels differ between forked and serial frames"
