"""Bump-arena overflow and the grow-and-re-run protocol, driven at each arena's capacity boundary.

Seven arenas are sized by guesses (lines, binning, tiles, seg_counts, segments, blend, ptcl). A kernel that allocates from
one compares against its capacity, keeps counting past it and sets its stage bit in bump.failed; later stages skip, fine
paints nothing, and the renderer grows every arena whose counter exceeds its capacity and runs the frame again. A fresh
renderer takes this path on the first frames of every new scene size, in every entry point.

`Renderer.limit_arena` lowers the capacity the kernels see without shrinking the allocation and fills the bytes past the
limit with a canary. Every limit here is set on a renderer that has already rendered the same frame, so every write a kernel
could make lies inside an allocation: a missing or off-by-one capacity check shows up as a changed canary byte, or as a
frame that fails at exactly its need, never as an out-of-bounds access. Run with `pytest -m gpu`.
"""
import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, resolve
from vello_b200.shapes import Affine, Circle

from . import parity

pytestmark = pytest.mark.gpu

W = H = 512
N_TILES = (W // 16) * (H // 16)
ARENAS = ["lines", "binning", "tiles", "seg_counts", "segments", "blend", "ptcl"]
# VB_STAGE_* bit each arena's overflow raises, and the stage that allocates from it (the last one whose output a failed
# attempt still has to have computed in full is the one before it)
FLATTEN, BINNING, TILE_ALLOC, PATH_COUNT, COARSE, FINE_SEGMENTS = 0x4, 0x1, 0x2, 0x8, 0x10, 0x20
BIT = {"lines": FLATTEN, "binning": BINNING, "tiles": TILE_ALLOC, "seg_counts": PATH_COUNT, "segments": FINE_SEGMENTS,
       "blend": COARSE, "ptcl": COARSE}
STAGE = {"lines": "flatten", "binning": "binning", "tiles": "tile_alloc", "seg_counts": "path_count", "segments": "path_tiling",
         "blend": "coarse", "ptcl": "coarse"}
GUARDS = {a: [a] for a in ARENAS}
GUARDS["lines"] = ["lines", "line_scratch", "flatten_jobs"]
SMALLEST = {a: 1 for a in ARENAS}
SMALLEST["ptcl"] = N_TILES * 64  # the static area: every dynamic chunk overflows
GUARD_BYTE = 0xA5


def composite():
    """One 512x512 frame in which every bump counter is non-zero: a paris-like cut (lines, binning, tiles, crossings),
    stroke_styles (round joins: both the lean and the general flatten kernels run), deep_blend (nesting deeper than
    VB_BLEND_STACK_SPLIT: blend spill) and a stack of translucent circles over a few tiles (many dynamic PTCL chunks)."""
    s = scenes.paris_like(600, 512, seed=11)
    s.append(scenes.stroke_styles()[0], Affine.translate(0.0, 250.0) * Affine.scale(0.45))
    s.append(scenes.deep_blend()[0], Affine.translate(300.0, 300.0))
    for k in range(160):
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8((37 * k) % 256, (91 * k) % 256, 200, 40), None,
               Circle(430.0 + (k % 5) * 3.0, 80.0 + (k % 7) * 2.0, 36.0))
    return resolve(s.encoding)


@pytest.fixture(scope="module")
def packed():
    return composite()


def needs(bump):
    """Each arena's need in the units of its limit, from the bump counters of an attempt."""
    return {"lines": int(bump["lines"]), "binning": int(bump["binning"]), "tiles": int(bump["tile"]),
            "seg_counts": int(bump["seg_counts"]), "segments": int(bump["segments"]), "blend": int(bump["blend"]),
            "ptcl": N_TILES * 64 + int(bump["ptcl"])}


def gpu_bump(r):
    from oracle.vbo import DTYPES
    return r.download("bump", DTYPES["bump"])[0]


def ample(packed, aa, **options):
    """A renderer whose arenas hold the frame: vb_render grows them, then one single attempt gives the counters."""
    from vello_b200.renderer import Renderer, RendererOptions, VelloB200Error
    r = Renderer(RendererOptions(**options))
    p = RenderParams(BLACK, W, H, aa)
    for attempt in range(3):  # a small max_retries may need more than one call to grow from the first guesses
        try:
            r.render_to_texture(packed, p)
            break
        except VelloB200Error:
            assert attempt < 2
    r.upload(packed)
    r.run_stages(p, "pathtag", "fine")
    b = gpu_bump(r)
    assert int(b["failed"]) == 0
    return r, p, needs(b)


def assert_pixels(img, ref, aa):
    d = np.abs(img.astype(np.int32) - ref.astype(np.int32))
    assert d.max() <= (1 if aa == AA_AREA else 0), f"aa={aa}: max diff {d.max()}, {int((d > 0).sum())} channel values differ"


def assert_guards(r, arena):
    for g in GUARDS[arena]:
        guard = r.download_guard(g)
        assert g != arena or len(guard) > 0, "the limit is below the allocation: a guard region exists"
        bad = np.nonzero(guard != GUARD_BYTE)[0]
        assert len(bad) == 0, f"{g}: {len(bad)} of {len(guard)} guard bytes overwritten, first at byte {int(bad[0])} past the limit"


def test_composite_counters(packed, oracle):
    """The scene reaches every arena; two ample attempts count the same; the counters are the oracle's."""
    r, p, need = ample(packed, AA_MSAA16)
    print("need", need)
    assert all(v > 0 for v in need.values()), need
    assert need["ptcl"] > N_TILES * 64 + 2 * 256, "several dynamic PTCL chunks"
    r.run_stages(p, "pathtag", "fine")
    assert needs(gpu_bump(r)) == need
    oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    ob = oracle.buffer("bump")[0]
    holes = int(r.download("seg_holes", np.uint32)[0])
    got = dict(need, segments=need["segments"] - holes)
    for a, f in (("lines", "lines"), ("tiles", "tile"), ("seg_counts", "seg_counts"), ("segments", "segments"), ("binning", "binning"),
                 ("blend", "blend")):
        assert got[a] == int(ob[f]), (a, got[a], int(ob[f]))
    r.close()


BOUNDARY = [(a, AA_MSAA16) for a in ARENAS] + [("lines", AA_AREA), ("ptcl", AA_AREA)]


@pytest.mark.parametrize("arena,aa", BOUNDARY)
def test_limit_equal_to_need_fits(packed, oracle, arena, aa):
    """limit = need: the attempt succeeds and is the oracle's frame, stage by stage and in pixels."""
    r, p, need = ample(packed, aa)
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), aa)
    r.limit_arena(arena, need[arena])
    r.run_stages(p, "pathtag", "fine")
    assert int(gpu_bump(r)["failed"]) == 0
    parity.compare_all(r, oracle, packed.layout, W, H)
    assert_pixels(r.download_target(p), ref, aa)
    assert_guards(r, arena)
    r.close()


@pytest.mark.parametrize("which", ["need-1", "smallest"])
@pytest.mark.parametrize("arena,aa", BOUNDARY)
def test_limit_below_need_fails_cleanly(packed, oracle, arena, aa, which):
    """limit < need, one attempt: exactly this arena's stage bit, its counter still reaches the full need (so one re-run
    with a grown arena is enough), nothing written past the limit, fine paints nothing, and every stage before the failing
    one computed exactly what the oracle computes."""
    r, p, need = ample(packed, aa)
    oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), aa)
    before = r.download_target(p)
    limit = need[arena] - 1 if which == "need-1" else SMALLEST[arena]
    r.limit_arena(arena, limit)
    r.run_stages(p, "pathtag", "fine")
    b = gpu_bump(r)
    assert int(b["failed"]) == BIT[arena], (hex(int(b["failed"])), arena, limit)
    assert needs(b)[arena] == need[arena]
    assert_guards(r, arena)
    assert np.array_equal(r.download_target(p), before), "fine painted a failed attempt"
    parity.compare_all(r, oracle, packed.layout, W, H, before=STAGE[arena])
    r.close()


@pytest.mark.parametrize("arena", ARENAS)
def test_render_recovers_with_one_retry(packed, oracle, arena):
    """vb_render with limit = need - 1: one re-run, the oracle's pixels, and the limit is gone for the next frame."""
    r, p, need = ample(packed, AA_MSAA16)
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    r.limit_arena(arena, need[arena] - 1)
    img = r.render_to_texture(packed, p)
    assert r.last_stats.retries == 1
    assert np.array_equal(img, ref)
    assert np.array_equal(r.render_to_texture(packed, p), ref)
    assert r.last_stats.retries == 0
    r.close()


# Every arena at its smallest limit. A stage skips while an earlier one has failed (k_binning: flatten; k_tile_alloc:
# binning or flatten; k_path_count and k_backdrop: any bit; k_coarse: binning, tile_alloc, flatten or path_count), and a
# limit is dropped only once its own counter has exceeded it, so the overflows surface one attempt at a time. coarse
# raises its bit for ptcl and blend, and k_path_tiling checks the segments coarse reserved in the same attempt.
CASCADE = [FLATTEN, BINNING, TILE_ALLOC, PATH_COUNT, COARSE | FINE_SEGMENTS]


def limit_all(r):
    for a in ARENAS:
        r.limit_arena(a, SMALLEST[a])


def test_cascade_bits_per_attempt(packed):
    """The attempts of the cascade one by one: dropping the limits of the arenas that overflowed (what growing does)
    surfaces the next stage's overflow."""
    r, p, need = ample(packed, AA_MSAA16)
    limit_all(r)
    seen = []
    for _ in range(len(CASCADE) + 1):
        r.run_stages(p, "pathtag", "fine")
        b = gpu_bump(r)
        seen.append(int(b["failed"]))
        if not seen[-1]:
            break
        for a, v in needs(b).items():
            if v > SMALLEST[a]:
                r.limit_arena(a, r.NO_LIMIT)
    assert seen == CASCADE + [0], [hex(v) for v in seen]
    r.close()


def test_cascade_retry_budget(packed, oracle):
    """vb_render needs len(CASCADE) re-runs: with max_retries equal to that it is exact; with one fewer the call reports
    VB_E_BUMP_OVERFLOW with a message, and the same renderer then renders the next frame exactly."""
    from vello_b200.renderer import VelloB200Error
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    r, p, _ = ample(packed, AA_MSAA16, max_retries=len(CASCADE))
    limit_all(r)
    assert np.array_equal(r.render_to_texture(packed, p), ref)
    assert r.last_stats.retries == len(CASCADE)
    r.close()
    r, p, _ = ample(packed, AA_MSAA16, max_retries=len(CASCADE) - 1)
    limit_all(r)
    with pytest.raises(VelloB200Error, match="bump arena overflow") as e:
        r.render_to_texture(packed, p)
    assert "[bump overflow persisted]" in str(e.value)  # vb_last_error
    assert np.array_equal(r.render_to_texture(packed, p), ref)
    r.close()


# ---- the other entry points, for one early arena (lines: flatten) and one late one (ptcl: coarse) -----------------------
ENTRY_ARENAS = ["lines", "ptcl"]


def stats_need(st):
    return needs({f: getattr(st, f) for f in ("lines", "binning", "tile", "seg_counts", "segments", "blend", "ptcl")})


@pytest.mark.parametrize("arena", ENTRY_ARENAS)
@pytest.mark.parametrize("window", [dict(tile_rows=(5, 23)), dict(bin_rows=(1, 2))])
def test_one_overflow_in_a_stripe(packed, oracle, arena, window):
    """A tile-row stripe and a bin-row stripe without tile 0: one re-run, the oracle's rows."""
    from vello_b200.renderer import Renderer
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    r = Renderer()
    p = RenderParams(BLACK, W, H, AA_MSAA16)
    h0, h1 = r.stripe_rows(p, window.get("bin_rows", (0, 0)), window.get("tile_rows", (0, 0)))
    assert np.array_equal(r.render_to_texture(packed, p, **window), ref[h0:h1])
    need = stats_need(r.last_stats)
    r.limit_arena(arena, need[arena] - 1)
    assert np.array_equal(r.render_to_texture(packed, p, **window), ref[h0:h1])
    assert r.last_stats.retries == 1
    assert np.array_equal(r.render_to_texture(packed, p, **window), ref[h0:h1])
    assert r.last_stats.retries == 0
    r.close()


@pytest.mark.parametrize("arena", ENTRY_ARENAS)
@pytest.mark.parametrize("graph", [True, False])
def test_one_overflow_with_and_without_graphs(packed, oracle, arena, graph):
    """The limit changes the config, which is part of the graph key: a captured and replayed frame is captured again for
    the failing attempt and for the re-run."""
    from vello_b200.renderer import Renderer
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    r = Renderer()
    r.set_cuda_graph(graph)
    p = RenderParams(BLACK, W, H, AA_MSAA16)
    r.render_to_texture(packed, p)
    r.upload(packed)
    for _ in range(2):  # captured, then replayed
        r.render_resident(p)
    need = stats_need(r.last_stats)
    assert np.array_equal(r.download_target(p), ref)
    r.limit_arena(arena, need[arena] - 1)
    assert r.render_resident(p).retries == 1
    assert np.array_equal(r.download_target(p), ref)
    assert r.render_resident(p).retries == 0
    assert np.array_equal(r.download_target(p), ref)
    r.close()


@pytest.mark.parametrize("arena", ENTRY_ARENAS)
@pytest.mark.parametrize("younger_overflows", [False, True])
def test_one_overflow_while_streaming(packed, arena, younger_overflows):
    """render_stream with the limit set before frame k. The frame enqueued behind it either fits (only k is re-run) or
    overflows too (both are re-run). Either way every frame arrives, in order, equal to the blocking frame."""
    from vello_b200.renderer import Renderer
    light = resolve(scenes.paris_like(150, 512, seed=12).encoding)
    k = 3
    seq = [packed, light, packed, packed, packed if younger_overflows else light, packed]
    p = RenderParams(BLACK, W, H, AA_MSAA16)
    r = Renderer()
    want, need = [], {}
    for s in seq:  # blocking frames: the arenas hold every frame of the sequence
        want.append(r.render_to_texture(s, p))
        need[id(s)] = stats_need(r.last_stats)
    limit = need[id(packed)][arena] - 1
    assert (need[id(seq[k + 1])][arena] > limit) == younger_overflows
    got = []
    for img in r.render_stream(seq, p):
        got.append(img.copy())
        if len(got) == k - 2:  # vb_render_begin(k - 1) has returned; frame k is the next one submitted
            r.limit_arena(arena, limit)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), i
    assert np.array_equal(r.render_to_texture(packed, p), want[0])
    assert r.last_stats.retries == 0
    r.close()


@pytest.mark.parametrize("arena", ENTRY_ARENAS)
@pytest.mark.parametrize("exchange", [False, True])
def test_one_overflow_in_a_group(packed, oracle, arena, exchange):
    """RendererGroup([0] * 3) with the limit on renderer 1 only: re-run by that renderer alone (exchange off) or re-issued
    on every renderer together (exchange on); the assembled frame is the oracle's."""
    from vello_b200.renderer import RendererGroup
    ref = oracle.render(packed, W, H, BLACK.premul_rgba8_u32(), AA_MSAA16)
    p = RenderParams(BLACK, W, H, AA_MSAA16)
    g = RendererGroup([0] * 3)
    g.set_balancing(False)  # the same stripes every frame: renderer 1's arenas hold its next frame
    g.set_exchange(exchange)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    need = stats_need(g.last_stats[1])
    g.renderer(1).limit_arena(arena, need[arena] - 1)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    if not exchange:
        assert [int(s.retries) for s in g.last_stats] == [0, 1, 0]
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    assert all(int(s.retries) == 0 and int(s.failed) == 0 for s in g.last_stats)
    g.close()
