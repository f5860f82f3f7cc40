"""k_flatten against the exact geometry of what it approximates (tests/flatten_ref.py), on the GPU's own lines, and at
the edges of its own machinery.

Every case of tests/test_flatten_geometry.py runs pathtag -> flatten on the GPU: its `lines` must meet the same contract
and equal the oracle's byte for byte, and so must `path_bboxes`. The kernel-edge cases below first show, from flatten's
own scratch records and counters (vb_debug_download "line_scratch", "flatten_jobs", "flatten_counters"), that they reach
the edge they are named for: deferred jobs of FL_DEFER_MIN (3) lines and arcs of FL_ARC_MAX (64), an Euler segment at
the clamp of 100 lines, tags that fill the shared-memory literal cache (6 lines) or spill past it (7), partitions where
only lane 0 or lane 31 needs the general kernel, more than 32 jobs per k_flatten_place warp with runs that cross its
32-line windows, and more than 8,192 partitions for k_flatten_scan. Stripes must equal the whole frame where a miter
tip reaches just into, or stops just short of, the other stripe. Every case also goes through `compare_all`, the
replayed fine in area AA and the pixel bar against the oracle in MSAA16.
"""
import numpy as np
import pytest

from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, STYLE_CAP_BUTT, STYLE_JOIN_MITER, Scene, resolve
from vello_b200.shapes import Affine, BezPath

from . import flatten_ref as ref
from . import parity
from .test_flatten_geometry import (BLOB, CASES, EPS_FILL, EPS_STRAIGHT, FAR_CASES, WHITE, Case, check_case, cubic_path, fill,
                                    polyline, scaled, stroke, tags)

pytestmark = pytest.mark.gpu

LIT = np.dtype([("tag_ix", "<u4"), ("rel", "<u4"), ("path_ix", "<u4"), ("pad", "<u4"), ("p", "<f4", 4)])
JOB = np.dtype([("f", "<f4", 16), ("tex", "<f4"), ("tey", "<f4"), ("tag_ix", "<u4"), ("rel", "<u4"), ("path_ix", "<u4"),
                ("trans_ix", "<u4"), ("meta", "<u4"), ("pad", "<u4")])
FJ_ARC = 0x2000
FL_CACHE, FL_DEFER_MIN, FL_ARC_MAX = 6, 3, 64
GUARDED = ("lines", "line_scratch", "flatten_jobs")


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


def flatten_state(r):
    from oracle.vbo import DTYPES
    bump = r.download("bump", DTYPES["bump"])[0]
    ctr = r.download("flatten_counters", np.uint32)
    lits, jobs = r.download("line_scratch", LIT), r.download("flatten_jobs", JOB)
    assert len(lits) == int(ctr[0]) and len(jobs) == int(ctr[1])
    return dict(lines=r.download("lines", DTYPES["lines"])[: int(bump["lines"])], bump=bump, counters=ctr, lits=lits, jobs=jobs,
                bboxes=r.download("path_bboxes", DTYPES["path_bboxes"]))


def gpu_flatten(r, oracle, case, packed=None):
    """A frame on the GPU (which grows the arenas to what it needs), pathtag -> flatten on the oracle: lines and path
    boxes byte-equal; returns the GPU's flatten state."""
    packed = packed or resolve(case.scene().encoding)
    r.render_to_texture(packed, RenderParams(BLACK, case.w, case.h, AA_AREA))
    st = flatten_state(r)
    assert int(st["bump"]["failed"]) == 0
    oracle.bind(packed, case.w, case.h, BLACK.premul_rgba8_u32(), AA_AREA)
    oracle.run("pathtag", "flatten")
    want = oracle.buffer("lines")
    assert st["lines"].shape == want.shape and st["lines"].tobytes() == want.tobytes(), f"{case.name}: lines differ from the oracle's"
    assert st["bboxes"].tobytes() == oracle.buffer("path_bboxes").tobytes(), f"{case.name}: path_bboxes differ"
    return packed, st


def frame_parity(r, oracle, case, packed):
    from .test_gpu_parity import assert_pixels
    w, h = case.w, case.h
    img = r.render_to_texture(packed, RenderParams(BLACK, w, h, AA_AREA))
    oracle.render(packed, w, h, BLACK.premul_rgba8_u32(), AA_AREA)
    parity.compare_all(r, oracle, packed.layout, w, h)
    parity.assert_replay(r, oracle, packed, img, w, h, AA_AREA, BLACK)
    img16 = r.render_to_texture(packed, RenderParams(BLACK, w, h, AA_MSAA16))
    assert_pixels(img16, oracle.render(packed, w, h, BLACK.premul_rgba8_u32(), AA_MSAA16), AA_MSAA16)


def guarded(r, packed, case, need):
    """The frame again with `lines` limited to exactly what it needs: nothing is written past it, nor past the two scratch
    arenas sized from it."""
    try:
        r.limit_arena("lines", need)
        r.render_to_texture(packed, RenderParams(BLACK, case.w, case.h, AA_AREA))
        st = flatten_state(r)
        assert int(st["bump"]["failed"]) == 0 and int(st["bump"]["lines"]) == need
        for g in GUARDED:
            b = r.download_guard(g)
            over = np.nonzero(b != r.GUARD_BYTE)[0]
            assert len(over) == 0, f"{case.name}: {len(over)} bytes written past {g}, first at byte {int(over[0])}"
    finally:
        r.limit_arena("lines", r.NO_LIMIT)


def n_of(jobs):
    return jobs["meta"] & 0xFF


@pytest.mark.parametrize("case", CASES + FAR_CASES, ids=repr)
def test_gpu_flatten_geometry(renderer, oracle, case):
    packed, st = gpu_flatten(renderer, oracle, case)
    paths, _ = check_case(case, st["lines"])
    assert case.expect <= tags(paths), (case.name, sorted(case.expect - tags(paths)))
    frame_parity(renderer, oracle, case, packed)
    if case.runaway or case.name.startswith(("far-", "circle-1e+06", "round-cap-1e+06")):
        guarded(renderer, packed, case, int(st["bump"]["lines"]))


# ---- the kernel's own edges ----------------------------------------------------------------------------------------------
CUSP2 = [(0.0, 0.0), (1.0, 1.0), (0.0, 1.0), (1.4, 0.2)]


def radius_for_arc_lines(n):
    """A round cap's radius whose half turn flattens to n lines: the angle step 2 acos(1 - 0.25 / r) in the middle of
    [pi / n, pi / (n - 1))."""
    theta = np.pi / (n - 0.5)
    return 0.25 / (1.0 - np.cos(theta / 2))


def test_gpu_defer_min(renderer, oracle):
    """Euler segments of 2 lines stay literal and of 3 become jobs; so do round-join arcs of 2 and 3 lines."""
    case = Case("defer-min", lambda s: (fill(cubic_path(*scaled(CUSP2, 9.25, (10.0, 10.0))))(s),
                                        fill(cubic_path(*scaled([(0.0, 0.5), (0.45, -0.5), (0.55, 1.5), (1.0, 0.5)], 100,
                                                                (14.0, 14.0))))(s),
                                        stroke(polyline([(20.0, 100.0), (70.0, 100.0), (95.0, 57.0)]), width=12.0,
                                               start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT)(s),
                                        stroke(polyline([(20.0, 120.0), (70.0, 120.0), (70.0, 70.0)]), width=12.0,
                                               start_cap=STYLE_CAP_BUTT, end_cap=STYLE_CAP_BUTT)(s)),
                EPS_FILL)
    packed, st = gpu_flatten(renderer, oracle, case)
    check_case(case, st["lines"])
    jobs = st["jobs"]
    euler, arcs = jobs[(jobs["meta"] & FJ_ARC) == 0], jobs[(jobs["meta"] & FJ_ARC) != 0]
    assert n_of(euler).min() == FL_DEFER_MIN, sorted(set(n_of(euler).tolist()))
    assert set(n_of(arcs).tolist()) == {3}, n_of(arcs)  # the 90 degree join; the 60 degree one has 2 lines, literal
    assert set(arcs["path_ix"].tolist()) == {3}
    c = ref.classify_path(ref.decode(case.scene().encoding)[0])
    assert 2 in [e["n"] for e in c["euler"]]
    frame_parity(renderer, oracle, case, packed)


@pytest.mark.parametrize("n", [FL_ARC_MAX, FL_ARC_MAX + 1])
def test_gpu_arc_max(renderer, oracle, n):
    """Round caps of FL_ARC_MAX lines are deferred; one more and they are emitted in place, past the literal cache."""
    r = float(np.float32(radius_for_arc_lines(n)))
    case = Case(f"arc-{n}", stroke(polyline([(64.0 - 3 * r, 64.0), (64.0, 64.0)]), width=2 * r), EPS_STRAIGHT, {f"arc:{n}"})
    packed, st = gpu_flatten(renderer, oracle, case)
    paths, _ = check_case(case, st["lines"])
    assert case.expect <= tags(paths)
    arcs = st["jobs"][(st["jobs"]["meta"] & FJ_ARC) != 0]
    if n <= FL_ARC_MAX:
        assert sorted(n_of(arcs).tolist()) == [n, n]
    else:
        assert len(arcs) == 0
        per_tag = np.bincount(st["lits"]["tag_ix"])
        assert per_tag.max() >= n > FL_CACHE and int(st["counters"][2]) >= 1
    frame_parity(renderer, oracle, case, packed)


def test_gpu_euler_clamp(renderer, oracle):
    """A circle of radius 10^6 px: Euler segments at the clamp of 100 lines, deferred as jobs with FJ_N = 100."""
    case = next(c for c in FAR_CASES if c.name == "circle-1e+06")
    packed, st = gpu_flatten(renderer, oracle, case)
    check_case(case, st["lines"])
    euler = st["jobs"][(st["jobs"]["meta"] & FJ_ARC) == 0]
    assert n_of(euler).max() == 100 and (n_of(euler) == 100).sum() >= 4


def test_gpu_literal_cache_and_spill(renderer, oracle):
    """Two fills whose cubic tag emits 6 literal lines (the whole shared-memory cache) and 7 (one spills)."""
    case = Case("cache-spill", lambda s: (fill(cubic_path(*scaled(CUSP2, 9.25, (10.0, 10.0))))(s),
                                          fill(cubic_path(*scaled(CUSP2, 11.0, (60.0, 60.0))))(s)), EPS_FILL)
    packed, st = gpu_flatten(renderer, oracle, case)
    check_case(case, st["lines"])
    lits = st["lits"]
    assert len(st["jobs"]) == 0
    per_path = {int(p): np.bincount(lits["tag_ix"][lits["path_ix"] == p]).max() for p in (0, 1)}
    assert per_path == {0: FL_CACHE, 1: FL_CACHE + 1}, per_path
    frame_parity(renderer, oracle, case, packed)


@pytest.mark.parametrize("lane", [0, 31])
def test_gpu_one_lane_needs_the_general_kernel(renderer, oracle, lane):
    """A polygon of line-tos (the lean kernel) with one cubic whose tag is lane `lane` of its partition: exactly that
    partition goes on the general kernel's work list."""
    def build(s):
        from vello_b200.encoding import TAG_CUBIC_TO_F32
        p = BezPath()
        n = 150
        pts = [(64 + 50 * np.cos(2 * np.pi * k / n), 64 + 50 * np.sin(2 * np.pi * k / n)) for k in range(n)]
        head = len(s.encoding.path_tags) + 2  # transform and style tags, then the segments
        at = 2 * 32 + lane - head
        p.move_to(*pts[0])
        for k in range(1, n):
            if k - 1 == at:
                a, b = pts[k - 1], pts[k]
                p.curve_to(a[0] + 6, a[1] - 9, b[0] + 9, b[1] + 6, *b)
            else:
                p.line_to(*pts[k])
        p.close_path()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, WHITE, None, p)
        assert s.encoding.path_tags.index(TAG_CUBIC_TO_F32) == 2 * 32 + lane
    case = Case(f"lane-{lane}", build, EPS_FILL)
    packed, st = gpu_flatten(renderer, oracle, case)
    check_case(case, st["lines"])
    assert int(st["counters"][2]) == 1
    assert (st["jobs"]["tag_ix"] == 64 + lane).all()
    assert (st["lits"]["tag_ix"] == 64 + lane).sum() + (st["jobs"]["tag_ix"] == 64 + lane).sum() >= 2  # the cubic's lines
    frame_parity(renderer, oracle, case, packed)


def test_gpu_place_windows(renderer, oracle):
    """More than 32 jobs per k_flatten_place warp, with job runs that cross the warp's 32-line windows (so lane 0
    recomputes its predecessor's end point)."""
    def build(s):
        for k in range(120):
            sc = 20.0 + (k % 7) * 9.0
            fill(cubic_path(*scaled(BLOB, sc, (4.0 + (k % 12) * 10.0, 4.0 + (k // 12) * 11.0))))(s)
    case = Case("place-windows", build, EPS_FILL)
    packed, st = gpu_flatten(renderer, oracle, case)
    check_case(case, st["lines"])
    jobs = st["jobs"]
    assert len(jobs) > 64
    crossing = 0
    for b in range(0, len(jobs) - 31, 32):
        n = n_of(jobs[b: b + 32]).astype(np.int64)
        start = np.cumsum(n) - n
        crossing += int(((start % 32 != 0) & (start // 32 != (start + n - 1) // 32)).sum())
    assert crossing > 0
    frame_parity(renderer, oracle, case, packed)


def test_gpu_scan_past_one_cta(renderer, oracle):
    """More than 8,192 partitions of 32 tags: k_flatten_scan's second CTA and the look-back between them. The scan's
    scalar tail (a partition count that is not a multiple of 8) is unreachable: the tag stream is padded to 1,024 tags,
    so a frame has a multiple of 32 partitions, and a sharded share of one starts and ends on multiples of 8."""
    n = 270_000
    p = BezPath([("M", 2.0, 2.0)] + [("L", 2.0 + 120.0 * (k % 2), 2.0 + 120.0 * k / n) for k in range(1, n)] + [("Z",)])
    s = Scene()
    s.fill(FILL_NON_ZERO, Affine.IDENTITY, WHITE, None, p)
    packed = resolve(s.encoding)
    parts = ((packed.layout.path_data_base - packed.layout.path_tag_base) * 4 + 31) // 32
    assert parts > 8192, parts
    case = Case("scan", lambda sc: None, EPS_FILL)
    _, st = gpu_flatten(renderer, oracle, case, packed)
    assert int(st["bump"]["lines"]) == n
    frame_parity(renderer, oracle, case, packed)


@pytest.mark.parametrize("d", [-2.0, -0.5, 0.5, 2.0])
def test_gpu_stripes_at_the_cull_edge(renderer, oracle, d):
    """Tile-row stripes skip tags whose control points, grown by R = 1 + (w/2) max(miter limit, 1.5) |M|_1, miss the
    stripe's rows. Two mitred V strokes sit on either side of the stripe boundary at y = 256, each turning at just under
    its miter limit, so that its miter tip reaches (w/2) x 3.9 from the vertex, to `d` px past the boundary (inside the
    other stripe for d > 0). The stripes must equal the whole frame: a cull radius below the true miter reach would drop
    the tips."""
    w, lim, ratio = 10.0, 4.0, 3.9
    half = np.arcsin(1.0 / ratio)  # half the V's inner angle: the miter is (w/2) / sin(half) long
    reach = 0.5 * w * ratio

    def build(s):
        for sg in (1, -1):  # apex below the boundary pointing up, and above it pointing down
            ya = 256.0 - sg * d + sg * reach
            legs = (40.0 * np.sin(half), sg * 40.0 * np.cos(half))
            pts = [(100.0 - legs[0], ya + legs[1]), (100.0, ya), (100.0 + legs[0], ya + legs[1])]
            stroke(polyline(pts), width=w, join=STYLE_JOIN_MITER, miter_limit=lim, start_cap=STYLE_CAP_BUTT,
                   end_cap=STYLE_CAP_BUTT)(s)
    case = Case(f"stripes-{d:g}", build, EPS_STRAIGHT, {"join:miter"}, w=200, h=512)
    packed, st = gpu_flatten(renderer, oracle, case)
    paths, _ = check_case(case, st["lines"])
    assert case.expect <= tags(paths)
    ln = st["lines"]
    tip0 = float(ln["p0"][ln["path_ix"] == 0][:, 1].min())
    tip1 = float(ln["p0"][ln["path_ix"] == 1][:, 1].max())
    assert abs(tip0 - (256.0 - d)) < 0.01 and abs(tip1 - (256.0 + d)) < 0.01, (tip0, tip1)
    frame_parity(renderer, oracle, case, packed)
    p = RenderParams(BLACK, case.w, case.h, AA_MSAA16)
    whole = renderer.render_to_texture(packed, p)
    parts = [renderer.render_to_texture(packed, p, bin_rows=(b, b + 1)) for b in range(2)]
    assert np.array_equal(np.concatenate(parts, axis=0), whole)
    if d > 1:  # the tips do put coverage into the other stripe
        assert whole[254:256, :, 0].any() and whole[256:258, :, 0].any()
