"""The decoupled look-back (vb_lookback, vb_device.cuh) under forced schedules, against a serial fold.

A look-back that meets an inclusive prefix at its nearest predecessor combines one value. Only when predecessors have
published an aggregate and not yet a prefix does it reduce whole 32-partition windows, and for a non-commutative monoid
(backdrop's segmented sum) in partition order: `vb_warp_reduce_rev` and the order of `Op::combine(window, excl)`. Which case
a frame meets depends on timing, so `vb_debug_lookback` runs the look-back alone and lets partition p wait delay_ns[p]
before it publishes: a delayed partition holds every later one at its aggregate. Every partition's exclusive prefix is then
compared word for word with a serial fold. Delays are at most a few hundred microseconds; a launch lasts milliseconds.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M32 = 0xFFFFFFFF
SUM1, SUM5, BACKDROP, AFFINE = 0, 1, 2, 3
WORDS = {SUM1: 1, SUM5: 5, BACKDROP: 3, AFFINE: 2}
OP_NAMES = {SUM1: "sum1", SUM5: "sum5", BACKDROP: "backdrop", AFFINE: "affine"}


def combine(op, a, b):
    """a (+) b, a the earlier operand, in Python integers."""
    if op in (SUM1, SUM5):
        return tuple((x + y) & M32 for x, y in zip(a, b))
    if op == BACKDROP:  # {crossings, row start seen, backdrop since the last row start}
        return ((a[0] + b[0]) & M32, a[1] | b[1], b[2] if b[1] else (a[2] + b[2]) & M32)
    ma, mb = a[0] + 1, b[0] + 1  # x -> m x + c stored as (m - 1, c); a applies first
    return ((mb * ma - 1) & M32, (mb * a[1] + b[1]) & M32)


def serial_excl(op, agg):
    acc = (0,) * WORDS[op]
    out = np.zeros_like(agg)
    for p in range(agg.shape[0]):
        out[p] = acc
        acc = combine(op, acc, tuple(int(v) for v in agg[p]))
    return out


def aggregates(op, n, rng):
    if op in (SUM1, SUM5):
        return rng.integers(0, 1 << 32, (n, WORDS[op]), dtype=np.uint64).astype(np.uint32)
    if op == AFFINE:
        return rng.integers(0, 1 << 32, (n, 2), dtype=np.uint64).astype(np.uint32)
    # backdrop: row starts rare, with runs of f = 0 far longer than a 32-partition window, and sums that wrap
    a = np.zeros((n, 3), np.uint32)
    a[:, 0] = rng.integers(0, 1 << 20, n)
    f = rng.random(n) < 0.05
    for lo, hi in ((3, 80), (200, 330), (600, 1700)):  # no row start in these partitions
        f[lo:hi] = False
    a[:, 1] = f
    a[:, 2] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    return a


def schedule(kind, n, rng):
    d = np.zeros(n, np.uint32)
    if kind == "p0-200us":
        d[0] = 200_000
    elif kind == "every-97th":
        d[::97] = 60_000
    elif kind == "random-10pct":
        pick = rng.random(n) < 0.1
        d[pick] = rng.integers(1_000, 150_000, int(pick.sum()))
    elif kind == "ramp-down":  # late tickets finish first
        d[:] = (np.arange(n, 0, -1, dtype=np.int64) * min(200_000 // n, 5_000)).astype(np.uint32)
    return d


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


@pytest.mark.parametrize("kind", ["none", "p0-200us", "every-97th", "random-10pct", "ramp-down"])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 64, 65, 1000, 5000])
@pytest.mark.parametrize("op", [SUM1, SUM5, BACKDROP, AFFINE], ids=lambda o: OP_NAMES[o])
def test_lookback_matches_serial_fold(renderer, op, n, kind):
    rng = np.random.default_rng(1000 * op + n + len(kind))
    agg = aggregates(op, n, rng)
    delay = schedule(kind, n, rng)
    assert int(delay.max()) <= renderer.LOOKBACK_MAX_DELAY_NS
    got = renderer.debug_lookback(op, agg, delay)
    want = serial_excl(op, agg)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, f"{OP_NAMES[op]} n={n} {kind}: {len(bad)} partitions differ, first {int(bad[0])}: got {got[bad[0]]}, want {want[bad[0]]}"


def test_affine_monoid_is_order_sensitive():
    """The test monoid catches a fold in the wrong order: swapping two neighbours changes the result."""
    a, b = (6, 11), (2, 5)
    assert combine(AFFINE, a, b) != combine(AFFINE, b, a)
    assert combine(AFFINE, (0, 0), a) == a == combine(AFFINE, a, (0, 0))


def test_lookback_rejects_bad_arguments(renderer):
    from vello_b200.renderer import VelloB200Error
    with pytest.raises(VelloB200Error):
        renderer.debug_lookback(SUM1, np.zeros((4, 1), np.uint32), np.array([0, renderer.LOOKBACK_MAX_DELAY_NS + 1, 0, 0]))
    with pytest.raises(VelloB200Error):
        renderer.debug_lookback(SUM1, np.zeros((0, 1), np.uint32))
