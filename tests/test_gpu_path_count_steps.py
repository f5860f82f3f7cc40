"""k_path_count's crossing phase against the oracle's path_count, at the edges of its 768-line steps.

On a frame of enough lines to give every resident CTA a step, k_path_count takes its lines 768 at a time, three 256-line
segments, and reserves the step's records with one atomic (otherwise 256 at a time, as test_gpu_path_count_expand.py
checks). Thread t sets up lines t, 256 + t and 512 + t; one scan of the three segments lays the step's crossings end to
end in line order, and the threads take them in strides of 256 as before. So the edges are: a step with each one of its
segments empty and the others not; one with no crossings at all (no reservation); and a last step that ends inside its
first segment. The edges of the 256-item strides are in test_gpu_path_count_expand.py.

Checks, as test_gpu_path_count_expand.py does, after path_count alone on the GPU and on the oracle: the tiles' backdrop
deltas and crossing counts are equal, the records are the same multiset, and every tile's slots are 0..count-1.
"""
import numpy as np
import pytest

from vello_b200.encoding import Scene, resolve

from .test_gpu_path_count_expand import _block_path, _crossings, _fill, _zigzag, assert_slots, gpu_after_path_count
from .test_gpu_path_count_expand import oracle_after_path_count
from .test_gpu_path_count_expand import renderer  # noqa: F401  (fixture)

SEG = 256     # lines per segment: one per thread of a k_path_count CTA
LPT = 3       # segments per step (PC_LPT in k_path_count.cu)
STEP = LPT * SEG
W = H = 128


def _flat(y):
    """256 lines along the tile edge y, back and forth: none of them crosses a tile."""
    return [(3.0 + 0.25 * k, y) for k in range(SEG)]


def scene(reps):
    """`reps` times: for each segment u, a step whose segment u has no crossings and whose others have 300 and 257; then a
    step with no crossings at all. Then 100 lines, so that the frame ends inside a step's first segment."""
    s = Scene()
    for _ in range(reps):
        for u in range(LPT):
            totals = iter((300, 257, 300))
            for v in range(LPT):
                if v == u:
                    _fill(s, _flat(32.0 + 16.0 * v), v)
                else:
                    _fill(s, _block_path(v % 2, next(totals)), v)
        for v in range(LPT):
            _fill(s, _flat(48.0 + 16.0 * v), v)
    _fill(s, _zigzag(100), 6)
    return s


def reps_for_steps():
    """Repetitions that give the frame enough lines for 768-line steps on this GPU (k_path_count takes 256 at a time when
    fewer than SMs x 6 x 768 lines would leave CTAs idle)."""
    import torch
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return -(-sms * 6 * STEP // ((LPT + 1) * STEP)) + 1


def reached(lines, seg_counts):
    tags = set()
    per_line = np.bincount(seg_counts["line_ix"].astype(np.int64), minlength=len(lines))
    segs = np.bincount(np.arange(len(lines)) // SEG, weights=per_line).astype(np.int64)
    segs = np.append(segs, [0] * (-len(segs) % LPT)).reshape(-1, LPT)
    for step in segs:
        if step.sum() == 0:
            tags.add("step-empty")
        else:
            tags |= {f"segment-{u}-empty" for u in range(LPT) if step[u] == 0}
    if len(lines) % STEP != 0:
        tags.add("partial-last-step")
    return tags


EXPECT = {f"segment-{u}-empty" for u in range(LPT)} | {"step-empty", "partial-last-step"}


def test_oracle_reaches_step_edges(oracle):
    o = oracle_after_path_count(oracle, resolve(scene(2).encoding), W, H)
    assert int(o["bump"]["failed"]) == 0
    got = reached(o["lines"], o["seg_counts"])
    assert EXPECT <= got, sorted(EXPECT - got)


@pytest.mark.gpu
def test_gpu_path_count_steps_match_oracle(renderer, oracle):  # noqa: F811
    import torch
    packed = resolve(scene(reps_for_steps()).encoding)
    o = oracle_after_path_count(oracle, packed, W, H)
    g = gpu_after_path_count(renderer, packed, W, H)
    assert int(g["bump"]["failed"]) == 0
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    assert len(g["lines"]) >= sms * 6 * STEP, "too few lines for whole steps"
    assert g["lines"].tobytes() == o["lines"].tobytes()
    assert np.array_equal(g["tiles"]["backdrop"], o["tiles"]["backdrop"]), "backdrop deltas differ"
    assert np.array_equal(g["tiles"]["segment_count_or_ix"], o["tiles"]["segment_count_or_ix"]), "crossing counts differ"
    assert int(g["bump"]["seg_counts"]) == int(o["bump"]["seg_counts"])
    assert np.array_equal(_crossings(g["seg_counts"]), _crossings(o["seg_counts"])), "the (line, i, outside) multiset differs"
    assert assert_slots(g["lines"], g["paths"], g["seg_counts"], g["tiles"]["segment_count_or_ix"]) > 0
    assert EXPECT <= reached(g["lines"], g["seg_counts"])
