"""The upload diff's matching and draw-object records (tests/upload_diff_ref.py, the serial form of k_upload_diff.cu), on
synthetic key lists and packed scenes; no GPU needed. The matching must pair only equal keys, preserve order on both sides,
pair the whole common prefix and suffix, and pair the middle by position."""
import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.encoding import resolve

from . import upload_diff_ref as ref
from .test_i16_path import integral_scene, to_i16


def edit(keys, g, n_edits, alphabet):
    k = list(keys)
    for _ in range(n_edits):
        op = int(g.integers(0, 3))
        at = int(g.integers(0, len(k) + 1))
        if op == 0 or not k:
            k.insert(at, int(g.integers(0, alphabet)))
        elif op == 1:
            del k[min(at, len(k) - 1)]
        else:
            k[min(at, len(k) - 1)] = int(g.integers(0, alphabet))
    return k


def check(old, new):
    mp, unmatched = ref.match(old, new)
    pairs = [(int(i), j) for j, i in enumerate(mp) if i != ref.NONE]
    assert all(old[i] == new[j] for i, j in pairs), "a pair of unequal keys"
    olds = [i for i, _ in pairs]
    assert olds == sorted(olds) and len(set(olds)) == len(olds), "the matching does not preserve order"
    assert sorted(np.flatnonzero(~unmatched).tolist()) == olds
    m = min(len(old), len(new))
    p = next((k for k in range(m) if old[k] != new[k]), m)
    assert all(mp[k] == k for k in range(p)), "the common prefix is not paired"
    if len(old) != len(new):
        s = next((k for k in range(m - p) if old[-1 - k] != new[-1 - k]), m - p)
        assert all(mp[len(new) - 1 - k] == len(old) - 1 - k for k in range(s)), "the common suffix is not paired"
    else:
        assert all((mp[k] == k) == (old[k] == new[k]) for k in range(m)), "equal sizes: the pairs are the equal positions"
    return mp, unmatched


@pytest.mark.parametrize("seed", range(40))
def test_matching_on_random_edits(seed):
    g = np.random.default_rng(seed)
    n, alphabet = int(g.integers(0, 60)), int(g.integers(2, 40))
    old = [int(v) for v in g.integers(0, alphabet, n)]
    check(old, edit(old, g, int(g.integers(0, 6)), alphabet))


def test_matching_cases():
    a = list(range(10))
    mp, un = check(a, a)
    assert (mp == np.arange(10)).all() and not un.any()
    mp, un = check(a, [99] + a)  # inserted at the start: the suffix pairs everything
    assert mp[0] == ref.NONE and (mp[1:] == np.arange(10)).all() and not un.any()
    mp, un = check(a, a[:5] + a[6:])  # deleted in the middle
    assert un.tolist() == [i == 5 for i in range(10)]
    mp, un = check(a, a[:4] + [50, 51] + a[4:])  # inserted in the middle
    assert (mp == np.array(list(range(4)) + [ref.NONE] * 2 + list(range(4, 10)))).all()
    mp, un = check(a, a[:3] + [77] + a[4:])  # one replaced: the middle by position
    assert mp.tolist() == [0, 1, 2, ref.NONE] + list(range(4, 10)) and un.tolist() == [i == 3 for i in range(10)]
    check([], a)
    check(a, [])
    check([1, 1, 1], [1, 1])  # a suffix that would overlap the prefix is capped


def test_records_tile_the_streams():
    """Every draw object's tag range starts after the previous path's end tag and ends with its own; the path data ranges
    follow each other without a gap, f32 and i16 alike."""
    for packed in (resolve(scenes.tiger(256, 256).encoding), to_i16(resolve(integral_scene().encoding))):
        L = packed.layout
        rec = ref.records(packed.scene, L)
        tags = packed.scene[L.path_tag_base:L.path_data_base].view(np.uint8)
        assert rec[0][0] == 0 and rec[0][2] == 0
        for a, b in zip(rec, rec[1:]):
            assert b[0] == a[1] and b[2] == a[3]
        for r in rec:
            assert tags[r[1] - 1] & 0x10 and not (tags[r[0]:r[1] - 1] & 0x10).any()
        k = ref.keys(packed.scene, L, packed.ramps, packed.atlas)
        assert len(k) == L.n_draw_objects
        mp, un = ref.match(k, k)
        assert (mp == np.arange(len(k))).all() and not un.any()
