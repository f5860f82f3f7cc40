"""The instance matching of vb_recompose (vb_diff.h), through the test-only vb_debug_match_instances on plain integer keys (no
GPU needed). A recompose's damage is sound for every order-preserving matching between equal keys and smallest for a longest
one, so: the matching is always order-preserving and between equal keys; with at most VB_RECOMPOSE_MAX_EDITS insertions and
deletions it pairs a longest common subsequence (checked against an O(NM) dynamic programme); past that, the common prefix and
suffix and then the middle by position."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.renderer import load_library

MAX_EDITS = 32  # VB_RECOMPOSE_MAX_EDITS (include/vello_b200.h)
NONE = 0xFFFFFFFF


def match(old, new):
    lib = load_library()
    a = np.ascontiguousarray(old, dtype=np.uint32)
    b = np.ascontiguousarray(new, dtype=np.uint32)
    m = np.zeros(max(len(b), 1), dtype=np.uint32)
    edits = lib.vb_debug_match_instances(a.ctypes.data if a.size else None, len(a), b.ctypes.data if b.size else None, len(b),
                                         m.ctypes.data)
    return m[:len(b)], int(edits)


def lcs(a, b):
    n, m = len(a), len(b)
    t = np.zeros((n + 1, m + 1), dtype=np.int32)
    for i in range(n - 1, -1, -1):
        eq = b == a[i]
        nxt = t[i + 1]
        row = t[i]
        for j in range(m - 1, -1, -1):
            row[j] = nxt[j + 1] + 1 if eq[j] else max(nxt[j], row[j + 1])
    return int(t[0, 0])


def check_sound(old, new, m):
    pairs = [(int(i), j) for j, i in enumerate(m) if i != NONE]
    for i, j in pairs:
        assert i < len(old) and old[i] == new[j], f"new {j} paired with old {i}: keys {old[i] if i < len(old) else '?'} != {new[j]}"
    olds = [i for i, _ in pairs]
    assert olds == sorted(olds) and len(set(olds)) == len(olds), "the matching does not preserve order"
    return len(pairs)


def edit_script(g, old, n_edits, n_keys):
    """old with n_edits random edits: replace, insert, delete, move to the front or back, change a key in place."""
    new = list(old)
    for _ in range(n_edits):
        op = g.integers(0, 6)
        if op == 0 and new:
            new[g.integers(0, len(new))] = int(g.integers(0, n_keys))
        elif op == 1:
            new.insert(int(g.integers(0, len(new) + 1)), int(g.integers(0, n_keys)))
        elif op == 2 and new:
            del new[g.integers(0, len(new))]
        elif op == 3 and new:
            new.insert(0, new.pop(g.integers(0, len(new))))
        elif op == 4 and new:
            new.append(new.pop(g.integers(0, len(new))))
        elif new:
            new[g.integers(0, len(new))] = 1_000_000 + int(g.integers(0, 1000))
    return new


@pytest.mark.parametrize("seed", range(12))
def test_matching_is_a_longest_common_subsequence_within_the_edit_bound(seed):
    g = np.random.default_rng(seed)
    n_keys = [3, 40, 10_000][seed % 3]  # many repeated keys, some, all distinct
    for _ in range(25):
        old = [int(v) for v in g.integers(0, n_keys, int(g.integers(0, 120)))]
        new = edit_script(g, old, int(g.integers(0, 12)), n_keys)
        m, edits = match(old, new)
        got = check_sound(old, new, m)
        best = lcs(np.array(old, dtype=np.int64), np.array(new, dtype=np.int64))
        d = len(old) + len(new) - 2 * best
        if d <= MAX_EDITS:
            assert got == best, f"{got} pairs, the longest common subsequence has {best} (edit distance {d})"
            assert edits <= d
        else:
            assert edits == MAX_EDITS + 1


def positional(old, new):
    """The fallback's pairs: the common prefix and suffix, then the middle by position where the keys are equal."""
    pre = 0
    while pre < min(len(old), len(new)) and old[pre] == new[pre]:
        pre += 1
    suf = 0
    while suf < min(len(old), len(new)) - pre and old[-1 - suf] == new[-1 - suf]:
        suf += 1
    mid = sum(1 for x in range(min(len(old), len(new)) - pre - suf) if old[pre + x] == new[pre + x])
    return pre + suf + mid


@pytest.mark.parametrize("case", ["reverse", "shuffle", "many_inserts"])
def test_past_the_edit_bound_pairs_by_position(case):
    g = np.random.default_rng(3)
    old = list(range(5000))
    if case == "reverse":
        new = old[::-1]
    elif case == "shuffle":
        new = old[:100] + list(g.permutation(old[100:4900])) + old[4900:]
    else:  # inserts spread over the list: most of the middle stays in place by position only where it did not shift
        new = list(old)
        for k in sorted(g.choice(5000, 40, replace=False), reverse=True):
            new.insert(int(k), 100_000 + int(k))
    new = [int(v) for v in new]
    m, edits = match(old, new)
    assert edits == MAX_EDITS + 1
    assert check_sound(old, new, m) == positional(old, new)


def test_edges():
    for old, new, pairs in [([], [], 0), ([], [1, 2], 0), ([1, 2], [], 0), ([1, 2, 3], [1, 2, 3], 3), ([1, 2, 3], [3, 2, 1], 1),
                            ([5] * 40, [5] * 41, 40), ([1, 2, 3, 4], [1, 9, 3, 4], 3)]:
        m, edits = match(old, new)
        assert check_sound(old, new, m) == pairs, (old, new)
    # one edit among 10,000: a raise (move to the end) and an insertion at the front
    old = list(range(10_000))
    m, edits = match(old, old[:17] + old[18:] + [17])
    assert edits == 2 and check_sound(old, old[:17] + old[18:] + [17], m) == 9_999
    m, edits = match(old, [123_456] + old)
    assert edits == 1 and check_sound(old, [123_456] + old, m) == 10_000
    # exactly at the bound, and one past it
    for k, want in [(MAX_EDITS, MAX_EDITS), (MAX_EDITS + 1, MAX_EDITS + 1)]:
        new = [100_000 + i for i in range(k)] + old
        m, edits = match(old, new)
        assert edits == want
        assert check_sound(old, new, m) == (10_000 if k <= MAX_EDITS else positional(old, new))
