"""The dashes of vb_fragment_from_device_dashes (k_device_dashes.cu), stated in Python: each ring of two or more points is
dashed on its own by the host dasher (`shapes.dash`), and its dashes become sub-rings, closed or conditional, that the kernels
of k_device_paths.cu encode. `encode` applies the device's rules to those sub-rings, so that the tests can hold them against
`Scene.stroke` of the dashed paths."""
import numpy as np

from vello_b200.encoding import Encoding
from vello_b200.shapes import dash

from . import device_curves_ref as curves

CLOSED, CONDITIONAL = 1, 2  # VB_DP_RING_*


def ring_elements(pts, kinds, a, b, closed):
    """Ring a..b as the Scene sees it: M, its segments, Z when closed."""
    return curves.elements(pts, kinds, a, b) + ([("Z",)] if closed else [])


def shape(pts, kinds, roff, poff, i, closed):
    """The element list of path i in the dashes contract: its rings of two or more points."""
    els = []
    for k in range(int(poff[i]), int(poff[i + 1])):
        a, b = int(roff[k]), int(roff[k + 1])
        if b - a >= 2:
            els += ring_elements(pts, kinds, a, b, closed)
    return els


def subrings(els, first):
    """The sub-rings of one ring's dashed elements: [points (f32), kinds, flags]. M starts one; a piece appends its points
    after the first; Z flags the current one closed, and the one segment after it starts a conditional sub-ring at the ring's
    first point."""
    out, tail = [], False
    for e in els:
        k = e[0]
        if k == "M":
            assert not tail, els
            out.append([[(e[1], e[2])], [0], 0])
        elif k == "Z":
            assert out and not tail, els
            out[-1][2] |= CLOSED
            tail = True
        else:
            if tail:
                out.append([[first], [0], CONDITIONAL])
                tail = False
            assert out, els
            p = list(zip(e[1::2], e[2::2]))
            out[-1][0] += p
            out[-1][1] += [1] * (len(p) - 1) + [0]
    assert not tail, els
    return [[np.array(p, np.float32).reshape(-1, 2), k, f] for p, k, f in out]


def intermediate(pts, kinds, roff, poff, closed, pattern, offsets):
    """The intermediate the device writes: (points, kinds, ring offsets, path offsets over the sub-rings, flags)."""
    P, K, R, F, Q = [], [], [0], [], [0]
    for i in range(len(poff) - 1):
        for k in range(int(poff[i]), int(poff[i + 1])):
            a, b = int(roff[k]), int(roff[k + 1])
            if b - a < 2:
                continue
            els = dash(ring_elements(pts, kinds, a, b, closed), float(offsets[i]), pattern)
            for p, kk, f in subrings(els, (float(pts[a][0]), float(pts[a][1]))):
                P += [tuple(map(float, q)) for q in p]
                K += kk
                R.append(len(P))
                F.append(f)
        Q.append(len(R) - 1)
    return np.array(P, np.float32).reshape(-1, 2), np.array(K, np.uint8), R, Q, F


def keeps(p, k):
    """Whether a sub-ring keeps a segment: the encoder, fresh, encodes one."""
    e = Encoding()
    return e.encode_path_elements(curves.elements(p, k, 0, len(p)), False) > 0


def encode(mid):
    """(tag bytes, path-data words) of the intermediate under the device's rules: a closed sub-ring is M .. Z, others open; a
    conditional one is drawn only after a kept unconditional sub-ring of its path (the lowest such index, path_min)."""
    P, K, R, Q, F = mid
    e = Encoding()
    for i in range(len(Q) - 1):
        rings = range(Q[i], Q[i + 1])
        kept = [r for r in rings if not F[r] & CONDITIONAL and keeps(P[R[r]:R[r + 1]], K[R[r]:R[r + 1]])]
        lo = min(kept) if kept else None
        els = []
        for r in rings:
            if F[r] & CONDITIONAL and not (lo is not None and lo < r):
                continue
            els += curves.elements(P, K, R[r], R[r + 1]) + ([("Z",)] if F[r] & CLOSED else [])
        e.encode_path_elements(els, False)
    return list(e.path_tags), np.array(e.path_data, np.float32)


def host(pts, kinds, roff, poff, closed, pattern, offsets):
    """(tag bytes, path-data words) of Scene.stroke's dashes of each path."""
    e = Encoding()
    for i in range(len(poff) - 1):
        e.encode_path_elements(dash(shape(pts, kinds, roff, poff, i, closed), float(offsets[i]), pattern), False)
    return list(e.path_tags), np.array(e.path_data, np.float32)
