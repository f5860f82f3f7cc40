"""The oracle's fine on installed buffers (`vbo_set_buffer` with ptcl / segments / info_bin_data / blend_spill, and
`parity.replay_fine`), and the MSAA resolve's byte arithmetic where a winding number does not fit in a biased byte.

The GPU parity tests replay the GPU's command lists in the oracle to compare area AA byte for byte; here the replay is
pinned on the CPU: fed the oracle's own buffers it must reproduce the oracle's own image, and it must refuse buffers
that reference past their end instead of reading or writing there."""
import numpy as np
import pytest

from oracle.vbo import DTYPES, Oracle
from vello_b200 import scenes
from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16
from vello_b200.encoding import BLACK, TRANSPARENT, Scene, resolve

from . import parity


class _OracleBuffers:
    """Serves an oracle context's buffers through the renderer's `download` interface."""

    def __init__(self, o):
        self.o = o

    def download(self, name, dtype):
        return self.o.buffer(name).view(np.uint8).view(dtype)


@pytest.mark.parametrize("name", ["deep_blend", "many_clips", "fill_types", "blend_grid", "brushes"])
@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
def test_replay_of_own_buffers_reproduces_image(name, aa):
    s, w, h = getattr(scenes, name)()
    packed = resolve(s.encoding)
    src, dst = Oracle(threads=4), Oracle(threads=4)
    want = src.render(packed, w, h, BLACK.premul_rgba8_u32(), aa)
    if name == "deep_blend":
        assert int(src.buffer("bump")["blend"][0]) > 0  # levels past the blend-stack split spill
    got = parity.replay_fine(_OracleBuffers(src), dst, packed, w, h, aa, BLACK)
    assert np.array_equal(got, want)


def test_replay_in_a_bin_row_window():
    s = scenes.paris_like(600, 1024, seed=3)
    packed = resolve(s.encoding)
    src, dst = Oracle(threads=4), Oracle(threads=4)
    for aa in (AA_AREA, AA_MSAA16):
        want = src.render(packed, 1024, 700, TRANSPARENT.premul_rgba8_u32(), aa, bin_rows=(1, 3))
        got = parity.replay_fine(_OracleBuffers(src), dst, packed, 1024, 700, aa, TRANSPARENT, window=(1, 3))
        assert np.array_equal(got, want)
        assert not got[:256].any() and got[256:700].any()


def test_replay_refuses_references_past_a_buffer():
    """A FILL whose segment slice, or a command list that runs past the installed ptcl, or a spill past the installed
    blend spill fails the run instead of reading or writing outside the buffer."""
    s, w, h = scenes.deep_blend()
    packed = resolve(s.encoding)
    src = Oracle()
    src.render(packed, w, h, BLACK.premul_rgba8_u32(), AA_AREA)
    ptcl, segs, info = src.buffer("ptcl"), src.buffer("segments"), src.buffer("info_bin_data")
    blend = int(src.buffer("bump")["blend"][0])
    assert blend > 0 and len(segs) > 0
    o = Oracle()

    def run(p, sg, n_spill):
        o.bind(packed, w, h, BLACK.premul_rgba8_u32(), AA_AREA)
        o.set_buffer("ptcl", p)
        o.set_buffer("segments", sg)
        o.set_buffer("info_bin_data", info)
        o.set_buffer("blend_spill", np.zeros(n_spill, np.uint32))
        return o.run("fine", "fine")

    run(ptcl, segs, blend)
    for p, sg, n in ((ptcl, segs[:-1], blend), (ptcl[: len(ptcl) - 300], segs, blend), (ptcl, segs, blend - 1)):
        with pytest.raises(AssertionError):
            run(p, sg, n)


# ---- the MSAA resolve of a nonzero fill: fine.wgsl:397-468 (msaa8) and :470-495 (msaa16), in plain Python -------------
M32 = 0xFFFFFFFF


def wgsl_row_winding(words, wind_y=0):
    """fine.wgsl:397-418 for one pixel row: its 4 sh_winding words (biased bytes, one per pixel, u32 carries included) ->
    t = ((packed_w >> 8i) + wind_y) & 0xff for its 16 pixels (:448)."""
    pw = []
    for w in words:
        w = (w + (((w - 0x808080) & M32) << 8)) & M32
        w = (w + (((w - 0x8080) & M32) << 16)) & M32
        pw.append(w)
    prefix = [(((w >> 24) - 0x80) * 0x1010101) & M32 for w in pw]
    t = []
    for k in range(4):
        p = (pw[k] + sum(prefix[:k])) & M32
        t += [((p >> (8 * i)) + wind_y) & 0xFF for i in range(4)]
    return t


def wgsl_resolve(backdrop, t, samples, msaa16):
    """fine.wgsl:448-468 / :470-495: the coverage of one pixel from its row winding byte `t`, the fill's backdrop and its
    sample words (2 for msaa8, 4 for msaa16)."""
    expected_zero = (t - backdrop) & M32  # (... & 0xffu) - u32(fill.backdrop), in u32
    if expected_zero >= 256:
        return 1.0
    ez = (expected_zero * 0x1010101) & M32
    if not msaa16:
        x0 = ez ^ samples[0]
        x0_2 = (x0 | (x0 * 2)) & M32
        x1 = ez ^ samples[1]
        x1_2 = x1 | (x1 >> 1)
        x2 = (x0_2 & 0xAAAAAAAA) | (x1_2 & 0x55555555)
        x4 = (x2 | (x2 * 4)) & M32
        x8 = (x4 | (x4 * 16)) & M32
        return bin(x8 & 0xC0C0C0C0).count("1") * 0.125
    x0 = ez ^ samples[0]
    x0_2 = (x0 | (x0 * 2)) & M32
    x1 = ez ^ samples[1]
    x1_2 = x1 | (x1 >> 1)
    x01 = (x0_2 & 0xAAAAAAAA) | (x1_2 & 0x55555555)
    x01_4 = (x01 | (x01 * 4)) & M32
    x2 = ez ^ samples[2]
    x2_2 = (x2 | (x2 * 2)) & M32
    x3 = ez ^ samples[3]
    x3_2 = x3 | (x3 >> 1)
    x23 = (x2_2 & 0xAAAAAAAA) | (x3_2 & 0x55555555)
    x23_4 = x23 | (x23 >> 2)
    x4 = (x01_4 & 0xCCCCCCCC) | (x23_4 & 0x33333333)
    x8 = (x4 | (x4 * 16)) & M32
    return bin(x8 & 0xF0F0F0F0).count("1") * 0.0625


def test_wgsl_resolve_formula_by_hand():
    """A few triples worked out by hand: a pixel is uncovered exactly when every sample byte equals expected_zero, and
    expected_zero out of a byte's range (a backdrop past what a biased byte holds) is full coverage."""
    untouched8, untouched16 = [0x80808080] * 2, [0x80808080] * 4
    assert wgsl_resolve(0, 0x80, untouched8, False) == 0.0
    assert wgsl_resolve(5, 0x85, untouched16, True) == 0.0
    assert wgsl_resolve(-128, 0x00, untouched8, False) == 0.0
    assert wgsl_resolve(127, 0xFF, untouched16, True) == 0.0
    assert wgsl_resolve(128, 0x00, untouched8, False) == 1.0   # expected_zero = -128 as u32
    assert wgsl_resolve(-129, 0xFF, untouched16, True) == 1.0  # expected_zero = 384
    assert wgsl_resolve(0, 0x81, untouched8, False) == 1.0
    # msaa8: three sample bytes hold expected_zero = 0x83 (zero winding), the other five are covered
    assert wgsl_resolve(3, 0x86, [0x83808083, 0x80808083], False) == 5 * 0.125
    # msaa16: expected_zero = 0x80; three sample bytes differ from it
    assert wgsl_resolve(-2, 0x7E, [0x80808080, 0x80807F80, 0x80808080, 0x7F807F80], True) == 3 * 0.0625


@pytest.mark.parametrize("aa", [AA_MSAA8, AA_MSAA16])
@pytest.mark.parametrize("backdrop,down,up", [(0, 0, 0), (0, 256, 0), (0, 0, 256), (1, 257, 0), (-127, 0, 127), (-128, 0, 128),
                                              (-128, 128, 0), (127, 127, 0), (128, 0, 128), (-129, 129, 0), (255, 0, 1),
                                              (-256, 300, 44), (300, 44, 0), (0, 200, 72)])
def test_oracle_resolve_follows_wgsl_byte_arithmetic(aa, backdrop, down, up):
    """One 16x16 tile, one FILL with the given backdrop and `down` + `up` vertical segments at x = 3.5, then an opaque
    COLOR over a transparent base: the pixels right of the segments sit at a winding of backdrop + down - up (in the sign
    convention of the resolve), beyond a byte's range for most rows of the table. Pixels off column 3 receive no sample
    mask, so their coverage is wgsl_resolve(backdrop, t, untouched samples) with t from wgsl_row_winding -- including
    where fine.wgsl's biased bytes wrap and the answer differs from the geometric one. The oracle must follow the WGSL."""
    msaa16 = aa == AA_MSAA16
    n = down + up
    segs = np.zeros(n, DTYPES["segments"])
    segs["p0"][:down] = (3.5, 0.0)
    segs["p1"][:down] = (3.5, 16.0)
    segs["p0"][down:] = (3.5, 16.0)
    segs["p1"][down:] = (3.5, 0.0)
    segs["y_edge"] = 1e9
    ptcl = np.zeros(64, np.uint32)
    # blend offset, FILL (n << 1 | nonzero, seg_ix 0, backdrop), COLOR opaque white, END
    ptcl[:8] = [0, 1, n << 1, 0, backdrop & M32, 5, 0xFFFFFFFF, 0]
    o = Oracle()
    o.bind(resolve(Scene().encoding), 16, 16, TRANSPARENT.premul_rgba8_u32(), aa)
    o.set_buffer("ptcl", ptcl)
    o.set_buffer("segments", segs)
    o.set_buffer("info_bin_data", np.zeros(4, np.uint32))
    o.set_buffer("blend_spill", np.zeros(0, np.uint32))
    alpha = o.run("fine", "fine")[..., 3]
    words = [0x80808080, (0x80808080 + down - up) & M32, 0x80808080, 0x80808080]  # the delta lands on pixel 4 of each row
    t = wgsl_row_winding(words)
    untouched = [0x80808080] * (4 if msaa16 else 2)
    want = np.array([np.floor(0.5 + 255.0 * wgsl_resolve(backdrop, t[x], untouched, msaa16)) for x in range(16)])
    cols = [x for x in range(16) if x != 3]
    for y in range(16):
        assert np.array_equal(alpha[y, cols], want[cols]), (y, alpha[y].tolist(), want.tolist())
    if (backdrop, down, up) == (0, 256, 0):
        # a winding of 256 reads as zero in pixel 4; its carry into the next byte makes pixels 5.. read as covered
        assert (alpha[:, 4] == 0).all() and (alpha[:, 5:] == 255).all()
