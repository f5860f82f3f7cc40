"""The blend edge cases of test_blend_ref.py on the GPU: all 16 mixes x 14 compose operators, layer alpha, clip layers,
luminance masks and the six-level chain across VB_BLEND_STACK_SPLIT.

Each case renders in area AA, MSAA8 and MSAA16 (each a separate k_fine instantiation) and is checked stage by stage
against the oracle (`compare_all`), pixel for pixel against the oracle's fine replayed on the GPU's buffers
(`assert_replay`), and against the float64 reference (test_blend_ref.check). The oracle keeps one blend stack without a
split, so the chain's levels 4 and 5, which the kernel keeps in blend_spill, are held to the reference here."""
import pytest

from vello_b200.config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams
from vello_b200.encoding import TRANSPARENT

from . import parity
from .test_blend_ref import CASES_GPU, H, W, check, packed_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def renderer():
    from vello_b200.renderer import Renderer
    r = Renderer()
    yield r
    r.close()


@pytest.mark.parametrize("aa", [AA_AREA, AA_MSAA8, AA_MSAA16])
@pytest.mark.parametrize("case", CASES_GPU, ids=[c.name for c in CASES_GPU])
def test_blend_edges(renderer, oracle, case, aa):
    packed = packed_scene(case)
    img = renderer.render_to_texture(packed, RenderParams(TRANSPARENT, W, H, aa))
    oracle.render(packed, W, H, 0, aa)  # compare_all reads the oracle's buffers of this scene
    parity.compare_all(renderer, oracle, packed.layout, W, H)
    parity.assert_replay(renderer, oracle, packed, img, W, H, aa, TRANSPARENT)
    check(case, img)
