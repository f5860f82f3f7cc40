"""The device resolve (vb_scene_upload_streams) refuses a scene whose packed layout passes 32-bit word offsets, as vb_compose
does: before it reads or copies a stream, and leaving the scene it had in place."""
import ctypes as C

import numpy as np
import pytest

from vello_b200.config import AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color
from vello_b200.shapes import Affine, Circle

pytestmark = pytest.mark.gpu

VB_E_INVALID = -1


def test_upload_streams_past_32_bit_word_offsets():
    from vello_b200.renderer import Renderer, _EncodingStreams
    from vello_b200.scene_native import NativeScene
    r = Renderer()
    try:
        s = NativeScene()
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color.from_rgba8(200, 60, 30), None, Circle(40.0, 30.0, 20.0))
        s.upload_device(r)
        p = RenderParams(BLACK, 64, 64, AA_MSAA16)
        r.render_resident(p)
        before = r.download_target(p)
        # 6 words per transform: 0x2AAAAAAB transforms pass 2^32 words. The buffer holds one transform; it is never read.
        xf = np.zeros(6, dtype=np.float32)
        e = _EncodingStreams()
        e.transforms = xf.ctypes.data
        e.n_transforms = 0x2AAAAAAB
        assert r.lib.vb_scene_upload_streams(r.handle, C.byref(e), None) == VB_E_INVALID
        assert b"32-bit word offsets" in r.lib.vb_last_error(r.handle)
        r.render_resident(p)
        assert np.array_equal(r.download_target(p), before)
        assert before.any()
    finally:
        r.close()
