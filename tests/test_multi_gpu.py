"""Real multi-device tests (need >= 2 GPUs: `python -m pytest tests/test_multi_gpu.py -m gpu`); skipped on a
single-GPU box. The single-GPU suite covers the same code with several renderers on device 0 (test_group_one_call_one_frame)."""
import ctypes as C

import numpy as np
import pytest

from vello_b200 import scenes
from vello_b200.config import AA_MSAA16, RenderParams
from vello_b200.encoding import BLACK, resolve

pytestmark = pytest.mark.gpu


def _n_devices():
    try:
        rt = C.CDLL("libcudart.so")
    except OSError:
        try:
            rt = C.CDLL("libcudart.so.12")
        except OSError:
            return 0
    n = C.c_int(0)
    return n.value if rt.cudaGetDeviceCount(C.byref(n)) == 0 else 0


@pytest.mark.parametrize("n", [2, 4, 8])
def test_group_across_devices(oracle, n):
    if _n_devices() < n:
        pytest.skip(f"needs {n} GPUs")
    from vello_b200.renderer import RendererGroup
    packed = resolve(scenes.paris_like(4000, 2048, seed=12).encoding)
    p = RenderParams(BLACK, 2048, 2048, AA_MSAA16)
    ref = oracle.render(packed, 2048, 2048, BLACK.premul_rgba8_u32(), AA_MSAA16)
    g = RendererGroup(list(range(n)))
    assert np.array_equal(g.render_to_texture(packed, p), ref)      # host destination: every device reads its stripe back
    g.upload(packed)
    for k in range(5):                                              # device frame on devices[0]: fine stores over NVLink
        g.render_resident(p)
        assert np.array_equal(g.frame_to_host(p), ref), k
    g.set_exchange(True)                                            # flatten sharded by tag range, lines exchanged over NVLink
    g.upload(packed)
    for k in range(5):
        g.render_resident(p)
        assert np.array_equal(g.frame_to_host(p), ref), ("exchange", k)
    assert np.array_equal(g.render_to_texture(packed, p), ref)
    g.close()
