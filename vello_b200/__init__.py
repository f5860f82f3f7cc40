"""vello_b200 -- a Hopper-native (H100, sm_90a) drop-in for the GPU compute path behind
`vello::Renderer::render_to_texture` (see DESIGN.md and include/vello_b200.h)."""
from .config import AA_AREA, AA_MSAA8, AA_MSAA16, RenderParams  # noqa: F401
from .encoding import Scene, Packed, resolve  # noqa: F401

# The native scene front end (NativeScene, NativePath) lives in vello_b200.scene_native and the GPU renderer in
# vello_b200.renderer; both load libvello_b200.so on first use and are not imported here so that the pure-Python encoder
# stays usable where the library has not been built.
