import os, sys, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vello_b200 import scenes
from vello_b200.config import RenderParams
from vello_b200.encoding import BLACK, resolve
from vello_b200.renderer import RendererGroup
packed = resolve(scenes.paris_like(2500, 1024, seed=4).encoding)
p = RenderParams(BLACK, 1024, 1024, 2)
g = RendererGroup([0])
for k in range(3):
    img = g.render_to_texture(packed, p)
    print(k, img[..., 3].min(), img[..., 3].max(), len(np.unique(img.reshape(-1, 4), axis=0)), [ (int(s.failed), int(s.retries), int(s.lines)) for s in g.last_stats], g.stripes())
g.upload(packed)
g.render_resident(p)
f = g.frame_to_host(p)
print('resident', f[..., 3].min(), len(np.unique(f.reshape(-1, 4), axis=0)))
