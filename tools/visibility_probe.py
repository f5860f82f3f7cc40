"""Bound visibility (Renderer.bind_draw_visibility, vb_bind_draw_visibility) on the paris-like 30k scene at 4096^2 MSAA16.
For 100 %, 50 %, 10 % and 1 % of the draw objects shown (a seeded random choice), prints frames/s and ms per frame (host wall
time of --steps blocking frames after --warmup, each ending in a synchronise) of:
  bound   the whole scene installed, the flags bound (rewritten on vb_stream every frame, so the graph replays)
  full    the whole scene, unbound
  subset  the scene re-encoded with only the shown draw objects and uploaded (the frame alone is timed, not the upload)
and the pixels of the last bound frame against the subset's (they must be equal), with the card, its power limit and SM clock.
Hidden tags still pass the tag scan and flatten's tag threads, and draw, clip and binning still see every draw object, so a
bound frame is expected to sit between the subset's and the full scene's; this tool measures where, and nothing else. With
--out the result also goes to DIR/visibility_probe.json:
    python tools/visibility_probe.py [--steps 30] [--warmup 5] [--out DIR]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compose_probe import card  # noqa: E402
from points_probe import parity, timed  # noqa: E402
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, Scene, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402

SIZE = 4096
SHARES = (1.0, 0.5, 0.1, 0.01)


class _Recorder:
    """Stands in for a Scene's encoding while scenes.paris_like runs: records each path's encoder calls, which end with its
    colour, so that any subset of the paths can be encoded again in order."""

    def __init__(self):
        self.paths, self.cur = [], []

    def __getattr__(self, name):
        def call(*args):
            self.cur.append((name, args))
            if name == "encode_color":
                self.paths.append(self.cur)
                self.cur = []
            return True
        return call


def paris_paths():
    """The encoder calls of each draw object of scenes.paris_like(30000, SIZE), in order."""
    rec = _Recorder()
    bulk = {k: getattr(scenes, k) for k in ("_bulk_fill_polygon", "_bulk_stroke_polyline", "_bulk_fill_cubics")}
    real_scene = scenes.Scene

    class RecScene:
        encoding = rec

    try:
        scenes.Scene = RecScene
        for k in bulk:
            setattr(scenes, k, lambda e, *args, k=k: e.__getattr__(k)(*args))
        scenes.paris_like(30000, SIZE)
    finally:
        scenes.Scene = real_scene
        for k, f in bulk.items():
            setattr(scenes, k, f)
    return rec.paths, bulk


def encode(paths, bulk, keep):
    s = Scene()
    e = s.encoding
    for path, k in zip(paths, keep):
        if not k:
            continue
        for name, args in path:
            if name in bulk:
                bulk[name](e, *args)
            else:
                getattr(e, name)(*args)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    paths, bulk = paris_paths()
    n = len(paths)
    full = resolve(encode(paths, bulk, [True] * n).encoding)
    assert full.layout.n_draw_objects == n
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    res = {"card_before": card(), "scene": f"paris-like 30k ({n} draw objects) at {SIZE}^2 MSAA16", "shares": {}}
    r, ref = Renderer(), Renderer()
    r.upload(full)
    res["full"] = timed(a.steps, a.warmup, lambda s: r.render_resident(p))
    g = np.random.default_rng(1)
    st = torch.cuda.ExternalStream(r.stream)
    for share in SHARES:
        keep = g.permutation(n) < round(share * n)
        flags = torch.from_numpy(keep.astype(np.uint8)).cuda()
        t = torch.empty_like(flags)
        torch.cuda.synchronize()
        r.upload(full)
        r.bind_draw_visibility(t)

        def bound(s):
            with torch.cuda.stream(st):
                t.copy_(flags)
            r.render_resident(p)

        caps = r.debug_graph_captures()
        row = {"shown": int(keep.sum()), "bound": timed(a.steps, a.warmup, bound)}
        row["graph_replayed"] = r.debug_graph_captures() == caps + 1
        img = r.download_target(p)
        ref.upload(resolve(encode(paths, bulk, keep).encoding))
        row["subset"] = timed(a.steps, a.warmup, lambda s: ref.render_resident(p))
        row["parity"] = parity(img, ref.download_target(p))
        res["shares"][f"{share:.0%}"] = row
        print(f"{share:>5.0%} shown: bound {row['bound']['ms_per_frame']:.3f} ms  subset {row['subset']['ms_per_frame']:.3f} ms  "
              f"full {res['full']['ms_per_frame']:.3f} ms  parity {row['parity']}", flush=True)
    r.close()
    ref.close()
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "visibility_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
