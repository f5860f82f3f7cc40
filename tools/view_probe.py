"""Views of a resident scene (Renderer.set_view) against the host route, on the headline scene (paris-like, 30k paths,
4096^2, MSAA16). For each view: the frame time of the resident scene under the view, bump.lines, per-stage times (timing on,
a separate renderer), and the host route for the same view -- the packed scene's transform words mapped on the host
(encoding.viewed), then vb_scene_upload + vb_render_resident, timed on the host around both. Prints the card, its power
limit and SM clock first. frame_ms is device time (events around the frame); host_route_ms is wall time of the mapping,
the upload and the blocking render. With --out, the rows also go to DIR/view_probe.jsonl:
    python tools/view_probe.py [--steps 20] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, resolve, viewed  # noqa: E402
from vello_b200.renderer import Renderer, RendererOptions  # noqa: E402
from vello_b200.shapes import Affine  # noqa: E402

SIZE = 4096


def zoom(k, rot=0.0):
    """Zoom by k about the frame's centre."""
    c = SIZE / 2
    return Affine.translate(c, c) * Affine.rotate(rot) * Affine.scale(k) * Affine.translate(-c, -c)


VIEWS = {  # "none": no view at all (the unviewed pipeline, no culling)
    "none": None,
    "identity": Affine(),
    "pan_fractional": Affine.translate(137.25, -61.5),
    "zoom2": zoom(2.0),
    "zoom4": zoom(4.0),
    "zoom16_rot": zoom(16.0, 0.35),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def frame_ms(r, p, steps):
    """Median device time of `steps` resident frames (events around each frame, vb_last_frame_ms)."""
    r.render_resident(p)
    ms = []
    for _ in range(steps):
        r.render_resident(p)
        ms.append(r.lib.vb_last_frame_ms(r.handle))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("view_probe: no CUDA device")
    print("card (name, power limit, SM clock, max SM clock):", card(), flush=True)
    packed = resolve(scenes.paris_like(30000, SIZE, seed=30000).encoding)
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    r = Renderer()
    r.upload(packed)
    rt = Renderer(RendererOptions(timing=True))
    rt.upload(packed)
    host = Renderer()
    rows = []
    for name, v in VIEWS.items():
        r.set_view(v)
        ms = frame_ms(r, p, a.steps)
        lines = int(r.last_stats.lines)
        img = r.download_target(p)
        rt.set_view(v)
        rt.render_resident(p)
        stage = {}
        for _ in range(5):
            d = rt.render_resident(p).as_dict()
            for s, t in d["stage_ms"].items():
                stage[s] = stage.get(s, 0.0) + t / 5
        hv = packed if v is None else viewed(packed, v)
        host.upload(hv)
        host.render_resident(p)
        hms = []
        for _ in range(max(3, a.steps // 4)):
            t0 = time.perf_counter()
            host.upload(packed if v is None else viewed(packed, v))  # map the transform words, upload, render
            host.render_resident(p)
            hms.append((time.perf_counter() - t0) * 1e3)
        same = bool(np.array_equal(img, host.download_target(p)))
        row = dict(view=name, frame_ms=round(ms, 3), lines=lines, host_lines=int(host.last_stats.lines),
                   stage_ms={s: round(t, 3) for s, t in stage.items()}, host_route_ms=round(float(np.median(hms)), 3),
                   pixels_equal_host=same)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "view_probe.jsonl"), "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for row in rows:
                f.write(json.dumps(row) + "\n")
    for x in (r, rt, host):
        x.close()


if __name__ == "__main__":
    main()
