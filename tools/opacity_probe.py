"""Bound opacity (Renderer.bind_draw_opacity, vb_bind_draw_opacity) on the paris-like 30k scene at 4096^2 MSAA16, its paths
grouped into about 1,000 layers (blend layers and clip layers alternating) with an image after every 16th group. Prints, with
the card, its power limit and SM clock, frames/s and ms per frame of four routes:
  unbound   the scene as encoded
  bound_1   every row 1, rewritten on vb_stream before each frame (the graph must replay): clip layers stay clip layers
  bound_05  every row 0.5, rewritten likewise: every layer and image at half alpha, the clip layers drawn as blend layers
  host      the host route for the rows of 0.5: re-encoding the scene (Python encoder and resolve), uploading it and its frame,
            each timed alone, and their sum as the cost of one frame; and the pixels of the last bound frame against the
            re-encoded scene's (must be equal)
and the device time per frame of k_draw_data, which writes the frame's draw data with the bound words (torch.profiler, in a
run of its own).
With --out the result also goes to DIR/opacity_probe.json:
    python tools/opacity_probe.py [--steps 30] [--warmup 5] [--out DIR]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compose_probe import card  # noqa: E402
from points_probe import parity, timed  # noqa: E402
from visibility_probe import SIZE, paris_paths  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, COMPOSE_SRC_OVER, FILL_NON_ZERO, MIX_MULTIPLY, MIX_NORMAL, Image, Scene, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402
from vello_b200.shapes import Affine, Rect  # noqa: E402

GROUP = 30        # paths per layer: about 1,000 layers
IMAGE_EVERY = 16  # groups between images
IMG = np.random.default_rng(7).integers(0, 256, (64, 64, 4), dtype=np.uint8)


def encode(paths, bulk, alpha=None):
    """The grouped scene, every layer and image with `alpha` in place of its encoded one (None: as encoded). A clip layer with
    an alpha below 1 is encoded as push_layer(MIX_NORMAL, COMPOSE_SRC_OVER, alpha), as a bound frame draws it."""
    s = Scene()
    e = s.encoding
    g = np.random.default_rng(3)
    for i in range(0, len(paths), GROUP):
        j = i // GROUP
        x0, y0 = (float(v) for v in g.uniform(-SIZE / 4, SIZE / 2, 2))
        clip = Rect(x0, y0, x0 + 0.75 * SIZE, y0 + 0.75 * SIZE)
        if j % 2:
            if alpha is None or alpha >= 1:
                s.push_clip_layer(FILL_NON_ZERO, Affine.IDENTITY, clip)
            else:
                s.push_layer(FILL_NON_ZERO, MIX_NORMAL, COMPOSE_SRC_OVER, alpha, Affine.IDENTITY, clip)
        else:
            s.push_layer(FILL_NON_ZERO, MIX_MULTIPLY if j % 4 == 0 else MIX_NORMAL, COMPOSE_SRC_OVER, 0.9 if alpha is None else alpha,
                         Affine.IDENTITY, clip)
        for path in paths[i:i + GROUP]:
            for name, args in path:
                if name in bulk:
                    bulk[name](e, *args)
                else:
                    getattr(e, name)(*args)
        s.pop_layer()
        if j % IMAGE_EVERY == 0:
            x, y = (float(v) for v in g.uniform(0, SIZE - 512, 2))
            s.draw_image(Image(IMG, alpha=1.0 if alpha is None else alpha), Affine.translate(x, y) * Affine.scale(8.0))
    return s


def kernel_us(frame, steps, names):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            frame(s)
    torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for n in names:
            if e.key.startswith(n + "(") or e.key == n:
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[n] = round(us / max(e.count, 1), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    paths, bulk = paris_paths()
    full = resolve(encode(paths, bulk).encoding)
    n = full.layout.n_draw_objects
    n_layers = (len(paths) + GROUP - 1) // GROUP
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    res = {"card_before": card(),
           "scene": f"paris-like 30k in {n_layers} layers (half clip layers) with {(n_layers + IMAGE_EVERY - 1) // IMAGE_EVERY} images "
                    f"({n} draw objects) at {SIZE}^2 MSAA16"}
    r, ref = Renderer(), Renderer()
    r.upload(full)
    res["unbound"] = timed(a.steps, a.warmup, lambda s: r.render_resident(p))
    unbound_launches = r.render_resident(p).kernel_launches

    t = torch.empty(n, dtype=torch.float32, device="cuda")
    st = torch.cuda.ExternalStream(r.stream)
    r.bind_draw_opacity(t)
    for name, v in (("bound_1", 1.0), ("bound_05", 0.5)):
        rows = torch.full((2, n), v, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

        def bound(s, rows=rows):
            with torch.cuda.stream(st):
                t.copy_(rows[s % 2])
            r.render_resident(p)

        bound(0)
        caps = r.debug_graph_captures()
        res[name] = timed(a.steps, a.warmup, bound)
        res[name]["graph_replayed"] = r.debug_graph_captures() == caps
        res[name]["extra_launches"] = r.render_resident(p).kernel_launches - unbound_launches
    img = r.download_target(p)

    # the host route for the rows of 0.5
    t0 = time.perf_counter()
    host = resolve(encode(paths, bulk, 0.5).encoding)
    encode_ms = (time.perf_counter() - t0) * 1e3
    ups = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref.upload(host)
        torch.cuda.synchronize()
        ups.append((time.perf_counter() - t0) * 1e3)
    fr = timed(a.steps, a.warmup, lambda s: ref.render_resident(p))
    total = encode_ms + min(ups) + fr["ms_per_frame"]
    res["host"] = {"encode_resolve_ms": round(encode_ms, 1), "upload_ms": round(min(ups), 3), "frame": fr,
                   "ms_per_frame": round(total, 3), "fps": round(1e3 / total, 2)}
    res["parity"] = parity(img, ref.download_target(p))

    rows = torch.full((2, n), 0.5, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()

    def bound05(s):
        with torch.cuda.stream(st):
            t.copy_(rows[s % 2])
        r.render_resident(p)

    res["kernel_us"] = kernel_us(bound05, a.steps, ["k_draw_data"])
    for k in ("unbound", "bound_1", "bound_05", "host"):
        print(f"{k:9s} {res[k]['fps']:9.2f} frames/s {res[k]['ms_per_frame']:9.3f} ms/frame", flush=True)
    print(f"host route: encode+resolve {encode_ms:.0f} ms, upload {res['host']['upload_ms']:.3f} ms, frame "
          f"{fr['ms_per_frame']:.3f} ms; parity {res['parity']}; kernels {res['kernel_us']} us", flush=True)
    r.close()
    ref.close()
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "opacity_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
