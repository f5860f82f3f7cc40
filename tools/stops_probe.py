"""Bound gradient stops (Renderer.bind_gradient_stops, vb_bind_gradient_stops) on 10,000 gradient-filled bars (a 100 x 100
grid of linear gradients of three stops each, every ramp distinct) at 4096^2 MSAA16. Prints the card, its power limit and SM
clock before and after, then frames/s and ms per frame (host wall time of --steps blocking frames after --warmup, each frame
ending in a synchronise) of:
  (a) resident     the scene resident and unbound, nothing changed (vb_render_resident)
  (b) bound        all 30,000 stop rows rewritten by one torch op on vb_stream, then the frame
  (c) reupload     the route without bound stops: the scene's stops replaced in its encoding on the host and the streams
                   installed again (vb_scene_upload_streams, which resolves and makes the ramps on the device), then the frame
  (d) bound_damage as (b), but the stops of 1 % of the gradients changed per frame and damage tracking on into a device
                   destination; also the mean damaged tile count per frame
and the device time of one k_bound_ramps and one k_draw_data from torch.profiler (a separate pass). (b) and (c) check one frame's pixels against
each other. With --out the result also goes to DIR/stops_probe.json:
    python tools/stops_probe.py [--steps 50] [--warmup 5] [--out DIR]"""
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
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Gradient, Scene  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402
from vello_b200.shapes import Affine, Rect  # noqa: E402

SIZE, GRID = 4096, 100


def bars(g):
    """GRID x GRID bars, each a linear gradient of three seeded stops."""
    s = Scene()
    cell = SIZE / GRID
    for i in range(GRID * GRID):
        x, y = (i % GRID) * cell, (i // GRID) * cell
        c = g.uniform(0, 1, (3, 4)).astype(np.float32)
        c[:, 3] = 1.0
        stops = [(o, Color(*map(float, c[k]))) for k, o in enumerate((0.0, float(np.float32(g.uniform(0.2, 0.8))), 1.0))]
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, Gradient.linear((x, y), (x + cell, y), stops), None,
               Rect(x + 2, y + 2, x + cell - 2, y + cell - 2))
    return s


def timed(steps, warmup, frame):
    for s in range(warmup):
        frame(s)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(steps):
        frame(warmup + s)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    return {"fps": round(1e3 / ms, 1), "ms_per_frame": round(ms, 4)}


def kernel_us(r, t, all_rows, p, steps):
    from torch.profiler import ProfilerActivity, profile
    st = torch.cuda.ExternalStream(r.stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            with torch.cuda.stream(st):
                t.copy_(all_rows[s % all_rows.shape[0]])
            r.render_resident(p)
    out = {}
    for e in prof.key_averages():
        for name in ("k_bound_ramps", "k_draw_data"):
            if e.key.startswith(name + "("):
                us = getattr(e, "device_time_total", None)
                if us is None:
                    us = getattr(e, "cuda_time_total", 0.0)
                out[name] = round(us / max(e.count, 1), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card_before": card()}
    g = np.random.default_rng(1)
    scene = bars(g)
    n = scene.n_stops
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    base = np.array([(o, c.r, c.g, c.b, c.a) for q in scene.encoding.ramp_patches for o, c in q["stops"]], dtype=np.float32)
    K = 8  # distinct stop sets, cycled: colours recoloured, middle offsets slid
    rows_h = np.repeat(base[None], K, 0)
    rows_h[:, :, 1:4] = g.uniform(0, 1, (K, n, 3)).astype(np.float32)
    rows_h[:, 1::3, 0] = g.uniform(0.1, 0.9, (K, n // 3)).astype(np.float32)
    all_rows = torch.from_numpy(rows_h).cuda()
    res["workload"] = f"{GRID * GRID} gradient bars {SIZE}x{SIZE} MSAA16, {n} stops"

    r = Renderer()
    r.upload_scene(scene)
    res["a_resident"] = timed(args.steps, args.warmup, lambda s: r.render_resident(p))
    res["a_resident"]["launches"] = int(r.render_resident(p).kernel_launches)

    t = torch.empty((n, 5), dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_gradient_stops(t)
    st = torch.cuda.ExternalStream(r.stream)

    def bound(s):
        with torch.cuda.stream(st):
            t.copy_(all_rows[s % K])
        r.render_resident(p)

    res["b_bound"] = timed(args.steps, args.warmup, bound)
    res["b_bound"]["launches"] = int(r.render_resident(p).kernel_launches)
    caps = r.debug_graph_captures()
    bound(3)
    img_b = r.download_target(p)
    res["b_bound"]["graph_captures_during_run"] = int(r.debug_graph_captures() - caps)

    rc = Renderer()
    work = bars(np.random.default_rng(1))
    sets = [[[(float(rows_h[k, 3 * i + j, 0]), Color(*map(float, rows_h[k, 3 * i + j, 1:]))) for j in range(3)]
             for i in range(GRID * GRID)] for k in range(K)]

    def reupload(s):
        for q, stops in zip(work.encoding.ramp_patches, sets[s % K]):  # the host edit ...
            q["stops"] = stops
        rc.upload_scene(work)                                          # ... and the installation
        rc.render_resident(p)

    res["c_reupload"] = timed(max(args.steps // 5, 3), 2, reupload)
    reupload(3)
    d = np.abs(rc.download_target(p).astype(np.int32) - img_b.astype(np.int32))
    res["b_vs_c_pixels"] = {"max_diff": int(d.max()), "differing": int((d > 0).sum())}
    rc.close()

    dst = torch.zeros((SIZE, SIZE, 4), dtype=torch.uint8, device="cuda")
    r.set_damage_tracking(True)
    m = max(1, (GRID * GRID) // 100)
    picks = []
    for _ in range(K):
        gr = g.choice(GRID * GRID, m, replace=False)
        picks.append(np.concatenate([3 * gr, 3 * gr + 1, 3 * gr + 2]))
    picks = torch.from_numpy(np.stack(picks)).cuda()

    def bound_damage(s):
        with torch.cuda.stream(st):
            # a stop set other than the one these rows got a cycle ago, so that every picked gradient changes
            t[picks[s % K]] = all_rows[(s + 1 + s // K) % K][picks[s % K]]
        r.render_resident(p, dst.data_ptr())

    res["d_bound_damage"] = timed(args.steps, args.warmup, bound_damage)
    damaged = []
    for s in range(K):  # the damage of further frames, outside the timed ones (vb_last_damage synchronises)
        bound_damage(s)
        damaged.append(int(r.last_damage().sum()))
    tiles = ((SIZE + 15) // 16) ** 2
    res["d_bound_damage"].update(gradients_changed=m, damaged_tiles_mean=round(float(np.mean(damaged)), 1), tiles=tiles)
    r.set_damage_tracking(False)
    res["kernel_us"] = kernel_us(r, t, all_rows, p, 20)
    r.close()
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stops_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
