"""Bound stroke widths (Renderer.bind_stroke_widths, vb_bind_stroke_widths) on the paris-like 30k scene at 4096^2 MSAA16, whose
stroked polylines (about 25 % of the draw objects) give thousands of strokes. Prints, with the card, its power limit and SM
clock:
  bound     ms per frame with every row rewritten on vb_stream before each frame (two row sets alternating, so every frame
            strokes with other widths; the graph must replay), and the unbound scene's frame for comparison
  host      the host route for the same widths: re-encoding the scene with them (Python encoder and resolve), uploading it, and
            its frame, each timed alone; and the pixels of the last bound frame against the re-encoded scene's (must be equal)
  damage    damage tracking on, 1 % of the strokes widened in each frame (another 1 % every frame): ms per frame and the tiles
            repainted, against the frame's tile count
  snapshot  the snapshot kernel k_stroke_widths's device time per frame (torch.profiler, in a run of its own)
With --out the result also goes to DIR/width_probe.json:
    python tools/width_probe.py [--steps 30] [--warmup 5] [--out DIR]"""
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
from vello_b200.encoding import BLACK, Scene, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402


def encode(paths, bulk, widths):
    """The scene of `paths` with stroke k's width taken from widths[k] where it is finite and > 0."""
    s = Scene()
    e = s.encoding
    for k, path in enumerate(paths):
        for name, args in path:
            if name in bulk:
                bulk[name](e, *args)
            elif name == "encode_stroke_style" and np.isfinite(widths[k]) and widths[k] > 0:
                st = args[0]
                e.encode_stroke_style(type(st)(**{**st.__dict__, "width": float(widths[k])}))
            else:
                getattr(e, name)(*args)
    return s


def snapshot_us(r, frame, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            frame(s)
    torch.cuda.synchronize()
    for e in prof.key_averages():
        if "k_stroke_widths" in e.key:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            return round(us / max(e.count, 1), 2)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    paths, bulk = paris_paths()
    n = len(paths)
    stroke = np.array([any(name == "encode_stroke_style" for name, _ in path) for path in paths])
    enc_w = np.array([next((args[0].width for name, args in path if name == "encode_stroke_style"), np.nan) for path in paths],
                     dtype=np.float32)
    full = resolve(encode(paths, bulk, np.full(n, np.nan)).encoding)
    assert full.layout.n_draw_objects == n
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    g = np.random.default_rng(1)
    res = {"card_before": card(), "scene": f"paris-like 30k ({n} draw objects, {int(stroke.sum())} strokes) at {SIZE}^2 MSAA16"}
    r, ref = Renderer(), Renderer()
    r.upload(full)
    res["unbound"] = timed(a.steps, a.warmup, lambda s: r.render_resident(p))
    unbound_launches = r.render_resident(p).kernel_launches

    # every row rewritten on the stream before each frame: the encoded widths scaled by 0.5 .. 2, two sets alternating
    sets = [np.where(stroke, enc_w * g.uniform(0.5, 2.0, n).astype(np.float32), np.float32(7.0)).astype(np.float32) for _ in range(2)]
    rows = torch.from_numpy(np.stack(sets)).cuda()
    t = torch.empty(n, dtype=torch.float32, device="cuda")
    t.copy_(rows[0])
    torch.cuda.synchronize()
    r.bind_stroke_widths(t)
    st = torch.cuda.ExternalStream(r.stream)

    def bound(s):
        with torch.cuda.stream(st):
            t.copy_(rows[s % 2])
        r.render_resident(p)

    bound(0)
    caps = r.debug_graph_captures()
    res["bound"] = timed(a.steps, a.warmup, bound)
    res["bound"]["graph_replayed"] = r.debug_graph_captures() == caps
    res["bound"]["extra_launches"] = r.render_resident(p).kernel_launches - unbound_launches
    last = (a.warmup + a.steps - 1) % 2
    with torch.cuda.stream(st):
        t.copy_(rows[last])
    r.render_resident(p)
    img = r.download_target(p)

    # the host route for the same widths
    t0 = time.perf_counter()
    host = resolve(encode(paths, bulk, sets[last]).encoding)
    encode_ms = (time.perf_counter() - t0) * 1e3
    ups = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref.upload(host)
        torch.cuda.synchronize()
        ups.append((time.perf_counter() - t0) * 1e3)
    res["host"] = {"encode_resolve_ms": round(encode_ms, 1), "upload_ms": round(min(ups), 3),
                   "frame": timed(a.steps, a.warmup, lambda s: ref.render_resident(p))}
    res["parity"] = parity(img, ref.download_target(p))
    print(f"bound {res['bound']['ms_per_frame']:.3f} ms/frame (unbound {res['unbound']['ms_per_frame']:.3f}); host route: "
          f"encode+resolve {encode_ms:.0f} ms, upload {res['host']['upload_ms']:.3f} ms, frame {res['host']['frame']['ms_per_frame']:.3f} ms; "
          f"parity {res['parity']}", flush=True)

    # damage tracking, 1 % of the strokes widened each frame
    ks = np.nonzero(stroke)[0]
    m = max(1, len(ks) // 100)
    base = np.full(n, np.nan, dtype=np.float32)
    wide = [base.copy() for _ in range(4)]
    for j in range(4):
        wide[j][g.choice(ks, m, replace=False)] = np.float32(12.0)
    wide_t = torch.from_numpy(np.stack(wide)).cuda()
    dst = torch.zeros((SIZE, SIZE, 4), dtype=torch.uint8, device="cuda")
    t.copy_(wide_t[0])
    torch.cuda.synchronize()
    r.set_damage_tracking(True)
    tiles = []

    def tracked(s):
        with torch.cuda.stream(st):
            t.copy_(wide_t[s % 4])
        r.render_resident(p, dst.data_ptr())
        if s >= a.warmup:
            tiles.append(int(r.last_damage().sum()))

    r.render_resident(p, dst.data_ptr())
    res["damage"] = timed(a.steps, a.warmup, tracked)
    n_tiles = ((SIZE + 15) // 16) ** 2
    res["damage"].update({"strokes_widened": m, "tiles_repainted_mean": round(float(np.mean(tiles)), 1), "tiles": n_tiles})
    r.set_damage_tracking(False)
    print(f"damage: {m} strokes widened per frame, {res['damage']['ms_per_frame']:.3f} ms/frame, "
          f"{res['damage']['tiles_repainted_mean']:.0f} of {n_tiles} tiles repainted (includes last_damage's read-back)", flush=True)

    res["snapshot_us"] = snapshot_us(r, bound, a.steps)
    print(f"k_stroke_widths: {res['snapshot_us']} us per frame", flush=True)
    r.close()
    ref.close()
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "width_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
