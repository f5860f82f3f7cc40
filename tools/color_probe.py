"""Bound draw colours (Renderer.bind_draw_colors, vb_bind_draw_colors) on the headline workload, paris-like 30k at 4096^2
MSAA16, with every draw object recoloured every frame. Prints the card, its power limit and SM clock before and after, then
frames/s and ms per frame (host wall time of --steps blocking frames after --warmup, each frame ending in a synchronise) of:
  (a) resident     the scene resident and unbound, nothing changed (vb_render_resident)
  (b) bound        all 30k rows rewritten by one torch op on vb_stream, then the frame
  (c) reupload     the route without bound colours: the packed scene's colour words patched on the host (numpy) and the scene
                   uploaded again (vb_scene_upload), then the frame
  (d) bound_damage as (b), but 1 % of the rows changed per frame and damage tracking on into a device destination; also the
                   mean damaged tile count per frame
and the device time of one k_draw_data from torch.profiler (a separate pass). (b) and (c) check one frame's pixels against
each other. With --out the result also goes to DIR/color_probe.json:
    python tools/color_probe.py [--steps 50] [--warmup 5] [--out DIR]"""
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
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402

COLOR_TAGS = (0x44, 0x2D4)  # FILL_COLOR, BLURRED_ROUNDED_RECT


def premul_words(rows):
    """The encoder's premultiply().to_rgba8().to_u32() of float32 (n, 4) rows (the host route's conversion)."""
    a = rows[:, 3]
    p = np.stack([rows[:, 0] * a, rows[:, 1] * a, rows[:, 2] * a, a], 1)
    v = np.clip(np.floor(p * np.float32(255.0) + np.float32(0.5)), 0, 255).astype(np.uint32)
    return v[:, 0] | v[:, 1] << 8 | v[:, 2] << 16 | v[:, 3] << 24


def colour_slots(packed):
    """The scene words of every draw object's colour, and the draw objects they belong to."""
    L = packed.layout
    tags = packed.scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects]
    off = np.concatenate([[0], np.cumsum((tags >> 2) & 7)[:-1]]).astype(np.int64)
    solid = np.isin(tags, COLOR_TAGS)
    return L.draw_data_base + off[solid], np.nonzero(solid)[0]


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
    for e in prof.key_averages():
        if e.key.startswith("k_draw_data("):
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = getattr(e, "cuda_time_total", 0.0)
            return round(us / max(e.count, 1), 2)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card_before": card()}
    size, n_paths = 4096, 30000
    packed = resolve(scenes.paris_like(n_paths, size, 30000).encoding)
    n = packed.layout.n_draw_objects
    p = RenderParams(BLACK, size, size, AA_MSAA16)
    K = 8  # distinct colour sets, cycled
    g = np.random.default_rng(1)
    rows_h = g.uniform(0, 1, (K, n, 4)).astype(np.float32)
    rows_h[:, :, 3] = np.where(g.random((K, n)) < 0.2, g.uniform(0.25, 0.9, (K, n)), 1.0).astype(np.float32)
    all_rows = torch.from_numpy(rows_h).cuda()
    slots, draws = colour_slots(packed)
    res["workload"] = f"paris-like-30k {size}x{size} MSAA16, {n} draw objects, {len(draws)} with one colour"

    r = Renderer()
    r.upload(packed)
    res["a_resident"] = timed(args.steps, args.warmup, lambda s: r.render_resident(p))
    res["a_resident"]["launches"] = int(r.render_resident(p).kernel_launches)

    t = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    r.bind_draw_colors(t)
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
    scene = packed.scene.copy()
    words = [premul_words(rows_h[k][draws]) for k in range(K)]
    work = type(packed)(scene, packed.layout, packed.ramps, packed.atlas)

    def reupload(s):
        scene[slots] = words[s % K]  # the host patch ...
        rc.upload(work)              # ... and the upload
        rc.render_resident(p)

    res["c_reupload"] = timed(args.steps, args.warmup, reupload)
    res["c_reupload"]["scene_mib_per_frame"] = round(packed.scene.nbytes / 2**20, 2)
    reupload(3)
    d = np.abs(rc.download_target(p).astype(np.int32) - img_b.astype(np.int32))
    res["b_vs_c_pixels"] = {"max_diff": int(d.max()), "differing": int((d > 0).sum())}
    rc.close()

    dst = torch.zeros((size, size, 4), dtype=torch.uint8, device="cuda")
    r.set_damage_tracking(True)
    m = max(1, n // 100)
    picks = torch.from_numpy(np.stack([g.choice(n, m, replace=False) for _ in range(K)])).cuda()

    def bound_damage(s):
        with torch.cuda.stream(st):
            t[picks[s % K]] = all_rows[(s + 1) % K][picks[s % K]]
        r.render_resident(p, dst.data_ptr())

    res["d_bound_damage"] = timed(args.steps, args.warmup, bound_damage)
    damaged = []
    for s in range(K):  # the damage of further frames, outside the timed ones (vb_last_damage synchronises)
        bound_damage(s)
        damaged.append(int(r.last_damage().sum()))
    tiles = ((size + 15) // 16) ** 2
    res["d_bound_damage"].update(rows_changed=m, damaged_tiles_mean=round(float(np.mean(damaged)), 1), tiles=tiles)
    r.set_damage_tracking(False)
    res["k_draw_data_us"] = kernel_us(r, t, all_rows, p, 20)
    r.close()
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "color_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
