"""Composition of resident fragments (Renderer.compose, vb_compose) against the host route that rebuilds the scene every frame
(vb_scene_append per instance + vb_scene_upload_device). Prints the card, its power limit and SM clock first, then per workload:
  compose_ms      device time of vb_compose (CUDA events around the call on the renderer's stream, behind a spin kernel so
                  that the host's part of the call is hidden), median of --steps frames
  compose_call_ms wall time of the vb_compose call on the host (the plan, the staging, the launches), median
  d2d_ms          a cudaMemcpyAsync device-to-device copy of the same number of bytes, same stream, median
  bytes           the composed scene's bytes (what k_compose_streams writes; it reads as many)
  frame_ms        device time of the frame rendered from the composed scene (events around the frame), median
  host_route_ms   wall time of the host route for the same frame (appends, device resolve), median
  scene_bytes_identical  the packed scene, ramps and atlas of the two routes are byte-identical (every frame is checked)
  compose_split_us  device time per compose of each kernel and copy of vb_compose (torch.profiler, a separate pass of 5
                  composes after the timed frames)
  pixels_max_diff / pixels_differing  between the two routes' frames, the largest over the frames (each route renders on
                  its own renderer)
Workloads: (a) 64 tiles of 470 paris-like paths (512 px, seed = tile) on an 8 x 8 grid at 4096^2 MSAA16, panned every frame;
(b) 10,000 instances of 16 small fragments (gradients, two with images) at 2048^2 Area, every transform changing. The tiles
are drawn with the native scene front end (NativeScene) so that both routes start from the same fragments. With --out the
rows also go to DIR/compose_probe.jsonl:
    python tools/compose_probe.py [--steps 20] [--out DIR]"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import (BLACK, EXTEND_REFLECT, FILL_EVEN_ODD, FILL_NON_ZERO, Color, Gradient, Image, Stroke,  # noqa: E402
                                 STYLE_CAP_BUTT, STYLE_CAP_ROUND, STYLE_CAP_SQUARE, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER, STYLE_JOIN_ROUND)
from vello_b200.renderer import Renderer, _Instance, _Layout  # noqa: E402
from vello_b200.scene_native import NativeScene  # noqa: E402
from vello_b200.shapes import Affine, BezPath, Circle, Rect, RoundedRect  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def native_paris_like(n_paths, size, seed):
    """The geometry of scenes.paris_like (same generator and draws), drawn through NativeScene calls."""
    rng = np.random.default_rng(seed)
    s = NativeScene()
    t = Affine.scale(size / 4096.0)
    f32 = np.float32

    def col():
        r, g, b = (int(v) for v in rng.integers(0, 256, 3))
        a = int(rng.integers(64, 230)) if rng.random() < 0.2 else 255
        return Color.from_rgba8(r, g, b, a)

    for _ in range(n_paths):
        kind = rng.random()
        cx, cy = rng.uniform(0, 4096, 2)
        extent = math.exp(rng.uniform(math.log(4.0), math.log(400.0)))
        c = col()
        p = BezPath()
        if kind < 0.70:
            n = int(rng.integers(8, 61))
            ang = np.sort(rng.uniform(0, 2 * math.pi, n))
            rad = rng.uniform(0.35, 1.0, n) * (extent * 0.5)
            pts = np.stack([cx + rad * np.cos(ang), cy + rad * np.sin(ang)], axis=1).astype(f32)
            p.move_to(*pts[0])
            for q in pts[1:]:
                p.line_to(*q)
            p.close_path()
            s.fill(FILL_NON_ZERO if rng.random() < 0.9 else FILL_EVEN_ODD, t, c, None, p)
        elif kind < 0.95:
            n = int(rng.integers(20, 201))
            step = extent / 16.0 + 1.0
            heading = rng.uniform(0, 2 * math.pi) + np.cumsum(rng.normal(0, 0.25, n))
            d = np.stack([np.cos(heading), np.sin(heading)], axis=1) * step
            pts = (np.array([cx, cy]) + np.cumsum(d, axis=0)).astype(f32)
            join = (STYLE_JOIN_ROUND, STYLE_JOIN_BEVEL, STYLE_JOIN_MITER)[int(rng.integers(0, 3))]
            cap = (STYLE_CAP_ROUND, STYLE_CAP_BUTT, STYLE_CAP_SQUARE)[int(rng.integers(0, 3))]
            st = Stroke(float(f32(rng.uniform(0.5, 6.0))), join=join, start_cap=cap, end_cap=cap)
            p.move_to(*pts[0])
            for q in pts[1:]:
                p.line_to(*q)
            s.stroke(st, t, c, None, p)
        else:
            n = int(rng.integers(6, 13))
            ang = np.linspace(0, 2 * math.pi, n, endpoint=False) + rng.uniform(0, 1)
            rad = rng.uniform(0.5, 1.0, n) * (extent * 0.5)
            on = np.stack([cx + rad * np.cos(ang), cy + rad * np.sin(ang)], axis=1)
            tang = np.stack([-np.sin(ang), np.cos(ang)], axis=1) * (rad * (2 * math.pi / n) * 0.4)[:, None]
            p.move_to(*on[0])
            for i in range(n):
                j = (i + 1) % n
                p.curve_to(*(on[i] + tang[i]), *(on[j] - tang[j]), *on[j])
            p.close_path()
            s.fill(FILL_NON_ZERO, t, c, None, p)
    return s


def small_fragments(rng):
    """16 small fragments: gradients of every kind, two of them drawing images."""
    out = []
    imgs = [Image(rng.integers(0, 256, (16, 16, 4), dtype=np.uint8)), Image(rng.integers(0, 256, (24, 12, 4), dtype=np.uint8))]
    for k in range(16):
        s = NativeScene()
        stops = [(0.0, Color(*rng.uniform(0, 1, 3), 1.0)), (1.0, Color(*rng.uniform(0, 1, 3), float(rng.uniform(0.3, 1))))]
        g = [Gradient.linear((0, 0), (20, 8), stops), Gradient.radial((8, 8), 1, (10, 8), 12, stops, EXTEND_REFLECT),
             Gradient.sweep((8, 8), 0.0, 4.0, stops)][k % 3]
        s.fill(FILL_NON_ZERO, Affine.IDENTITY, g, None, RoundedRect(0, 0, 18, 14, 3))
        s.stroke(Stroke(1.5), Affine.IDENTITY, Color(*rng.uniform(0, 1, 3), 1.0), None, Circle(9, 7, 6))
        if k < 2:
            s.draw_image(imgs[k], Affine.translate(2, 2) * Affine.scale(0.5))
        out.append(s)
    return out


class Timer:
    """CUDA events around work enqueued on the renderer's stream. The stream is first given ~5 ms of device work (a spin
    kernel), so that the events measure the device time of the enqueued work and not the host time of enqueueing it."""

    def __init__(self, r):
        self.stream = torch.cuda.ExternalStream(r.stream)
        self.a, self.b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def __enter__(self):
        with torch.cuda.stream(self.stream):
            torch.cuda._sleep(10_000_000)
        self.a.record(self.stream)

    def __exit__(self, *exc):
        self.b.record(self.stream)

    def ms(self):
        self.b.synchronize()
        return self.a.elapsed_time(self.b)


def split(r, ids, instances_of, steps, n=5):
    """Where a compose's device time goes: a separate pass of n composes (after the timed frames, so that tracing does not
    touch them) under torch.profiler with CUDA activities; device time per compose of each kernel and copy, in us."""
    from torch.profiler import ProfilerActivity, profile
    arrs = []
    for s in range(n):
        inst = instances_of(steps + 2 + s)
        arr = (_Instance * len(inst))()
        for k, (i, t) in enumerate(inst):
            arr[k].fragment, arr[k].has_transform = ids[i], 1
            arr[k].transform[:] = [float(v) for v in t.coeffs]
        arrs.append(arr)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for arr in arrs:
            r._check(r.lib.vb_compose(r.handle, arr, len(arr), None, None), "vb_compose")
            torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0.0)
        if us > 0:
            name = e.key.split("(")[0][:48]
            out[name] = round(out.get(name, 0.0) + us / n, 2)
    return out


def run(name, frags, instances_of, w, h, aa, steps, out):
    r, host = Renderer(), Renderer()
    ids = [r.upload_fragment(f) for f in frags]
    p = RenderParams(BLACK, w, h, aa)
    tm = Timer(r)
    rows = {"compose_ms": [], "compose_call_ms": [], "d2d_ms": [], "frame_ms": [], "host_route_ms": []}
    same_bytes, max_diff, n_diff = True, 0, 0
    nbytes = 0
    for step in range(steps + 2):  # two warm-up frames
        inst = instances_of(step)
        arr = (_Instance * len(inst))()
        for k, (i, t) in enumerate(inst):
            arr[k].fragment, arr[k].has_transform = ids[i], 1
            arr[k].transform[:] = [float(v) for v in t.coeffs]
        lay = _Layout()
        with tm:
            t0 = time.perf_counter()
            rc = r.lib.vb_compose(r.handle, arr, len(inst), C.byref(lay), None)
            call_ms = (time.perf_counter() - t0) * 1e3
        r._check(rc, "vb_compose")
        c_ms = tm.ms()
        r.render_resident(p)
        f_ms = r.lib.vb_last_frame_ms(r.handle)
        img = r.download_target(p)
        if nbytes == 0:
            nbytes = r.download("scene", np.uint8).size
            src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            dst = torch.empty_like(src)
        with torch.cuda.stream(tm.stream), tm:
            dst.copy_(src)
        d_ms = tm.ms()
        t0 = time.perf_counter()
        s = NativeScene()
        for i, t in inst:
            s.append(frags[i], t)
        s.upload_device(host)
        host.render_resident(p)
        torch.cuda.synchronize()
        hr_ms = (time.perf_counter() - t0) * 1e3
        same_bytes = same_bytes and all(bool(np.array_equal(r.download(b, np.uint8), host.download(b, np.uint8)))
                                        for b in ("scene", "ramps", "atlas"))
        d = np.abs(host.download_target(p).astype(np.int32) - img.astype(np.int32))
        max_diff, n_diff = max(max_diff, int(d.max())), max(n_diff, int((d > 0).sum()))
        if step >= 2:
            for k, v in (("compose_ms", c_ms), ("compose_call_ms", call_ms), ("d2d_ms", d_ms), ("frame_ms", f_ms), ("host_route_ms", hr_ms)):
                rows[k].append(v)
    row = {"workload": name, "instances": len(instances_of(0)), "bytes": int(nbytes), "scene_bytes_identical": same_bytes,
           "pixels_max_diff": max_diff, "pixels_differing": n_diff}
    row.update({k: round(float(np.median(v)), 4) for k, v in rows.items()})
    row["compose_over_d2d"] = round(row["compose_ms"] / row["d2d_ms"], 2) if row["d2d_ms"] else None
    row["compose_split_us"] = split(r, ids, instances_of, steps)
    print(json.dumps(row), flush=True)
    if out:
        with open(os.path.join(out, "compose_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(row) + "\n")
    for i in ids:
        r.free_fragment(i)
    r.close()
    host.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    print(f"card: {card()}", flush=True)
    tiles = [native_paris_like(470, 512, k) for k in range(64)]
    run("a_tiles_8x8_4096_msaa16", tiles,
        lambda s: [(k, Affine.translate(512 * (k % 8) + 3.25 * s, 512 * (k // 8) - 1.5 * s)) for k in range(64)],
        4096, 4096, AA_MSAA16, a.steps, a.out)
    rng = np.random.default_rng(5)
    smalls = small_fragments(rng)
    base = rng.uniform(0, 2000, (10000, 2))
    run("b_10k_instances_2048_area", smalls,
        lambda s: [(k % 16, Affine.translate(*(base[k] + [0.7 * s, -0.4 * s])) * Affine.rotate(0.01 * s + k)) for k in range(10000)],
        2048, 2048, AA_AREA, a.steps, a.out)


if __name__ == "__main__":
    main()
