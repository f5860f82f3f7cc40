"""Fragments from device arrays (Renderer.upload_device_paths, vb_fragment_from_device_paths / _curves) against the host
route, on four inputs in a 4096^2 frame: about 30k paris-like polygons (1.5M points, a few with holes, filled), one 1M-point
polyline (stroked), 100k circles of four cubics each (1.3M points, filled, with point_kinds) and 20k glyph-like quadratic
contours (an outer contour and a counter each, filled, with point_kinds). Prints, with the card, its power limit and SM clock:
  call_ms     the call's wall time (it ends with its one synchronisation), and kernel_ms, the span of its work on vb_stream
              from CUDA events recorded around it (scratch clears, the four kernels and the read-back of the totals)
  host_ms     the host route for the same rows: the arrays copied to the host, one vb_scene_fill / vb_scene_stroke per path
              (ctypes calls over views of one verb and one coordinate array), and vb_scene_upload_fragment
  frames      a per-frame loop at 4096^2 MSAA16 of build + compose + render against native encode + upload + compose + render;
              both change the geometry every frame (points moved by the frame number on the device, or on the host), so the
              compose's stream lengths may change and the frame graph is captured anew (graph_captures counts it); and
              the cost of that capture: frames that cycle through six row counts (new lengths every frame, more than
              the four cached graphs, so a capture every frame), with frame graphs on and off
Dashed strokes (Renderer.upload_device_dashes, vb_fragment_from_device_dashes) on three more inputs: the 30k polygons' outlines
with pattern (6, 3), the 1M-point polyline with (4, 4) and the 100k circles with (2, 2). For each: call_ms and kernel_ms as
above; kernels_us, each kernel's time per call from torch.profiler; host_ms, the host route with vb_scene_stroke's dashes (on
the first `host_fraction` of the paths for the circles, whose host dash takes minutes); and `animated`, frames of build with
the dash offset moved by 0.5 per frame + recompose + render at 4096^2 MSAA16, with frame graphs on and off.
--inputs picks some of the inputs by name. With --out the result also goes to DIR/device_paths_probe.json:
    python tools/device_paths_probe.py [--reps 10] [--frames 20] [--inputs polygons_30k,...,dashes_polygons_30k] [--out DIR]"""
import argparse
import ctypes as C
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
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Stroke  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402
from vello_b200.scene_native import NativeScene, _Brush, _Color, _Path, _Stroke, _affine  # noqa: E402
from vello_b200.shapes import Affine  # noqa: E402

SIZE = 4096


def polygons(n=30_000, seed=1):
    """Paris-like blocks: n polygons of 20..80 points around random centres, every 10th with a hole."""
    rng = np.random.default_rng(seed)
    pts, roff, poff = [], [0], [0]
    for i in range(n):
        c = rng.uniform(0, SIZE, 2)
        for hole in range(2 if i % 10 == 0 else 1):
            k = int(rng.integers(20, 81))
            t = np.sort(rng.uniform(0, 2 * np.pi, k))
            rad = rng.uniform(20, 60, k) * (0.3 if hole else 1.0)
            pts.append(np.stack([c[0] + rad * np.cos(t), c[1] + rad * np.sin(t)], 1))
            roff.append(roff[-1] + k)
        poff.append(len(roff) - 1)
    cols = rng.uniform(0, 1, (n, 4)).astype(np.float32)
    cols[:, 3] = 0.8
    return np.concatenate(pts).astype(np.float32), np.array(roff, np.int32), np.array(poff, np.int32), cols


def polyline(n=1_000_000, seed=2):
    rng = np.random.default_rng(seed)
    x = np.linspace(8, SIZE - 8, n)
    y = SIZE / 2 + SIZE / 3 * np.sin(x / 300.0) + rng.normal(0, 3, n)
    return np.stack([x, y], 1).astype(np.float32), np.array([0, n], np.int32), None, np.array([[1, 0.9, 0.2, 1]], np.float32)


def circles(n=100_000, seed=3):
    """n circles of radius 4..40, each M and the four cubics of shapes.path_elements(Circle) (13 points, the last the first)."""
    rng = np.random.default_rng(seed)
    arm, unit = 0.551915024494, [(1.0, 0.0)]
    for ix in range(1, 5):
        th0, th1 = (ix - 1) * np.pi / 2, ix * np.pi / 2
        s0, c0 = np.sin(th0), np.cos(th0)
        s1, c1 = (0.0, 1.0) if ix == 4 else (np.sin(th1), np.cos(th1))
        unit += [(c0 - arm * s0, s0 + arm * c0), (c1 + arm * s1, s1 - arm * c1), (c1, s1)]
    c, rad = rng.uniform(0, SIZE, (n, 2)), rng.uniform(4, 40, n)
    pts = (c[:, None, :] + rad[:, None, None] * np.array(unit)[None]).reshape(-1, 2).astype(np.float32)
    kinds = np.tile(np.array([0] + [1, 1, 0] * 4, np.uint8), n)
    cols = rng.uniform(0, 1, (n, 4)).astype(np.float32)
    return pts, np.arange(0, 13 * n + 1, 13, dtype=np.int32), None, cols, kinds


def glyphs(n=20_000, seed=4):
    """n glyph-like outlines of 20..60 px: an outer quadratic contour of 8 quads and a counter wound the other way, with
    TrueType's implied on-curve points inserted (17 points a contour, the last the first)."""
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 2 * np.pi, 17)
    rad = np.where(np.arange(17) % 2 == 0, 1.0, 1.0 / np.cos(np.pi / 8))  # control points on the tangents' crossings
    unit = np.stack([np.cos(t) * rad, np.sin(t) * rad], 1)
    unit[-1] = unit[0]
    s, c = rng.uniform(10, 30, n), rng.uniform(0, SIZE, (n, 2))
    outer = c[:, None, :] + s[:, None, None] * unit[None] * (1.0, 1.3)
    inner = c[:, None, :] + 0.5 * s[:, None, None] * unit[None, ::-1]
    pts = np.concatenate([outer, inner], 1).reshape(-1, 2).astype(np.float32)
    kinds = np.tile((np.arange(17) % 2).astype(np.uint8), 2 * n)
    cols = rng.uniform(0, 1, (n, 4)).astype(np.float32)
    return pts, np.arange(0, 34 * n + 1, 17, dtype=np.int32), np.arange(0, 2 * n + 1, 2, dtype=np.int32), cols, kinds


def host_route(r, pts, roff, poff, cols, style, kinds=None):
    """Copy the device arrays to the host, encode one fill or stroke per path through the native scene, upload the fragment."""
    p, ro, po, co, ki = (t.cpu().numpy() if t is not None else None for t in (pts, roff, poff, cols, kinds))
    s = NativeScene()
    lib, h = s.lib, s.handle
    n_paths = len(po) - 1 if po is not None else len(ro) - 1
    # one verb and one coordinate array: per ring M, then L, Q or C per on-curve point after the first (the coordinates are
    # the points, in order), then Z (strokes here are open: no Z)
    stroke = isinstance(style, Stroke)
    on = np.ones(len(p), bool) if ki is None else ki == 0
    verb_of = np.frombuffer(b"?LQC", np.uint8)
    verbs, vstart = [], [0]
    for a, b in zip(ro[:-1], ro[1:]):
        ends = np.flatnonzero(on[a:b])
        verbs.append(np.concatenate([[ord("M")], verb_of[np.diff(ends)], [] if stroke else [ord("Z")]]).astype(np.uint8))
        vstart.append(vstart[-1] + len(verbs[-1]))
    verbs = np.concatenate(verbs)
    coords = p.astype(np.float64).reshape(-1)
    ident = _affine(Affine.IDENTITY)
    st = _Stroke(style.width, style.join, style.start_cap, style.end_cap, style.miter_limit, None, 0, 0.0) if stroke else None
    for i in range(n_paths):
        r0, r1 = (int(po[i]), int(po[i + 1])) if po is not None else (i, i + 1)
        b = _Brush()
        b.kind, b.color = 0, _Color(*[float(v) for v in co[i]])
        path = _Path(verbs.ctypes.data + int(vstart[r0]), int(vstart[r1] - vstart[r0]), coords.ctypes.data + 16 * int(ro[r0]))
        if stroke:
            lib.vb_scene_stroke(h, C.byref(st), ident, C.byref(b), None, C.byref(path))
        else:
            lib.vb_scene_fill(h, FILL_NON_ZERO, ident, C.byref(b), None, C.byref(path))
    return r.upload_fragment(s)


def measure(r, name, data, style, reps, n_frames):
    pts, roff, poff, cols, kinds = (torch.as_tensor(a).cuda() if a is not None else None for a in (tuple(data) + (None,))[:5])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.ExternalStream(r.stream)
    kw = dict(path_offsets=poff, style=style, closed=False)
    if kinds is not None:
        kw["point_kinds"] = kinds
    f, n = r.upload_device_paths(pts, roff, cols, **kw)  # warm-up
    r.free_fragment(f)
    call, kern = [], []
    for _ in range(reps):
        ev0.record(st)
        t0 = time.perf_counter()
        f, n = r.upload_device_paths(pts, roff, cols, **kw)
        call.append((time.perf_counter() - t0) * 1e3)
        ev1.record(st)
        ev1.synchronize()
        kern.append(ev0.elapsed_time(ev1))
        r.free_fragment(f)
    host = []
    for _ in range(max(2, reps // 3)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = host_route(r, pts, roff, poff, cols, style, kinds)
        host.append((time.perf_counter() - t0) * 1e3)
        r.free_fragment(f)
    # frames: the geometry moves every frame (by 0.25 px per frame), rebuilt on the device or encoded on the host
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    out = {}
    for route in ("device", "host"):
        cap0 = r.debug_graph_captures()
        torch.cuda.synchronize()
        t0 = None
        for k in range(n_frames + 3):
            if k == 3:
                torch.cuda.synchronize()
                t0, cap0 = time.perf_counter(), r.debug_graph_captures()
            with torch.cuda.stream(st):
                moved = pts + 0.25 * (k % 8)
            if route == "device":
                f, _ = r.upload_device_paths(moved, roff, cols, **kw)
            else:
                f = host_route(r, moved, roff, poff, cols, style, kinds)
            r.compose([(f, None)])
            r.render_resident(p)
            r.free_fragment(f)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / n_frames
        out[route] = {"fps": round(1e3 / ms, 2), "ms_per_frame": round(ms, 3), "graph_captures": r.debug_graph_captures() - cap0}
    # recapture: the frames cycle through fragments of six stream lengths (all the rows, then 5/6 .. 1/6 of them), more than
    # the renderer's four cached frame graphs, so every frame captures its graph anew; against the same cycle without graphs
    def part(v):
        if poff is None and len(roff) == 2:
            q = pts.shape[0] * (6 - v) // 6
            return pts[:q], torch.tensor([0, q], dtype=torch.int32, device="cuda"), None, cols, None
        n_p = (len(cols)) * (6 - v) // 6
        n_r = int(poff[n_p]) if poff is not None else n_p
        q = int(roff[n_r])
        return pts[:q], roff[:n_r + 1], None if poff is None else poff[:n_p + 1], cols[:n_p], None if kinds is None else kinds[:q]
    halves = [part(v) for v in range(6)]
    for graphs in (True, False):
        r.set_cuda_graph(graphs)
        for k in range(n_frames + 3):
            if k == 3:
                torch.cuda.synchronize()
                t0, cap0 = time.perf_counter(), r.debug_graph_captures()
            q, ro, po, co, ki = halves[k % 6]
            f, _ = r.upload_device_paths(q, ro, co, path_offsets=po, style=style, closed=False, **({} if ki is None else {"point_kinds": ki}))
            r.compose([(f, None)])
            r.render_resident(p)
            r.free_fragment(f)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / n_frames
        out["cycling_graphs" if graphs else "cycling_no_graphs"] = {
            "fps": round(1e3 / ms, 2), "ms_per_frame": round(ms, 3), "graph_captures": r.debug_graph_captures() - cap0}
    r.set_cuda_graph(True)
    return {"input": name, "points": int(pts.shape[0]), "paths": int(cols.shape[0]), "draw_objects": n,
            "call_ms_median": round(float(np.median(call)), 3), "kernel_ms_median": round(float(np.median(kern)), 3),
            "host_ms_median": round(float(np.median(host)), 3), "frames": out}


def host_dash_route(r, pts, roff, poff, cols, stroke, kinds, closed, n_paths):
    """The host route of a dashed stroke for the first n_paths paths: arrays to the host, one dashed vb_scene_stroke per path."""
    p, ro, po, co, ki = (t.cpu().numpy() if t is not None else None for t in (pts, roff, poff, cols, kinds))
    s = NativeScene()
    lib, h = s.lib, s.handle
    on = np.ones(len(p), bool) if ki is None else ki == 0
    verb_of = np.frombuffer(b"?LQC", np.uint8)
    verbs, vstart = [], [0]
    for a, b in zip(ro[:-1], ro[1:]):
        ends = np.flatnonzero(on[a:b])
        verbs.append(np.concatenate([[ord("M")], verb_of[np.diff(ends)], [ord("Z")] if closed else []]).astype(np.uint8))
        vstart.append(vstart[-1] + len(verbs[-1]))
    verbs = np.concatenate(verbs)
    coords = p.astype(np.float64).reshape(-1)
    ident = _affine(Affine.IDENTITY)
    pat = (C.c_double * len(stroke.dash_pattern))(*stroke.dash_pattern)
    st = _Stroke(stroke.width, stroke.join, stroke.start_cap, stroke.end_cap, stroke.miter_limit, C.cast(pat, C.c_void_p),
                 len(stroke.dash_pattern), stroke.dash_offset)
    for i in range(n_paths):
        r0, r1 = (int(po[i]), int(po[i + 1])) if po is not None else (i, i + 1)
        b = _Brush()
        b.kind, b.color = 0, _Color(*[float(v) for v in co[i]])
        path = _Path(verbs.ctypes.data + int(vstart[r0]), int(vstart[r1] - vstart[r0]), coords.ctypes.data + 16 * int(ro[r0]))
        lib.vb_scene_stroke(h, C.byref(st), ident, C.byref(b), None, C.byref(path))
    return r.upload_fragment(s)


def measure_dashes(r, name, data, stroke, closed, reps, n_frames, host_fraction=1.0):
    pts, roff, poff, cols, kinds = (torch.as_tensor(a).cuda() if a is not None else None for a in (tuple(data) + (None,))[:5])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.ExternalStream(r.stream)
    kw = dict(path_offsets=poff, closed=closed, point_kinds=kinds)
    f, n = r.upload_device_dashes(pts, roff, cols, stroke, **kw)  # warm-up
    r.free_fragment(f)
    call, kern = [], []
    for _ in range(reps):
        ev0.record(st)
        t0 = time.perf_counter()
        f, n = r.upload_device_dashes(pts, roff, cols, stroke, **kw)
        call.append((time.perf_counter() - t0) * 1e3)
        ev1.record(st)
        ev1.synchronize()
        kern.append(ev0.elapsed_time(ev1))
        r.free_fragment(f)
    prof_calls = max(1, min(reps, 5))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(prof_calls):
            f, _ = r.upload_device_dashes(pts, roff, cols, stroke, **kw)
            r.free_fragment(f)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if "k_device_" in e.key:
            total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kernels[e.key.split("(")[0]] = round(total / prof_calls, 1)
    n_paths = len(cols)
    n_host = max(1, int(n_paths * host_fraction))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f = host_dash_route(r, pts, roff, poff, cols, stroke, kinds, closed, n_host)
    host = (time.perf_counter() - t0) * 1e3
    r.free_fragment(f)
    # an animated dash offset: a new fragment each frame, recomposed beside nothing else and rendered
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    anim = {}
    for graphs in (True, False):
        r.set_cuda_graph(graphs)
        t0 = None
        for k in range(n_frames + 3):
            if k == 3:
                torch.cuda.synchronize()
                t0, cap0 = time.perf_counter(), r.debug_graph_captures()
            moving = Stroke(stroke.width, stroke.join, stroke.miter_limit, stroke.start_cap, stroke.end_cap, stroke.dash_pattern,
                            0.5 * k)
            f, _ = r.upload_device_dashes(pts, roff, cols, moving, **kw)
            r.recompose([(f, None)])
            r.render_resident(p)
            r.free_fragment(f)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / n_frames
        anim["graphs" if graphs else "no_graphs"] = {"fps": round(1e3 / ms, 2), "ms_per_frame": round(ms, 3),
                                                      "graph_captures": r.debug_graph_captures() - cap0}
    r.set_cuda_graph(True)
    return {"input": name, "pattern": list(stroke.dash_pattern), "points": int(pts.shape[0]), "paths": n_paths,
            "draw_objects": n, "call_ms": [round(v, 3) for v in call], "kernel_ms": [round(v, 3) for v in kern],
            "kernels_us": kernels, "host_ms": round(host, 1), "host_fraction": n_host / n_paths, "animated": anim}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--inputs", default="polygons_30k,polyline_1m,circles_100k,glyphs_20k,dashes_polygons_30k,dashes_polyline_1m,"
                                        "dashes_circles_100k")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    inputs = {"polygons_30k": (polygons, FILL_NON_ZERO), "polyline_1m": (polyline, Stroke(2.0)),
              "circles_100k": (circles, FILL_NON_ZERO), "glyphs_20k": (glyphs, FILL_NON_ZERO)}
    dashes = {"dashes_polygons_30k": (polygons, Stroke(1.5, dash_pattern=(6.0, 3.0)), True, 1.0),
              "dashes_polyline_1m": (polyline, Stroke(2.0, dash_pattern=(4.0, 4.0)), False, 1.0),
              "dashes_circles_100k": (circles, Stroke(1.5, dash_pattern=(2.0, 2.0)), True, 0.05)}
    r = Renderer()
    results = []
    for k in a.inputs.split(","):
        if k in dashes:
            make, stroke, closed, frac = dashes[k]
            results.append(measure_dashes(r, k, make(), stroke, closed, a.reps, a.frames, frac))
        else:
            results.append(measure(r, k, inputs[k][0](), inputs[k][1], a.reps, a.frames))
    res = {"card": card(), "results": results, "card_after": card()}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "device_paths_probe.json"), "w") as fh:
            json.dump(res, fh, indent=1)
    r.close()


if __name__ == "__main__":
    main()
