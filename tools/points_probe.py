"""Bound path points (Renderer.bind_path_points, vb_bind_path_points) against the host route (the packed scene's path-data words
patched on the host and the scene uploaded again, vb_scene_upload). Prints the card, its power limit and SM clock before and
after, then frames/s and ms per frame (host wall time of --steps blocking frames after --warmup, each frame ending in a
synchronise), kernel launches, flatten's line count and whether the graph replayed, of:
  (a) chart   a live line chart: 1,024 stroked polylines of 1,024 points at 4096x2048 MSAA16, every y value rewritten by a
              torch op on vb_stream each frame (bound), or the same rows patched into the packed scene and uploaded (host)
  (b) paris   paris-like 30k at 4096^2 MSAA16 with every point displaced each frame, bound and host; and bound with rows
              equal to the encoded points (the binding's own cost, on the unbound frame's geometry)
  (c) damage  (b) bound with the points of 1 % of the paths changed per frame, damage-tracked into a device destination; also
              the mean damaged tile count per frame
Parity: the last timed frame of the bound route is compared with the last timed frame of the host route (the same rows).
With --profile, instead, the device time of one k_path_points from torch.profiler on (a) and (b), nothing else timed. With
--out the result also goes to DIR/points_probe[_profile].json:
    python tools/points_probe.py [--steps 50] [--warmup 5] [--out DIR] [--profile]"""
import argparse
import json
import math
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
from vello_b200.encoding import BLACK, Color, Scene, Stroke, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402
from vello_b200.shapes import Affine  # noqa: E402

K = 8  # distinct row sets, cycled


def chart(n_lines=1024, n_pts=1024, w=4096, h=2048):
    """n_lines stroked polylines of n_pts points across the frame (what Scene.stroke encodes for them, in bulk: n_pts points,
    then the open cap marker's 2); the line of every point row."""
    s = Scene()
    e = s.encoding
    line_of = []
    g = np.random.default_rng(5)
    xs = np.linspace(8, w - 8, n_pts)
    e.encode_transform(Affine.IDENTITY)
    assert e.encode_stroke_style(Stroke(1.5))
    for i in range(n_lines):
        y = (i + 0.5) * h / n_lines + g.uniform(-2, 2, n_pts)
        a = s.n_points
        scenes._bulk_stroke_polyline(e, np.stack([xs, y], 1).astype(np.float32))
        e.encode_color(Color(*map(float, g.uniform(0.2, 1.0, 3)), 1.0))
        line_of.append(np.full(s.n_points - a, i, np.float32))
    return s, np.concatenate(line_of)


def path_first(packed):
    """The first point of every path (n_paths + 1), from the tag bytes (the table k_path_point_slots builds)."""
    L = packed.layout
    tags = packed.scene[L.path_tag_base:L.path_data_base].view(np.uint8).astype(np.int64)
    pts = np.cumsum((tags & 3) + ((tags >> 2) & 1))
    ends = np.nonzero(tags & 0x10)[0]
    return np.concatenate([[0], pts[ends]])[:L.n_paths + 1]


def timed(steps, warmup, frame):
    for s in range(warmup):
        frame(s)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(steps):
        frame(warmup + s)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    return {"fps": round(1e3 / ms, 1), "ms_per_frame": round(ms, 4)}


def bound_route(r, t, p, step, steps, warmup, dst=0):
    """Time `step(s)` (rows written on vb_stream) + a frame; launches and graph captures during the timed frames."""
    st = torch.cuda.ExternalStream(r.stream)

    def frame(s):
        with torch.cuda.stream(st):
            step(s)
        r.render_resident(p, dst)

    frame(0)
    frame(1)  # under damage tracking the first frame is full and the second the first incremental one
    caps = r.debug_graph_captures()
    res = timed(steps, warmup, frame)
    res["graph_replayed"] = r.debug_graph_captures() == caps
    with torch.cuda.stream(st):
        step(warmup + steps - 1)  # the last timed frame again, for its launch count
    last = r.render_resident(p, dst)
    res["launches"] = int(last.kernel_launches)
    res["lines"] = int(last.lines)  # flatten's lines in that frame
    return res


def host_route(rc, packed, p, rows_of, steps, warmup):
    """Time the host route: path-data words of the packed scene patched with rows_of(s), the scene uploaded, a frame."""
    L = packed.layout
    scene = packed.scene.copy()
    pd = scene[L.path_data_base:L.draw_tag_base].view(np.float32).reshape(-1, 2)
    work = type(packed)(scene, L, packed.ramps, packed.atlas)

    def frame(s):
        pd[:] = rows_of(s)  # the host patch ...
        rc.upload(work)     # ... and the upload
        return rc.render_resident(p)

    res = timed(steps, warmup, frame)
    res["launches"] = int(frame(warmup + steps - 1).kernel_launches)
    res["scene_mib_per_frame"] = round(packed.scene.nbytes / 2**20, 2)
    return res


def parity(a, b):
    d = np.abs(a.astype(np.int32) - b.astype(np.int32))
    return {"max_diff": int(d.max()), "differing": int((d > 0).sum())}


def kernel_us(r, frame, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            frame(s)
    torch.cuda.synchronize()
    for e in prof.key_averages():
        if e.key.startswith("k_path_points") or "k_path_points(" in e.key:
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
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    res = {"card_before": card()}

    # (a) the live line chart: y = centre of its line + A sin(k x + phase of the line + step phase), a torch op per frame
    cs, line_of = chart()
    cpacked = resolve(cs.encoding)
    cw, ch = 4096, 2048
    cp = RenderParams(BLACK, cw, ch, AA_MSAA16)
    base = torch.from_numpy(cpacked.scene[cpacked.layout.path_data_base:cpacked.layout.draw_tag_base].view(np.float32).reshape(-1, 2).copy()).cuda()
    line = torch.from_numpy(line_of).cuda()
    centre = (line + 0.5) * (ch / 1024.0)
    ct = base.clone()

    def chart_step(s):
        ph = 2.0 * math.pi * (s % K) / K
        ct[:, 1] = centre + torch.sin(base[:, 0] * 0.004 + line * 0.3 + ph) * (0.8 * ch / 1024.0)

    chart_rows = []
    for s in range(K):
        chart_step(s)
        chart_rows.append(ct.cpu().numpy().copy())
    res["a_workload"] = f"line chart {cs.n_draw_objects} stroked polylines, {cs.n_points} points, {cw}x{ch} MSAA16"

    # (b) paris-like 30k: every point displaced by one of K seeded sets
    size = 4096
    packed = resolve(scenes.paris_like(30000, size, 30000).encoding)
    pp = RenderParams(BLACK, size, size, AA_MSAA16)
    L = packed.layout
    pbase = packed.scene[L.path_data_base:L.draw_tag_base].view(np.float32).reshape(-1, 2).copy()
    g = np.random.default_rng(1)
    paris_rows = [(pbase + g.uniform(-1.5, 1.5, pbase.shape)).astype(np.float32) for _ in range(K)]
    all_paris = torch.from_numpy(np.stack(paris_rows)).cuda()
    pt = all_paris[0].clone()
    res["b_workload"] = f"paris-like-30k {size}x{size} MSAA16, {L.n_paths} paths, {len(pbase)} points"

    r = Renderer()
    if args.profile:
        r.upload(cpacked)
        r.bind_path_points(ct)
        st = torch.cuda.ExternalStream(r.stream)

        def cframe(s):
            with torch.cuda.stream(st):
                chart_step(s)
            r.render_resident(cp)

        for s in range(3):
            cframe(s)
        res["a_k_path_points_us"] = kernel_us(r, cframe, 20)
        res["a_points"] = int(cs.n_points)
        r.upload(packed)
        r.bind_path_points(pt)

        def pframe(s):
            with torch.cuda.stream(st):
                pt.copy_(all_paris[s % K])
            r.render_resident(pp)

        for s in range(3):
            pframe(s)
        res["b_k_path_points_us"] = kernel_us(r, pframe, 20)
        res["b_points"] = int(len(pbase))
        r.close()
    else:
        rc = Renderer()
        # (a)
        r.upload(cpacked)
        res["a_resident_unbound"] = timed(args.steps, args.warmup, lambda s: r.render_resident(cp))
        res["a_resident_unbound"]["launches"] = int(r.render_resident(cp).kernel_launches)
        r.bind_path_points(ct)
        res["a_bound"] = bound_route(r, ct, cp, chart_step, args.steps, args.warmup)
        img_b = r.download_target(cp)
        res["a_host"] = host_route(rc, cpacked, cp, lambda s: chart_rows[s % K], args.steps, args.warmup)
        res["a_parity_last_timed_frame"] = parity(img_b, rc.download_target(cp))
        # (b)
        r.upload(packed)
        res["b_resident_unbound"] = timed(args.steps, args.warmup, lambda s: r.render_resident(pp))
        last = r.render_resident(pp)
        res["b_resident_unbound"].update(launches=int(last.kernel_launches), lines=int(last.lines))
        # the binding's own cost: rows equal to the encoded points, copied each frame (the geometry of the unbound frame)
        penc = torch.from_numpy(pbase).cuda()
        pt.copy_(penc)
        r.bind_path_points(pt)
        res["b_bound_encoded_rows"] = bound_route(r, pt, pp, lambda s: pt.copy_(penc), args.steps, args.warmup)
        res["b_bound"] = bound_route(r, pt, pp, lambda s: pt.copy_(all_paris[s % K]), args.steps, args.warmup)
        img_b = r.download_target(pp)
        res["b_host"] = host_route(rc, packed, pp, lambda s: paris_rows[s % K], args.steps, args.warmup)
        res["b_parity_last_timed_frame"] = parity(img_b, rc.download_target(pp))
        rc.close()
        # (c) 1 % of the paths' points change per frame, damage-tracked into a device destination
        first = path_first(packed)
        m = max(1, L.n_paths // 100)
        picks = []
        for _ in range(K):
            paths = g.choice(L.n_paths, m, replace=False)
            picks.append(np.concatenate([np.arange(first[q], first[q + 1]) for q in paths]))
        picks = [torch.from_numpy(q).cuda() for q in picks]
        dst = torch.zeros((size, size, 4), dtype=torch.uint8, device="cuda")
        pt.copy_(all_paris[0])
        r.set_damage_tracking(True)

        def damage_step(s):
            q = picks[s % K]
            pt[q] = all_paris[(s + 1) % K][q]

        res["c_bound_damage"] = bound_route(r, pt, pp, damage_step, args.steps, args.warmup, dst.data_ptr())
        st = torch.cuda.ExternalStream(r.stream)
        damaged = []
        for s in range(K):  # the damage of further frames, outside the timed ones (vb_last_damage synchronises)
            with torch.cuda.stream(st):
                damage_step(s)
            r.render_resident(pp, dst.data_ptr())
            damaged.append(int(r.last_damage().sum()))
        # the last of them against a full frame of the same rows
        rows_now = pt.cpu().numpy()
        rf = Renderer()
        full = packed.scene.copy()
        full[L.path_data_base:L.draw_tag_base] = rows_now.reshape(-1).view(np.uint32)
        rf.upload(type(packed)(full, L, packed.ramps, packed.atlas))
        rf.render_resident(pp)
        res["c_parity_with_full_host_frame"] = parity(dst.cpu().numpy(), rf.download_target(pp))
        rf.close()
        tiles = ((size + 15) // 16) ** 2
        res["c_bound_damage"].update(paths_changed=m, damaged_tiles_mean=round(float(np.mean(damaged)), 1), tiles=tiles)
        r.set_damage_tracking(False)
        r.close()
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "points_probe_profile.json" if args.profile else "points_probe.json"
        with open(os.path.join(args.out, name), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
