"""Bound transforms (Renderer.bind_transforms, vb_bind_transforms) against the host route (the packed scene's transform entries
patched on the host and the scene uploaded again, vb_scene_upload). Prints the card, its power limit and SM clock before and
after, then frames/s and ms per frame (host wall time of --steps blocking frames after --warmup, each frame ending in a
synchronise), kernel launches and whether the graph replayed, of:
  (a) sprites  20,000 markers at 4096^2 MSAA16, each a filled star, a stroked outline and a gradient badge with a brush
               transform, each under its own transform (80,000 rows); every row rewritten by a torch op on vb_stream each
               frame (bound), the same rows patched into the packed scene and uploaded (host), and the scene unbound (resident)
  (b) paris    paris-like 30k at 4096^2 MSAA16 with its transforms bound and rotating about the centre, and unbound
  (c) damage   (a) bound with 1 % of the markers moving per frame, damage-tracked into a device destination; also the mean
               damaged tile count per frame
Parity: the last timed frame of the bound route is compared with the last timed frame of the host route (the same rows).
With --profile, instead, the device time of one k_bound_transforms from torch.profiler on (a) and (b), nothing else timed.
With --out the result also goes to DIR/transform_probe[_profile].json:
    python tools/transform_probe.py [--steps 50] [--warmup 5] [--out DIR] [--profile]"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compose_probe import card  # noqa: E402
from points_probe import bound_route, parity, timed  # noqa: E402
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Gradient, Stroke, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402
from vello_b200.scene_native import NativeScene  # noqa: E402
from vello_b200.shapes import Affine, BezPath, Circle  # noqa: E402

K = 8  # distinct row sets, cycled
SIZE = 4096


def star(r0, r1, n=5):
    a = np.arange(2 * n) * np.pi / n
    rad = np.where(np.arange(2 * n) % 2 == 0, r1, r0)
    p = BezPath()
    p.els = [("M", float(rad[0]), 0.0)] + [("L", float(q * np.cos(t)), float(q * np.sin(t))) for q, t in zip(rad[1:], a[1:])] + [("Z",)]
    return p


def sprites(n=20000, size=SIZE, seed=3):
    """n markers on a jittered grid; each marker's calls push 4 entries: the star's, the outline's, the badge's and the badge's
    brush transform. Returns the scene and each entry's marker."""
    g = np.random.default_rng(seed)
    s = NativeScene()
    side = int(math.ceil(math.sqrt(n)))
    step = size / side
    shape, badge = star(4.0, 10.0), Circle(0, 0, 5)
    stops = [(0.0, Color(1.0, 0.8, 0.1, 1.0)), (1.0, Color(0.9, 0.1, 0.4, 1.0))]
    owner = []
    for i in range(n):
        x, y = (i % side + 0.5) * step + g.uniform(-2, 2), (i // side + 0.5) * step + g.uniform(-2, 2)
        c = Color(*map(float, g.uniform(0.2, 1.0, 3)), 1.0)
        s.fill(FILL_NON_ZERO, Affine.translate(x, y), c, None, shape)
        s.stroke(Stroke(1.0), Affine.translate(x, y + 0.25), Color(0.05, 0.05, 0.05, 1.0), None, shape)
        s.fill(FILL_NON_ZERO, Affine.translate(x + 6, y - 6), Gradient.linear((-5, 0), (5, 0), stops),
               Affine.rotate(float(g.uniform(0.1, 3.0))), badge)
        owner += [i] * 4
    assert s.n_transforms == 4 * n
    return s, np.asarray(owner)


def transforms(packed):
    L = packed.layout
    return packed.scene[L.transform_base:L.style_base].view(np.float32).reshape(-1, 6).copy()


def host_route(rc, packed, p, rows_of, steps, warmup):
    """Time the host route: transform entries of the packed scene patched with rows_of(s), the scene uploaded, a frame."""
    L = packed.layout
    scene = packed.scene.copy()
    tr = scene[L.transform_base:L.style_base].view(np.float32).reshape(-1, 6)
    work = type(packed)(scene, L, packed.ramps, packed.atlas)

    def frame(s):
        tr[:] = rows_of(s)  # the host patch ...
        rc.upload(work)     # ... and the upload
        return rc.render_resident(p)

    res = timed(steps, warmup, frame)
    res["launches"] = int(frame(warmup + steps - 1).kernel_launches)
    res["scene_mib_per_frame"] = round(packed.scene.nbytes / 2**20, 2)
    return res


def wobble(base, out, s, rows=None):
    """Rows of step s: each entry's linear part rotated by a small angle that depends on its index and the step, and its
    translation moved by up to 3 pixels (only `rows`, when given)."""
    ph = 2.0 * math.pi * (s % K) / K
    idx = torch.arange(base.shape[0], device=base.device, dtype=torch.float32) if rows is None else rows.to(torch.float32)
    src = base if rows is None else base[rows]
    th = 0.15 * torch.sin(idx * 0.37 + ph)
    c, sn = torch.cos(th), torch.sin(th)
    new = torch.empty_like(src)
    new[:, 0] = c * src[:, 0] - sn * src[:, 1]
    new[:, 1] = sn * src[:, 0] + c * src[:, 1]
    new[:, 2] = c * src[:, 2] - sn * src[:, 3]
    new[:, 3] = sn * src[:, 2] + c * src[:, 3]
    new[:, 4] = src[:, 4] + 3.0 * torch.cos(idx * 0.11 + ph)
    new[:, 5] = src[:, 5] + 3.0 * torch.sin(idx * 0.13 + ph)
    if rows is None:
        out.copy_(new)
    else:
        out[rows] = new


def rotation_rows(base, s, size=SIZE):
    """paris: every entry rotated about the frame's centre by the step's angle, R * T in f32."""
    th = 2.0 * math.pi * (s % K) / (8 * K)
    c, sn, cx = math.cos(th), math.sin(th), size / 2
    R = np.array([[c, -sn, cx - c * cx + sn * cx], [sn, c, cx - sn * cx - c * cx]])
    out = np.empty_like(base, dtype=np.float64)
    a, b, cc, d, e, f = (base[:, i].astype(np.float64) for i in range(6))
    out[:, 0] = R[0, 0] * a + R[0, 1] * b
    out[:, 1] = R[1, 0] * a + R[1, 1] * b
    out[:, 2] = R[0, 0] * cc + R[0, 1] * d
    out[:, 3] = R[1, 0] * cc + R[1, 1] * d
    out[:, 4] = R[0, 0] * e + R[0, 1] * f + R[0, 2]
    out[:, 5] = R[1, 0] * e + R[1, 1] * f + R[1, 2]
    return out.astype(np.float32)


def kernel_us(frame, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            frame(s)
    torch.cuda.synchronize()
    for e in prof.key_averages():
        if "k_bound_transforms" in e.key:
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
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)

    ss, owner = sprites()
    spacked = ss.resolve()
    sbase_np = transforms(spacked)
    sbase = torch.from_numpy(sbase_np).cuda()
    st_rows = sbase.clone()
    sprite_rows = []
    for s in range(K):
        wobble(sbase, st_rows, s)
        sprite_rows.append(st_rows.cpu().numpy().copy())
    res["a_workload"] = f"sprites {len(owner) // 4} markers, {ss.n_draw_objects} draw objects, {len(owner)} transform rows, {SIZE}x{SIZE} MSAA16"

    packed = resolve(scenes.paris_like(30000, SIZE, 30000).encoding)
    pbase = transforms(packed)
    paris_rows = [rotation_rows(pbase, s) for s in range(K)]
    all_paris = torch.from_numpy(np.stack(paris_rows)).cuda()
    pt = all_paris[0].clone()
    res["b_workload"] = f"paris-like-30k {SIZE}x{SIZE} MSAA16, {packed.layout.n_paths} paths, {len(pbase)} transform rows"

    r = Renderer()
    st = torch.cuda.ExternalStream(r.stream)
    if args.profile:
        r.upload(spacked)
        r.bind_transforms(st_rows)

        def aframe(s):
            with torch.cuda.stream(st):
                wobble(sbase, st_rows, s)
            r.render_resident(p)

        for s in range(3):
            aframe(s)
        res["a_k_bound_transforms_us"] = kernel_us(aframe, 20)
        r.upload(packed)
        r.bind_transforms(pt)

        def bframe(s):
            with torch.cuda.stream(st):
                pt.copy_(all_paris[s % K])
            r.render_resident(p)

        for s in range(3):
            bframe(s)
        res["b_k_bound_transforms_us"] = kernel_us(bframe, 20)
        r.close()
    else:
        rc = Renderer()
        # (a)
        r.upload(spacked)
        res["a_resident_unbound"] = timed(args.steps, args.warmup, lambda s: r.render_resident(p))
        res["a_resident_unbound"]["launches"] = int(r.render_resident(p).kernel_launches)
        r.bind_transforms(st_rows)
        res["a_bound"] = bound_route(r, st_rows, p, lambda s: wobble(sbase, st_rows, s), args.steps, args.warmup)
        img_b = r.download_target(p)
        res["a_host"] = host_route(rc, spacked, p, lambda s: sprite_rows[s % K], args.steps, args.warmup)
        res["a_parity_last_timed_frame"] = parity(img_b, rc.download_target(p))
        # (b)
        r.upload(packed)
        res["b_resident_unbound"] = timed(args.steps, args.warmup, lambda s: r.render_resident(p))
        res["b_resident_unbound"]["launches"] = int(r.render_resident(p).kernel_launches)
        r.bind_transforms(pt)
        res["b_bound"] = bound_route(r, pt, p, lambda s: pt.copy_(all_paris[s % K]), args.steps, args.warmup)
        img_b = r.download_target(p)
        res["b_host"] = host_route(rc, packed, p, lambda s: paris_rows[s % K], args.steps, args.warmup)
        res["b_parity_last_timed_frame"] = parity(img_b, rc.download_target(p))
        rc.close()
        # (c) 1 % of the markers move per frame, damage-tracked into a device destination
        n_markers = len(owner) // 4
        m = max(1, n_markers // 100)
        g = np.random.default_rng(7)
        picks = []
        for _ in range(K):
            mk = g.choice(n_markers, m, replace=False)
            picks.append(torch.from_numpy((4 * mk[:, None] + np.arange(4)[None]).reshape(-1)).cuda())
        r.upload(spacked)
        st_rows.copy_(sbase)
        r.bind_transforms(st_rows)
        dst = torch.zeros((SIZE, SIZE, 4), dtype=torch.uint8, device="cuda")
        r.set_damage_tracking(True)

        def damage_step(s):
            wobble(sbase, st_rows, s, picks[s % K])

        res["c_bound_damage"] = bound_route(r, st_rows, p, damage_step, args.steps, args.warmup, dst.data_ptr())
        damaged = []
        for s in range(K):  # the damage of further frames, outside the timed ones (vb_last_damage synchronises)
            with torch.cuda.stream(st):
                damage_step(s)
            r.render_resident(p, dst.data_ptr())
            damaged.append(int(r.last_damage().sum()))
        rows_now = st_rows.cpu().numpy()
        rf = Renderer()
        full = spacked.scene.copy()
        L = spacked.layout
        full[L.transform_base:L.style_base] = rows_now.reshape(-1).view(np.uint32)
        rf.upload(type(spacked)(full, L, spacked.ramps, spacked.atlas))
        rf.render_resident(p)
        res["c_parity_with_full_host_frame"] = parity(dst.cpu().numpy(), rf.download_target(p))
        rf.close()
        tiles = ((SIZE + 15) // 16) ** 2
        res["c_bound_damage"].update(markers_moving=m, damaged_tiles_mean=round(float(np.mean(damaged)), 1), tiles=tiles)
        r.set_damage_tracking(False)
        r.close()
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "transform_probe_profile.json" if args.profile else "transform_probe.json"
        with open(os.path.join(args.out, name), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
