"""Bound instance transforms (Renderer.bind_instance_transforms, vb_bind_instance_transforms) against the compose route
(vb_compose with every instance's new transform, then the frame), on compose_probe's workloads with every instance moving every
frame. Prints the card, its power limit and SM clock first, then per workload (medians of --steps frames after two warm-up
frames):
  compose_host_ms   wall time of vb_compose + vb_render_resident (blocking) on the host, the ctypes table built beforehand
  bound_host_ms     wall time of the torch op that rewrites the bound rows on vb_stream + vb_render_resident (blocking)
  bound_op_ms       the torch op's part of bound_host_ms
  plain_host_ms     wall time of vb_render_resident alone, nothing moved (the compose route's renderer, scene unchanged)
  compose_device_ms device time of vb_compose + the frame (CUDA events on vb_stream behind a spin kernel, frame enqueued)
  bound_device_ms   device time of the torch op + the frame, measured the same way
  instance_kernel_us device time of one k_instance_transforms (torch.profiler, a separate pass of --steps bound frames)
  transforms_identical  the transform words the two routes' frames read are identical in every frame
  pixels_max_diff / pixels_differing  between the two routes' frames, the largest over the frames (each route renders on its
                    own renderer)
  launches          kernel_launches of a compose-route frame and of a bound frame
Workloads: (a) 64 tiles of 470 paris-like paths on an 8 x 8 grid at 4096^2 MSAA16; (b) 10,000 instances of 16 small fragments
at 2048^2 Area. With --out the rows also go to DIR/instance_probe.jsonl:
    python tools/instance_probe.py [--steps 20] [--out DIR]"""
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
from compose_probe import Timer, card, native_paris_like, small_fragments  # noqa: E402
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK  # noqa: E402
from vello_b200.renderer import Renderer, _Instance  # noqa: E402
from vello_b200.shapes import Affine  # noqa: E402


def instance_table(ids, frag_of, rows):
    arr = (_Instance * len(rows))()
    for k, row in enumerate(rows):
        arr[k].fragment, arr[k].has_transform = ids[frag_of[k]], 1
        arr[k].transform[:] = [float(v) for v in row]
    return arr


def kernel_us(r, t, all_rows, p, steps):
    """Device time of one k_instance_transforms, from torch.profiler over `steps` bound frames."""
    from torch.profiler import ProfilerActivity, profile
    st = torch.cuda.ExternalStream(r.stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            with torch.cuda.stream(st):
                t.copy_(all_rows[s % all_rows.shape[0]])
            r.render_resident(p)
    for e in prof.key_averages():
        if "k_instance_transforms" in e.key:
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = getattr(e, "cuda_time_total", 0.0)
            return round(us / max(e.count, 1), 2)
    return None


def run(name, frags, frag_of, rows_of, w, h, aa, steps, out):
    rc, rb = Renderer(), Renderer()  # the compose route, the bound route
    ids_c = [rc.upload_fragment(f) for f in frags]
    ids_b = [rb.upload_fragment(f) for f in frags]
    n = len(frag_of)
    p = RenderParams(BLACK, w, h, aa)
    all_rows_h = np.stack([rows_of(s) for s in range(steps + 2)]).astype(np.float32)
    tables = [instance_table(ids_c, frag_of, all_rows_h[s]) for s in range(steps + 2)]
    all_rows = torch.from_numpy(all_rows_h).cuda()
    t = torch.empty((n, 6), dtype=torch.float32, device="cuda")
    t.copy_(all_rows[0])
    torch.cuda.synchronize()
    rb._check(rb.lib.vb_compose(rb.handle, tables[0], n, None, None), "vb_compose")
    rb.bind_instance_transforms(t)
    tc, tb = Timer(rc), Timer(rb)
    res = {k: [] for k in ("compose_host_ms", "bound_host_ms", "bound_op_ms", "plain_host_ms", "compose_device_ms", "bound_device_ms")}
    same_tr, max_diff, n_diff, launches = True, 0, 0, None

    def compare():
        nonlocal same_tr, max_diff, n_diff
        same_tr = same_tr and bool(np.array_equal(rc.download("transforms", np.uint32), rb.download("transforms", np.uint32)))
        d = np.abs(rc.download_target(p).astype(np.int32) - rb.download_target(p).astype(np.int32))
        max_diff, n_diff = max(max_diff, int(d.max())), max(n_diff, int((d > 0).sum()))

    for s in range(steps + 2):
        # host time of a whole blocking frame per route
        t0 = time.perf_counter()
        rc._check(rc.lib.vb_compose(rc.handle, tables[s], n, None, None), "vb_compose")
        st_c = rc.render_resident(p)
        hc = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        rc.render_resident(p)
        hp = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        with torch.cuda.stream(tb.stream):
            t.copy_(all_rows[s])
        t1 = time.perf_counter()
        st_b = rb.render_resident(p)
        hb, ho = (time.perf_counter() - t0) * 1e3, (t1 - t0) * 1e3
        launches = (int(st_c.kernel_launches), int(st_b.kernel_launches))
        # device time of the update and the frame, enqueued behind a spin kernel
        with tc:
            rc._check(rc.lib.vb_compose(rc.handle, tables[s], n, None, None), "vb_compose")
            rc.enqueue(p)
        rc.finish()
        dc = tc.ms()
        with tb:
            with torch.cuda.stream(tb.stream):
                t.copy_(all_rows[s])
            rb.enqueue(p)
        rb.finish()
        db = tb.ms()
        compare()
        if s >= 2:
            for k, v in (("compose_host_ms", hc), ("bound_host_ms", hb), ("bound_op_ms", ho), ("plain_host_ms", hp), ("compose_device_ms", dc),
                         ("bound_device_ms", db)):
                res[k].append(v)
    row = {"workload": name, "instances": n, "transforms_identical": same_tr, "pixels_max_diff": max_diff, "pixels_differing": n_diff,
           "launches": launches}
    row.update({k: round(float(np.median(v)), 4) for k, v in res.items()})
    row["instance_kernel_us"] = kernel_us(rb, t, all_rows, p, steps)
    print(json.dumps(row), flush=True)
    if out:
        with open(os.path.join(out, "instance_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(row) + "\n")
    rb.bind_instance_transforms(None)
    for i in ids_c:
        rc.free_fragment(i)
    for i in ids_b:
        rb.free_fragment(i)
    rc.close()
    rb.close()
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
    run("a_tiles_8x8_4096_msaa16", tiles, list(range(64)),
        lambda s: np.array([Affine.translate(512 * (k % 8) + 3.25 * s, 512 * (k // 8) - 1.5 * s).coeffs for k in range(64)]),
        4096, 4096, AA_MSAA16, a.steps, a.out)
    rng = np.random.default_rng(5)
    smalls = small_fragments(rng)
    base = rng.uniform(0, 2000, (10000, 2))
    run("b_10k_instances_2048_area", smalls, [k % 16 for k in range(10000)],
        lambda s: np.array([(Affine.translate(*(base[k] + [0.7 * s, -0.4 * s])) * Affine.rotate(0.01 * s + k)).coeffs
                            for k in range(10000)]),
        2048, 2048, AA_AREA, a.steps, a.out)


if __name__ == "__main__":
    main()
