"""Recompose with damage tracking (Renderer.recompose, vb_recompose): frame time after a recompose that changes a few instances,
against a full frame. Prints the card, its power limit and SM clock first, then one JSON row per case. Each case alternates
between two instance lists A and B, one recompose and one frame per step (medians of --steps steps after two warm-up steps):
  full_ms        device time of the frame after vb_compose on a renderer with tracking off (a full frame)
  tracked_ms     device time of the frame after vb_recompose on a renderer with tracking on, into one device destination
  damaged_tiles  of the last tracked frame
  compose_call_ms / recompose_call_ms  host time of the vb_compose / vb_recompose call alone (instance arrays built beforehand);
                 the difference is the matching's cost
  k_recompose_damage_us  device time per frame of the kernel (torch.profiler, a separate pass of --steps tracked steps)
  exact          the last tracked frame equals the full frame
Workloads: 10,000 unbound instances of 16 small fragments at 2048^2 MSAA16 (replace 1 / 10 / 100, insert 1 at the front,
delete 1, raise 1), and 64 paris-like tiles at 4096^2 MSAA16 (replace one tile's fragment). With --out the rows also go to
DIR/recompose_probe.jsonl:
    python tools/recompose_probe.py [--steps 20] [--out DIR]"""
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
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK  # noqa: E402
from vello_b200.renderer import Renderer, _Instance, _Layout  # noqa: E402
from vello_b200.shapes import Affine  # noqa: E402


def instance_array(ids, inst):
    arr = (_Instance * max(len(inst), 1))()
    for k, (i, t) in enumerate(inst):
        arr[k].fragment = ids[i]
        if t is not None:
            arr[k].has_transform = 1
            for c, v in enumerate(t.coeffs):
                arr[k].transform[c] = float(v)
    return arr, len(inst)


def call_ms(r, fn, arr_n):
    arr, n = arr_n
    L = _Layout()
    t0 = time.perf_counter()
    rc = getattr(r.lib, fn)(r.handle, arr, n, C.byref(L), None)
    ms = (time.perf_counter() - t0) * 1e3
    r._check(rc, fn)
    return ms


def kernel_us(step, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            step(s)
    total = 0.0
    for e in prof.key_averages():
        if "k_recompose_damage" in e.key:
            us = getattr(e, "device_time_total", None)
            total += us if us is not None else getattr(e, "cuda_time_total", 0.0)
    return round(total / steps, 2)


def emit(row, out):
    print(json.dumps(row), flush=True)
    if out:
        with open(os.path.join(out, "recompose_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(row) + "\n")


def case(name, edit, frags, a_list, b_list, size, steps, out):
    r, ref = Renderer(), Renderer()
    ids, rids = [r.upload_fragment(f) for f in frags], [ref.upload_fragment(f) for f in frags]
    p = RenderParams(BLACK, size, size, AA_MSAA16)
    dst = torch.zeros((size, size, 4), dtype=torch.uint8, device="cuda")
    lists = [(instance_array(ids, a_list), instance_array(rids, a_list)), (instance_array(ids, b_list), instance_array(rids, b_list))]
    r.set_damage_tracking(True)
    t_r, t_ref = Timer(r), Timer(ref)
    ms = {"full": [], "tracked": [], "compose_call": [], "recompose_call": []}
    call_ms(r, "vb_compose", lists[0][0])  # the base: list A, blocking frames first (they grow the arenas; an enqueued
    call_ms(ref, "vb_compose", lists[0][1])  # frame is never re-run)
    r.render_resident(p, dst.data_ptr())
    ref.render_resident(p)
    for s in range(steps + 2):
        mine, theirs = lists[(s + 1) % 2]  # B, A, B, ...
        c_ms = call_ms(ref, "vb_compose", theirs)
        with t_ref:
            ref.enqueue(p)
        ref.finish()
        full = t_ref.ms()
        rc_ms = call_ms(r, "vb_recompose", mine)
        with t_r:
            r.enqueue(p, dst.data_ptr())
        r.finish()
        tracked = t_r.ms()
        if s >= 2:
            for k, v in (("full", full), ("tracked", tracked), ("compose_call", c_ms), ("recompose_call", rc_ms)):
                ms[k].append(v)
    exact = bool((dst.cpu().numpy() == ref.download_target(p)).all())
    dmg = r.last_damage()

    def step(s):  # the same alternation
        call_ms(r, "vb_recompose", lists[(s + 1) % 2][0])
        r.render_resident(p, dst.data_ptr())

    row = {"scene": name, "edit": edit, "full_ms": round(float(np.median(ms["full"])), 4),
           "tracked_ms": round(float(np.median(ms["tracked"])), 4), "damaged_tiles": int(dmg.sum()), "tiles": int(dmg.size),
           "compose_call_ms": round(float(np.median(ms["compose_call"])), 4),
           "recompose_call_ms": round(float(np.median(ms["recompose_call"])), 4), "k_recompose_damage_us": kernel_us(step, steps),
           "exact": exact}
    emit(row, out)
    r.set_damage_tracking(False)
    r.close()
    ref.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    print(f"card: {card()}", flush=True)
    rng = np.random.default_rng(5)
    smalls = small_fragments(rng)
    n, size = 10000, 2048
    pos = rng.uniform(0, size - 20, (n, 2))
    base = [(k % 16, Affine.translate(*pos[k])) for k in range(n)]
    name = "10k_instances_2048_msaa16"
    for m in (1, 10, 100):
        ks = rng.choice(n, m, replace=False)
        b = list(base)
        for k in ks:
            b[k] = ((b[k][0] + 1) % 16, b[k][1])
        case(name, f"replace {m}", smalls, base, b, size, a.steps, a.out)
    case(name, "insert 1 at the front", smalls, base, [(3, Affine.translate(1000.5, 1000.5))] + base, size, a.steps, a.out)
    case(name, "delete 1", smalls, base, base[:4321] + base[4322:], size, a.steps, a.out)
    case(name, "raise 1", smalls, base, base[:4321] + base[4322:] + [base[4321]], size, a.steps, a.out)
    tiles = [native_paris_like(470, 512, k) for k in range(65)]
    grid = [(k, Affine.translate(512 * (k % 8), 512 * (k // 8))) for k in range(64)]
    case("a_tiles_8x8_4096_msaa16", "replace 1 tile's fragment", tiles, grid, grid[:27] + [(64, grid[27][1])] + grid[28:], 4096,
         a.steps, a.out)


if __name__ == "__main__":
    main()
