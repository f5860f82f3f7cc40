"""Damage tracking (Renderer.set_damage_tracking / add_damage, vb_set_damage_tracking / vb_add_damage): frame time of an
incremental frame against a full one. Prints the card, its power limit and SM clock first, then one JSON row per case (medians of
--steps frames after two warm-up frames, device time from CUDA events behind a spin kernel, frames enqueued into the renderer's
own target):
  scene 1  10,000 bound instances of 16 small fragments at 2048^2 MSAA16; per case `moving` instances get a new row each
           frame (0, 1, 10, 100, all): tracked_ms with tracking on, full_ms with it off, damaged_tiles of the last tracked frame
  scene 2  paris-like 30k paths at 4096^2 MSAA16, uploaded; per case a caller rectangle covering `tiles_pct` % of the tiles
           (1, 10, 100) is added before every tracked frame
  k_damage_us  device time per frame of the k_damage* kernels (torch.profiler, a separate pass of --steps tracked frames)
  exact    the tracked frames' pixels equal the full frames' (checked on the last frame of each case)
With --out the rows also go to DIR/damage_probe.jsonl:
    python tools/damage_probe.py [--steps 20] [--out DIR]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compose_probe import Timer, card, small_fragments  # noqa: E402
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402


def damage_us(r, step, steps):
    """Device time per frame of the k_damage* kernels, from torch.profiler over `steps` tracked frames."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            step(s)
    total = 0.0
    for e in prof.key_averages():
        if "k_damage" in e.key:
            us = getattr(e, "device_time_total", None)
            total += us if us is not None else getattr(e, "cuda_time_total", 0.0)
    return round(total / steps, 2)


def timed(r, update, p, steps):
    r.render_resident(p)  # a blocking frame first: it grows the arenas (an enqueued frame is never re-run)
    t, ms = Timer(r), []
    for s in range(steps + 2):
        with t:
            update(s)
            r.enqueue(p)
        r.finish()
        if s >= 2:
            ms.append(t.ms())
    return round(float(np.median(ms)), 4)


def emit(row, out):
    print(json.dumps(row), flush=True)
    if out:
        with open(os.path.join(out, "damage_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(row) + "\n")


def scene1(steps, out):
    n, size = 10000, 2048
    rng = np.random.default_rng(5)
    r = Renderer()
    frags = small_fragments(rng)
    ids = [r.upload_fragment(f) for f in frags]
    r.compose([(ids[k % 16], None) for k in range(n)])
    base = np.zeros((n, 6), np.float32)
    base[:, 0] = base[:, 3] = 1.0
    base[:, 4:] = rng.uniform(0, size - 20, (n, 2))
    t = torch.from_numpy(base).cuda()
    torch.cuda.synchronize()
    r.bind_instance_transforms(t)
    p = RenderParams(BLACK, size, size, AA_MSAA16)
    st = torch.cuda.ExternalStream(r.stream)
    for moving in (0, 1, 10, 100, n):
        ks = torch.from_numpy(rng.choice(n, moving, replace=False)).cuda()

        def update(s):
            if moving:
                with torch.cuda.stream(st):
                    t[ks, 4] += 0.75 if s % 2 == 0 else -0.75

        r.set_damage_tracking(False)
        full = timed(r, update, p, steps)
        want = r.download_target(p)
        r.set_damage_tracking(True)
        tracked = timed(r, update, p, steps)
        exact = bool((r.download_target(p) == want).all()) if steps % 2 == 0 else None
        dmg = r.last_damage()

        def step(s):
            update(s)
            r.render_resident(p)

        row = {"scene": "10k_bound_instances_2048_msaa16", "moving": moving, "full_ms": full, "tracked_ms": tracked,
               "damaged_tiles": int(dmg.sum()), "tiles": int(dmg.size), "exact": exact, "k_damage_us": damage_us(r, step, steps)}
        emit(row, out)
    r.set_damage_tracking(False)
    r.bind_instance_transforms(None)
    for i in ids:
        r.free_fragment(i)
    r.close()


def scene2(steps, out):
    size = 4096
    r = Renderer()
    r.upload(resolve(scenes.paris_like(30000, size, seed=1).encoding))
    p = RenderParams(BLACK, size, size, AA_MSAA16)
    tw = (size + 15) // 16
    r.set_damage_tracking(False)
    full = timed(r, lambda s: None, p, steps)
    want = r.download_target(p)
    for pct in (1, 10, 100):
        side = max(1, int(round(tw * (pct / 100.0) ** 0.5)))  # a square of side^2 ~ pct % of the tiles
        x0 = (tw - side) // 2
        rect = np.array([[x0 * 16, x0 * 16, (x0 + side) * 16, (x0 + side) * 16]], np.uint32)
        r.set_damage_tracking(True)

        def update(s):
            r.add_damage(rect)

        tracked = timed(r, update, p, steps)
        exact = bool((r.download_target(p) == want).all())
        dmg = r.last_damage()

        def step(s):
            update(s)
            r.render_resident(p)

        row = {"scene": "paris_like_30k_4096_msaa16", "tiles_pct": pct, "full_ms": full, "tracked_ms": tracked,
               "damaged_tiles": int(dmg.sum()), "tiles": int(dmg.size), "exact": exact, "k_damage_us": damage_us(r, step, steps)}
        emit(row, out)
    r.set_damage_tracking(False)
    r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    print(f"card: {card()}", flush=True)
    scene1(a.steps, a.out)
    scene2(a.steps, a.out)


if __name__ == "__main__":
    main()
