"""Upload diff (Renderer.set_upload_diff, vb_set_upload_diff): frame time after a re-uploaded scene with a few draw objects
edited, against a full frame. Prints the card, its power limit and SM clock first, then one JSON row per case. Each case
alternates between two packed scenes A and B, one upload and one frame per step (medians of --steps steps after two warm-up
steps):
  full_ms        device time of the frame after the upload on a renderer with tracking off (a full frame)
  diffed_ms      device time of the frame after the upload on a renderer with tracking and the diff on, into one device array
  damaged_tiles  of the last diffed frame
  diff_us        device time per step of the k_upload_* kernels (the base's records at the upload; the new records, the
                 comparisons and the tables in the frame), from torch.profiler in a separate pass of --steps steps
  exact          every diffed frame equals the full frame
Workloads: paris-like 30k at 4096^2 MSAA16 with 0, 1, 10, 100 and 1,000 paths recoloured and with every path recoloured, and
the tiger at 1920x1080 Area with 0, 1 and 10 paths recoloured. With --out the rows also go to DIR/upload_diff_probe.jsonl:
    python tools/upload_diff_probe.py [--steps 20] [--out DIR]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compose_probe import Timer, card  # noqa: E402
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, DRAWTAG_COLOR, Packed, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402


def recoloured(packed, n, rng):
    """`packed` with the colour of n of its colour fills changed (n < 0: every one)."""
    L = packed.layout
    scene = np.array(packed.scene, dtype=np.uint32)
    dt = scene[L.draw_tag_base:L.draw_tag_base + L.n_draw_objects].astype(np.int64)
    dd = np.concatenate([[0], np.cumsum((dt >> 2) & 7)])[:-1]
    cols = np.flatnonzero(dt == DRAWTAG_COLOR)
    pick = cols if n < 0 else rng.choice(cols, n, replace=False)
    words = L.draw_data_base + dd[pick]
    scene[words] = scene[words] ^ np.uint32(0x00402000)
    return Packed(scene, L, packed.ramps, packed.atlas)


def emit(row, out):
    print(json.dumps(row), flush=True)
    if out:
        with open(os.path.join(out, "upload_diff_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(row) + "\n")


def diff_us(step, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            step(s)
    total = 0.0
    for e in prof.key_averages():
        if "k_upload_" in e.key:
            us = getattr(e, "device_time_total", None)
            total += us if us is not None else getattr(e, "cuda_time_total", 0.0)
    return round(total / steps, 2)


def case(name, edit, a, b, w, h, aa, steps, out):
    r, ref = Renderer(), Renderer()
    p = RenderParams(BLACK, w, h, aa)
    dst = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    r.set_damage_tracking(True)
    r.set_upload_diff(True)
    t_r, t_ref = Timer(r), Timer(ref)
    ms = {"full": [], "diffed": []}
    exact = True
    for x in (r, ref):  # the base: blocking frames first (they grow the arenas; an enqueued frame is never re-run)
        x.upload(a)
    r.render_resident(p, dst.data_ptr())
    ref.render_resident(p)
    for x in (r, ref):  # and B once, for the arenas of both scenes
        x.upload(b)
    r.render_resident(p, dst.data_ptr())
    ref.render_resident(p)
    for s in range(steps + 2):
        sc = (a, b)[s % 2]  # A, B, A, ...
        ref.upload(sc)
        with t_ref:
            ref.enqueue(p)
        ref.finish()
        r.upload(sc)
        with t_r:
            r.enqueue(p, dst.data_ptr())
        r.finish()
        exact &= bool((dst.cpu().numpy() == ref.download_target(p)).all())
        if s >= 2:
            ms["full"].append(t_ref.ms())
            ms["diffed"].append(t_r.ms())
    dmg = r.last_damage()

    def step(s):
        r.upload((a, b)[s % 2])
        r.render_resident(p, dst.data_ptr())

    row = {"scene": name, "edit": edit, "full_ms": round(float(np.median(ms["full"])), 4), "diffed_ms": round(float(np.median(ms["diffed"])), 4),
           "damaged_tiles": int(dmg.sum()), "tiles": int(dmg.size), "diff_us": diff_us(step, steps), "exact": exact}
    emit(row, out)
    r.set_upload_diff(False)
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
    paris = resolve(scenes.paris_like(30000, 4096).encoding)
    for n in (0, 1, 10, 100, 1000, -1):
        case("paris_like_30k_4096_msaa16", "every path recoloured" if n < 0 else f"{n} paths recoloured", paris, recoloured(paris, n, rng),
             4096, 4096, AA_MSAA16, a.steps, a.out)
    tiger = resolve(scenes.tiger(1920, 1080).encoding)
    for n in (0, 1, 10):
        case("tiger_1920x1080_area", f"{n} paths recoloured", tiger, recoloured(tiger, n, rng), 1920, 1080, AA_AREA, a.steps, a.out)


if __name__ == "__main__":
    main()
