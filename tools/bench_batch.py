#!/usr/bin/env python
"""bench_batch.py -- batched rendering (vb_set_cells) against rendering the same scenes one at a time.

    python tools/bench_batch.py --n 64 [--n 1024 ...] [--steps 5] [--warmup 2]

N seeded paris-like scenes (300 paths each, seeds seed .. seed + N - 1) of one cell size are rendered scene-resident:
  batch      : one upload of the batch, vb_set_cells, vb_render_resident into an [N, H, W, 4] CUDA tensor
  sequential : for every scene, upload + vb_render_resident into its slot of a second tensor
in Area and MSAA16 (--aa picks the modes and their order). Wall clock per step; both are synchronous (vb_render_resident returns once the frame is done). The
per-cell max difference between the two outputs is reported. Prints one JSON line per N, with the GPU's name, power limit
and SM clock read in the same run (nvidia-smi).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def hardware():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, power, sm = [v.strip() for v in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm}
    except Exception:
        return {"gpu": None, "power_limit": None, "sm_clock": None}


def run(n, args, r):
    import torch
    from vello_b200 import scenes
    from vello_b200.config import RenderParams
    from vello_b200.encoding import BLACK, batch, resolve
    cell = args.cell
    ss = [scenes.paris_like(args.paths, cell, seed=args.seed + i) for i in range(n)]
    bs, offsets = batch(ss)
    packed = resolve(bs.encoding)
    singles = [resolve(s.encoding) for s in ss]
    out_b = torch.zeros((n, cell, cell, 4), dtype=torch.uint8, device="cuda")
    out_s = torch.zeros_like(out_b)
    pb, ps, cell_bytes = out_b.data_ptr(), out_s.data_ptr(), cell * cell * 4
    modes = {}
    for aa in args.aa or [0, 2]:
        name = ("Area", "MSAA8", "MSAA16")[aa]
        p = RenderParams(BLACK, cell, cell, aa)

        def sequential():
            t0 = time.perf_counter()
            for i in range(n):
                r.upload(singles[i])
                r.render_resident(p, ps + i * cell_bytes)
            return time.perf_counter() - t0

        sequential()  # sizes the arenas for every scene
        t_seq = min(sequential() for _ in range(max(1, min(args.steps, 3))))
        r.upload(packed)
        r.set_cells(offsets)
        for _ in range(max(1, args.warmup)):
            r.render_resident(p, pb)
        t0 = time.perf_counter()
        for _ in range(args.steps):
            r.render_resident(p, pb)
        t_b = (time.perf_counter() - t0) / args.steps
        d = (out_b.to(torch.int16) - out_s.to(torch.int16)).abs().amax(dim=(1, 2, 3)).cpu().numpy()
        modes[name] = {"batch_ms": round(t_b * 1e3, 3), "batch_scenes_per_s": round(n / t_b, 1),
                       "sequential_ms": round(t_seq * 1e3, 3), "sequential_scenes_per_s": round(n / t_seq, 1),
                       "ratio": round(t_seq / t_b, 2), "cell_max_diff": int(d.max()), "cells_differing": int((d > 0).sum())}
    return {"n": n, "cell": f"{cell}x{cell}", "scene": f"paris-like {args.paths} paths, seeds {args.seed}..{args.seed + n - 1}",
            "modes": modes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, action="append", help="scenes per batch (repeatable; default 64 and 1024)")
    ap.add_argument("--cell", type=int, default=256)
    ap.add_argument("--paths", type=int, default=300)
    ap.add_argument("--seed", type=int, default=30000)
    ap.add_argument("--aa", type=int, action="append", choices=[0, 1, 2], help="AA modes in the order measured (default 0 then 2)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from vello_b200.renderer import Renderer
    r = Renderer()
    hw = hardware()
    for n in args.n or [64, 1024]:
        line = run(n, args, r)
        line["hardware"] = hw
        line["timing"] = "wall clock per step, synchronous; modes in the order measured: " + ",".join(line["modes"])
        print(json.dumps(line), flush=True)
    r.close()


if __name__ == "__main__":
    main()
