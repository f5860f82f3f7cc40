"""Hit testing (Renderer.hit_test) on the headline frame: paris-like, 30k paths, 4096^2, MSAA16, resident. Times the hit
test of 1, 1,024, 65,536 and 10^6 uniformly random points in the frame, in the host form (numpy in, numpy out, synchronous)
and the device form (CUDA tensors in and out, enqueued on the renderer's stream), both with CUDA events around the call on
that stream, after warm-up; prints the median of --steps calls beside the frame's own device time. Also reports where the
time of a point goes: the longest draw list of a bin and the longest segment slice of a tile. Then hit maps
(Renderer.hit_map, device form): the whole 4096^2 frame and a 1024^2 sub-rectangle, beside the device form of hit_test
over the same 16.7 M pixel centres (--test-steps calls: it is slow), with a check that its answers equal the map's. Prints
the card, its power limit and SM clock first, and again after the map rows. With --out, the rows also go to
DIR/hit_probe.jsonl:
    python tools/hit_probe.py [--steps 20] [--test-steps 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.vbo import DTYPES  # noqa: E402
from vello_b200 import scenes  # noqa: E402
from vello_b200.config import AA_MSAA16, RenderParams  # noqa: E402
from vello_b200.encoding import BLACK, resolve  # noqa: E402
from vello_b200.renderer import Renderer  # noqa: E402

SIZE = 4096
COUNTS = [1, 1024, 65536, 1_000_000]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def timed(r, fn, steps, warmup=3):
    """Median device time in ms of fn() between two events on the renderer's stream."""
    st = torch.cuda.ExternalStream(r.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--test-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hit_probe: no CUDA device")
    print("card (name, power limit, SM clock, max SM clock):", card(), flush=True)
    packed = resolve(scenes.paris_like(30000, SIZE, seed=30000).encoding)
    p = RenderParams(BLACK, SIZE, SIZE, AA_MSAA16)
    r = Renderer()
    r.upload(packed)
    r.render_resident(p)
    frames = []
    for _ in range(a.steps):
        r.render_resident(p)
        frames.append(r.lib.vb_last_frame_ms(r.handle))
    frame_ms = float(np.median(frames))
    # where a point's time goes: its bin's draw list, and the slices of the tiles it walks
    hdr = r.download("bin_headers", DTYPES["bin_headers"])
    n_parts = (packed.layout.n_draw_objects + 255) // 256
    per_bin = hdr["element_count"].reshape(n_parts, -1).sum(0, dtype=np.int64)
    bump = r.download("bump", DTYPES["bump"])[0]
    starts = (~r.download("tiles", DTYPES["tiles"])[: int(bump["tile"])]["segment_count_or_ix"]).astype(np.int64)
    slices = np.diff(np.append(starts, int(bump["segments"])))
    rows = [dict(frame_ms=round(frame_ms, 3), draws=int(packed.layout.n_draw_objects), lines=int(bump["lines"]),
                 bin_list_max=int(per_bin.max()), bin_list_mean=round(float(per_bin[per_bin > 0].mean()), 1),
                 tile_slice_max=int(slices.max()), tile_slice_mean=round(float(slices[slices > 0].mean()), 2))]
    print(json.dumps(rows[0]), flush=True)
    rng = np.random.default_rng(1)
    for n in COUNTS:
        pts = (rng.random((n, 2)) * SIZE).astype(np.float32)
        out = np.empty(n, np.int32)
        host_ms = timed(r, lambda: r.hit_test(pts, out), a.steps)
        dpts = torch.from_numpy(pts).cuda()
        dout = torch.empty(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        dev_ms = timed(r, lambda: r.hit_test(dpts, dout), a.steps)
        torch.cuda.synchronize()
        same = bool((dout.cpu().numpy() == out).all())
        row = dict(points=n, host_ms=round(host_ms, 4), device_ms=round(dev_ms, 4), device_us_per_1k=round(1e3 * dev_ms / max(n / 1e3, 1e-9), 3),
                   hit_share=round(float((out >= 0).mean()), 3), device_equals_host=same)
        rows.append(row)
        print(json.dumps(row), flush=True)
    # hit maps: the whole frame and a 1024^2 sub-rectangle, against hit_test over the same pixel centres
    dmap = torch.empty((SIZE, SIZE), dtype=torch.int32, device="cuda")
    sub = (1536, 1536, 1024, 1024)
    dsub = torch.empty((sub[3], sub[2]), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    map_ms = timed(r, lambda: r.hit_map(out=dmap), a.steps)
    sub_ms = timed(r, lambda: r.hit_map(sub, out=dsub), a.steps)
    torch.cuda.synchronize()
    c = torch.arange(SIZE, dtype=torch.float32, device="cuda") + 0.5
    centres = torch.stack([c.repeat(SIZE), c.repeat_interleave(SIZE)], 1).contiguous()  # row by row
    dtest = torch.empty(SIZE * SIZE, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    test_ms = timed(r, lambda: r.hit_test(centres, dtest), a.test_steps, warmup=1)
    torch.cuda.synchronize()
    same = bool(torch.equal(dtest.view(SIZE, SIZE), dmap))
    same_sub = bool(torch.equal(dsub, dmap[sub[1]:sub[1] + sub[3], sub[0]:sub[0] + sub[2]]))
    row = dict(map=f"{SIZE}x{SIZE}", map_ms=round(map_ms, 4), map_frames=round(map_ms / frame_ms, 3),
               sub_map=f"{sub[2]}x{sub[3]}", sub_map_ms=round(sub_ms, 4), hit_test_same_centres_ms=round(test_ms, 2),
               speedup=round(test_ms / map_ms, 1), map_equals_hit_test=same, sub_map_equals_map=same_sub,
               frame_ms=round(frame_ms, 3), hit_share=round(float((dmap >= 0).float().mean()), 3))
    rows.append(row)
    print(json.dumps(row), flush=True)
    print("card after the maps (name, power limit, SM clock, max SM clock):", card(), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hit_probe.jsonl"), "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for row in rows:
                f.write(json.dumps(row) + "\n")
    r.close()


if __name__ == "__main__":
    main()
