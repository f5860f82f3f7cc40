"""Per-kernel device times of the headline frame (the scene bench.py renders, resident in HBM) under torch.profiler.

    python tools/kernel_times.py OUT_DIR [--frames 20] [--warmup 10] [--paths 30000] [--size 4096] [--seed 30000] [--aa 2]

Renders --warmup frames, then --frames frames under the profiler with CUDA activities, each after the same 256 MB L2
flush bench.py does. Prints each kernel's mean device time per frame (µs, summed over its launches in the frame) and the
frame span (first kernel start to last kernel end; kernels of concurrent streams overlap in it), with the GPU's name,
power limit and SM clock read in the same run. Writes OUT_DIR/kernel_times.json and the Chrome trace beside it.
Tracing slows the host, not the device: take frame rates from bench.py, not from here."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info(index):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)], capture_output=True,
                             text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}
    return dict(zip(["name", "power_limit", "sm_clock", "sm_clock_max"], [c.strip() for c in out.split(",")]))


def kernel_name(full):
    n = full.split("(")[0]
    return n[5:] if n.startswith("void ") else n


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--paths", type=int, default=30000)
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--seed", type=int, default=30000)
    ap.add_argument("--aa", type=int, default=2)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from vello_b200 import scenes
    from vello_b200.config import RenderParams
    from vello_b200.encoding import BLACK, resolve
    from vello_b200.renderer import Renderer, RendererOptions

    if not torch.cuda.is_available():
        sys.exit("kernel_times.py: no CUDA device")
    dev = torch.cuda.current_device()
    packed = resolve(scenes.paris_like(args.paths, args.size, args.seed).encoding)
    r = Renderer(RendererOptions(device=dev))
    r.upload(packed)
    frame = C.c_void_p()
    assert r.lib.vb_frame_alloc(r.handle, args.size * args.size * 4, C.byref(frame)) == 0
    params = RenderParams(BLACK, args.size, args.size, args.aa)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=f"cuda:{dev}")
    for _ in range(args.warmup):
        r.render_resident(params, frame.value)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.frames):
            flush.fill_(1)
            torch.cuda.synchronize()
            st = r.render_resident(params, frame.value)
            assert st.failed == 0
            torch.cuda.synchronize()
    gpu = gpu_info(dev)  # right after the profiled frames, before the clock drops at idle
    stats = st.as_dict()
    r.close()

    trace = os.path.join(args.out_dir, "kernel_times_trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        kernels = sorted((e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    frames, cur = [], None
    for e in kernels:  # the flush kernel opens each frame
        if "at::native" in e["name"]:
            cur = []
            frames.append(cur)
        elif cur is not None:
            cur.append(e)
    assert len(frames) == args.frames and all(frames), "the trace does not hold one group of kernels per frame"
    per = {}
    for fr in frames:
        for e in fr:
            k = per.setdefault(kernel_name(e["name"]), {"us": 0.0, "launches": 0})
            k["us"] += e["dur"]
            k["launches"] += 1
    n = len(frames)
    table = {k: {"us_per_frame": round(v["us"] / n, 2), "launches_per_frame": v["launches"] / n}
             for k, v in sorted(per.items(), key=lambda kv: -kv[1]["us"])}
    spans = [max(e["ts"] + e["dur"] for e in fr) - min(e["ts"] for e in fr) for fr in frames]
    out = {"workload": f"paris-like-{args.paths} {args.size}x{args.size} aa={args.aa} seed={args.seed}", "frames": n, "gpu": gpu,
           "frame_span_us": {"mean": round(sum(spans) / n, 2), "min": round(min(spans), 2), "max": round(max(spans), 2)},
           "lines": stats.get("lines"), "kernels": table}
    with open(os.path.join(args.out_dir, "kernel_times.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(f"{gpu.get('name')}, power limit {gpu.get('power_limit')}, SM clock {gpu.get('sm_clock')} (max {gpu.get('sm_clock_max')})")
    print(f"{out['workload']}: {n} frames, frame span {out['frame_span_us']['mean']} us "
          f"({out['frame_span_us']['min']}-{out['frame_span_us']['max']})")
    for k, v in table.items():
        print(f"  {v['us_per_frame']:10.2f} us  x{v['launches_per_frame']:<5g} {k}")


if __name__ == "__main__":
    main()
