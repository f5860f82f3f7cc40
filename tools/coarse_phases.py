"""Where a k_coarse CTA's time goes in the headline frame (the scene bench.py renders, resident in HBM).

    tools/mkvariant.sh coarse_phases "-DVB_COARSE_PHASES" k_coarse.cu
    VELLO_B200_LIB=$PWD/variants/coarse_phases.so python tools/coarse_phases.py OUT_DIR [--frames 20] [--paths 30000] [--size 4096]

The library must be built with -DVB_COARSE_PHASES (k_coarse.cu): every CTA then stamps %globaltimer after the barriers that
end its phases. Renders --frames frames (each after the same 256 MB L2 flush bench.py does) and reads the stamps of the last
one. Prints the median and p99 over CTAs of each phase (partitions and bin list; draw set-up and coverage loop; emission;
epilogue) and of a CTA's life, how many CTAs were resident at once (and the occupancy bound: SMs x CTAs per SM), the covered
(draw, tile) pairs per tile (mean, max), with the GPU's name, power limit and SM clock read in the same run. Writes
OUT_DIR/coarse_phases.json. The stamps add a barrier per phase: take kernel times from tools/kernel_times.py, not from here."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

PHASES = ["partitions", "coverage", "emission", "epilogue"]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--paths", type=int, default=30000)
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--seed", type=int, default=30000)
    ap.add_argument("--aa", type=int, default=2)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)

    import torch
    from kernel_times import gpu_info
    from vello_b200 import scenes
    from vello_b200.config import RenderParams
    from vello_b200.encoding import BLACK, resolve
    from vello_b200.renderer import Renderer, RendererOptions

    if not torch.cuda.is_available():
        sys.exit("coarse_phases.py: no CUDA device")
    dev = torch.cuda.current_device()
    packed = resolve(scenes.paris_like(args.paths, args.size, args.seed).encoding)
    r = Renderer(RendererOptions(device=dev))
    if not hasattr(r.lib, "vb_debug_coarse_phases"):
        sys.exit("coarse_phases.py: the library was built without -DVB_COARSE_PHASES (set VELLO_B200_LIB to such a build)")
    r.upload(packed)
    frame = C.c_void_p()
    assert r.lib.vb_frame_alloc(r.handle, args.size * args.size * 4, C.byref(frame)) == 0
    params = RenderParams(BLACK, args.size, args.size, args.aa)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=f"cuda:{dev}")
    for _ in range(args.frames):
        flush.fill_(1)
        torch.cuda.synchronize()
        st = r.render_resident(params, frame.value)
        assert st.failed == 0
    torch.cuda.synchronize()
    gpu = gpu_info(dev)

    tiles_w = (args.size + 15) // 16
    bins_w = (tiles_w + 15) // 16
    n_ctas = (2 * bins_w) * (2 * bins_w)  # one stripe: the whole frame, four quadrant CTAs per bin
    cta = np.zeros((65536, 8), dtype=np.uint64)
    per_tile = np.zeros(1 << 20, dtype=np.uint32)
    fn = r.lib.vb_debug_coarse_phases
    fn.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    assert fn(cta.ctypes.data, cta.nbytes, per_tile.ctypes.data, per_tile.nbytes) == 0
    r.close()

    rec = cta[:n_ctas].astype(np.int64)
    rec = rec[rec[:, 1] > rec[:, 0]]  # CTAs that ran to the end (none returns early in this frame)
    life = (rec[:, 1] - rec[:, 0]) / 1e3
    phase = {p: rec[:, 2 + i] / 1e3 for i, p in enumerate(PHASES)}

    def stats(v):
        return {"median_us": round(float(np.median(v)), 2), "p99_us": round(float(np.percentile(v, 99)), 2),
                "mean_us": round(float(v.mean()), 2)}

    ev = sorted([(s, 1) for s in rec[:, 0]] + [(e, -1) for e in rec[:, 1]])
    live = peak = 0
    for _, d in ev:
        live += d
        peak = max(peak, live)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    pairs = per_tile[:tiles_w * tiles_w].astype(np.float64)
    out = {"workload": f"paris-like-{args.paths} {args.size}x{args.size} aa={args.aa} seed={args.seed}", "gpu": gpu,
           "ctas": int(len(rec)), "ctas_resident_peak": int(peak), "occupancy_bound": f"{sms} SMs x 5 = {sms * 5}",
           "kernel_span_us": round(float((rec[:, 1].max() - rec[:, 0].min()) / 1e3), 2),
           "cta_life": stats(life), "phases": {p: stats(v) for p, v in phase.items()},
           "phase_share_of_cta_time": {p: round(float(v.sum() / life.sum()), 3) for p, v in phase.items()},
           "pairs_per_tile": {"mean": round(float(pairs.mean()), 2), "max": int(pairs.max())},
           "pairs_per_cta": {"mean": round(float(rec[:, 7].mean()), 1), "max": int(rec[:, 7].max())}}
    with open(os.path.join(args.out_dir, "coarse_phases.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(f"{gpu.get('name')}, power limit {gpu.get('power_limit')}, SM clock {gpu.get('sm_clock')} (max {gpu.get('sm_clock_max')})")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
