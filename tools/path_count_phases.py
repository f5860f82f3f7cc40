"""Where a k_path_count CTA's time goes in the headline frame (the scene bench.py renders, resident in HBM).

    tools/mkvariant.sh path_count_phases "-DVB_PATH_COUNT_PHASES" k_path_count.cu
    VELLO_B200_LIB=$PWD/variants/path_count_phases.so python tools/path_count_phases.py OUT_DIR [--frames 20] [--paths 30000] [--size 4096]

The library must be built with -DVB_PATH_COUNT_PHASES (k_path_count.cu): every CTA then stamps %globaltimer after the
barriers that end its phases. Renders --frames frames (each after the same 256 MB L2 flush bench.py does) and reads the
stamps of the last one. Prints the median and p99 over CTAs of each phase, summed over a CTA's steps (line loads and
set-up; left-of-box backdrop; scan and seg_counts reservation; crossing phase) and of a CTA's life, how many CTAs were
resident at once, the distribution of left-of-box backdrop rows per line, with the GPU's name, power limit and SM clock
read in the same run. Writes OUT_DIR/path_count_phases.json. The stamps add barriers per phase: take kernel times
from tools/kernel_times.py, not from here."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

PHASES = ["load", "backdrop", "scan", "cross"]
ROW_BINS = 64  # PC_PH_ROWS in k_path_count.cu: the last bin counts lines of 63 rows or more


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
        sys.exit("path_count_phases.py: no CUDA device")
    dev = torch.cuda.current_device()
    packed = resolve(scenes.paris_like(args.paths, args.size, args.seed).encoding)
    r = Renderer(RendererOptions(device=dev))
    if not hasattr(r.lib, "vb_debug_path_count_phases"):
        sys.exit("path_count_phases.py: the library was built without -DVB_PATH_COUNT_PHASES (set VELLO_B200_LIB to such a build)")
    fn = r.lib.vb_debug_path_count_phases
    fn.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    r.upload(packed)
    frame = C.c_void_p()
    assert r.lib.vb_frame_alloc(r.handle, args.size * args.size * 4, C.byref(frame)) == 0
    params = RenderParams(BLACK, args.size, args.size, args.aa)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=f"cuda:{dev}")
    cta = np.zeros((65536, 8), dtype=np.uint64)
    rows = np.zeros(ROW_BINS, dtype=np.uint64)
    for f in range(args.frames):
        if f == args.frames - 1:  # clear the tables, so that they hold the last frame alone
            torch.cuda.synchronize()
            assert fn(cta.ctypes.data, cta.nbytes, rows.ctypes.data, rows.nbytes) == 0
        flush.fill_(1)
        torch.cuda.synchronize()
        st = r.render_resident(params, frame.value)
        assert st.failed == 0
    torch.cuda.synchronize()
    gpu = gpu_info(dev)
    assert fn(cta.ctypes.data, cta.nbytes, rows.ctypes.data, rows.nbytes) == 0
    n_lines = st.as_dict().get("lines")
    r.close()

    rec = cta.astype(np.int64)
    rec = rec[rec[:, 1] > rec[:, 0]]  # CTAs that ran to the end
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
    counted = rows.astype(np.float64)
    total = counted.sum()
    with_rows = counted[1:].sum()
    cum = np.cumsum(counted[1:]) / max(with_rows, 1.0)
    mean_rows = float((counted * np.arange(ROW_BINS)).sum() / max(total, 1.0))  # the last bin counted at its floor
    out = {"workload": f"paris-like-{args.paths} {args.size}x{args.size} aa={args.aa} seed={args.seed}", "gpu": gpu,
           "lines": n_lines, "ctas": int(len(rec)), "ctas_resident_peak": int(peak), "sms": sms,
           "steps_per_cta": {"mean": round(float(rec[:, 7].mean()), 2), "max": int(rec[:, 7].max())},
           "kernel_span_us": round(float((rec[:, 1].max() - rec[:, 0].min()) / 1e3), 2),
           "cta_life": stats(life), "phases": {p: stats(v) for p, v in phase.items()},
           "phase_share_of_cta_time": {p: round(float(v.sum() / life.sum()), 3) for p, v in phase.items()},
           "left_of_box_rows": {
               "lines_counted": int(total), "lines_with_rows": int(with_rows),
               "share_with_rows": round(float(with_rows / max(total, 1.0)), 4),
               "rows_total_at_least": int((counted * np.arange(ROW_BINS)).sum()), "mean_rows_per_line": round(mean_rows, 3),
               "median_rows_of_lines_with_rows": int(np.searchsorted(cum, 0.5) + 1),
               "p99_rows_of_lines_with_rows": int(np.searchsorted(cum, 0.99) + 1),
               "lines_with_63_or_more": int(counted[-1]),
               "histogram": {str(k): int(counted[k]) for k in range(ROW_BINS) if counted[k] != 0}}}
    with open(os.path.join(args.out_dir, "path_count_phases.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(f"{gpu.get('name')}, power limit {gpu.get('power_limit')}, SM clock {gpu.get('sm_clock')} (max {gpu.get('sm_clock_max')})")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
