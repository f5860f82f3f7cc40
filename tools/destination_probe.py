"""fine's device time into each kind of destination (vb_register_destination), against the copy a presenter needs without them.

For paris-like-30k at 4096^2 MSAA16 (bench.py's frame) and tiger at 1920x1080 Area: fine's time (the timing option's
stage_ms[FINE], mean over --frames frames after warm-up) into a plain pointer, a pitched BGRA8 buffer, an RGBA8 array and a
BGRA8 array, in --rounds alternating rounds; the time of the copy the feature removes (cudaMemcpy2DToArrayAsync of the linear
frame into the array, events); and a damage-tracked sequence with one moving instance: the incremental frame into an array
against the incremental frame into linear memory plus the full copy (device frame time, vb_last_frame_ms). Prints one JSON
object, with the card's name and power limit read in the same run, and writes it to --out when given.

    python tools/destination_probe.py --out destination_probe.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FINE = 10  # VB_STAGE_ID_FINE


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class _Fmt(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from vello_b200 import scenes
    from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
    from vello_b200.encoding import BLACK, Color, FILL_NON_ZERO, resolve
    from vello_b200.renderer import Renderer, RendererOptions
    from vello_b200.scene_native import NativeScene
    from vello_b200.shapes import Affine, Rect

    torch.zeros(1, device="cuda")
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_Fmt), C.c_size_t, C.c_size_t, C.c_uint]
    rt.cudaFreeArray.argtypes = [C.c_void_p]
    rt.cudaMemcpy2DToArrayAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
                                            C.c_void_p]

    def new_array(w, h):
        arr = C.c_void_p()
        assert rt.cudaMallocArray(C.byref(arr), C.byref(_Fmt(8, 8, 8, 8, 1)), w, h, 2) == 0
        return arr

    def copy_ms(lin, arr, w, h, n):
        """Mean time of cudaMemcpy2DToArrayAsync of a linear w x h frame into the array (events, n copies)."""
        st = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            rt.cudaMemcpy2DToArrayAsync(arr, 0, 0, C.c_void_p(lin.data_ptr()), w * 4, w * 4, h, 3, C.c_void_p(st.cuda_stream))
        e0.record()
        for _ in range(n):
            assert rt.cudaMemcpy2DToArrayAsync(arr, 0, 0, C.c_void_p(lin.data_ptr()), w * 4, w * 4, h, 3, C.c_void_p(st.cuda_stream)) == 0
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    res = {"card": card(), "frames": a.frames, "rounds": a.rounds, "configs": {}}
    configs = [("paris_like_30k_4096_msaa16", lambda: resolve(scenes.paris_like(30000, 4096).encoding), 4096, 4096, AA_MSAA16),
               ("tiger_1920x1080_area", lambda: resolve(scenes.tiger(1920, 1080).encoding), 1920, 1080, AA_AREA)]
    for name, make, w, h, aa in configs:
        r = Renderer(RendererOptions(timing=True))
        r.upload(make())
        p = RenderParams(BLACK, w, h, aa)
        lin = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        pitch = (w * 4 + 511) // 512 * 512
        big = torch.empty((h, pitch), dtype=torch.uint8, device="cuda")
        arr_rgba, arr_bgra = new_array(w, h), new_array(w, h)
        dests = {"plain": lin.data_ptr(),
                 "pitched_bgra8": r.register_destination(torch.as_strided(big, (h, w, 4), (pitch, 4, 1)), format="bgra8"),
                 "array_rgba8": r.register_destination(array=arr_rgba.value),
                 "array_bgra8": r.register_destination(array=arr_bgra.value, format="bgra8")}
        fine = {k: [] for k in dests}
        for _ in range(a.rounds):
            for k, out in dests.items():
                for _ in range(a.warmup):
                    r.render_resident(p, out)
                t = [r.render_resident(p, out).stage_ms[FINE] for _ in range(a.frames)]
                fine[k].append(float(np.mean(t)))
        copy = [copy_ms(lin, arr_rgba, w, h, a.frames) for _ in range(a.rounds)]
        res["configs"][name] = {"fine_ms": fine, "fine_ms_median": {k: float(np.median(v)) for k, v in fine.items()},
                                "copy_to_array_ms": copy, "copy_to_array_ms_median": float(np.median(copy))}
        for k, out in dests.items():
            if k != "plain":
                r.unregister_destination(out)
        r.close()
        rt.cudaFreeArray(arr_rgba)
        rt.cudaFreeArray(arr_bgra)

    # damage-tracked sequence: 200 small instances, one of them moving each frame
    w, h, n = 1920, 1080, 200
    r = Renderer()
    frag = NativeScene()
    frag.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.8, 0.3, 0.2, 1.0), None, Rect(0, 0, 20, 14))
    fid = r.upload_fragment(frag)
    r.compose([(fid, None)] * n)
    rows = np.zeros((n, 6), np.float32)
    rows[:, 0] = rows[:, 3] = 1.0
    rows[:, 4:] = np.random.default_rng(3).uniform([0, 0], [w - 20, h - 14], (n, 2))
    t = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    r.bind_instance_transforms(t)
    r.set_damage_tracking(True)
    p = RenderParams(BLACK, w, h, AA_AREA)
    lin = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    arr = new_array(w, h)
    key = r.register_destination(array=arr.value)
    seq = {"incremental_into_array_ms": [], "incremental_into_linear_ms": [], "full_copy_ms": []}
    for _ in range(a.rounds):
        for label, out in (("incremental_into_array_ms", key), ("incremental_into_linear_ms", lin.data_ptr())):
            r.render_resident(p, out)  # full: the base of the sequence
            ms = []
            for i in range(a.frames):
                t[17, 4] = float(100 + (i % 50) * 3)
                torch.cuda.synchronize()
                r.render_resident(p, out)
                ms.append(r.lib.vb_last_frame_ms(r.handle))
            seq[label].append(float(np.mean(ms[a.warmup:])))
        seq["full_copy_ms"].append(copy_ms(lin, arr, w, h, a.frames))
    res["damage_1920x1080_one_moving_of_200"] = {k: v for k, v in seq.items()}
    res["damage_1920x1080_one_moving_of_200"]["median"] = {k: float(np.median(v)) for k, v in seq.items()}
    r.unregister_destination(key)
    r.close()
    rt.cudaFreeArray(arr)

    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
