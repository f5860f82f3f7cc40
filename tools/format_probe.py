"""fine's device time into destinations of each format (vb_register_destination: RGBA8, BGRA8, RGBA8 premultiplied, RGBA16F,
RGBA32F; linear and CUDA arrays), and the cost of the route a float consumer had before float destinations existed.

For paris-like-30k at 4096^2 MSAA16 (bench.py's frame) and tiger at 1920x1080 Area: fine's time (the timing option's
stage_ms[FINE], mean over --frames frames after --warmup) into each destination, in --rounds alternating rounds. The old route
is an RGBA8 frame into a plain pointer followed by `t.float() / 255` in torch; its conversion is timed with CUDA events (it
does not give the same values: it divides the straight 8-bit bytes). `--eight-bit` measures only the destinations an
8-bit-only build accepts (plain, RGBA8 / BGRA8 linear and array), so that a parent build can be timed in alternation with
this one (VELLO_B200_LIB=... python tools/format_probe.py --eight-bit). Prints one JSON object, with the card's name, power
limit and SM clock read in the same run, and writes it to --out when given.

    python tools/format_probe.py --out format_probe.json
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
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class _Fmt(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--eight-bit", action="store_true", help="only the destinations an 8-bit-only build accepts")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from vello_b200 import scenes
    from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
    from vello_b200.encoding import BLACK, resolve
    from vello_b200.renderer import Renderer, RendererOptions

    torch.zeros(1, device="cuda")
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(_Fmt), C.c_size_t, C.c_size_t, C.c_uint]
    rt.cudaFreeArray.argtypes = [C.c_void_p]
    arrays = []

    def new_array(w, h, bits, kind):
        arr = C.c_void_p()
        assert rt.cudaMallocArray(C.byref(arr), C.byref(_Fmt(bits, bits, bits, bits, kind)), w, h, 2) == 0
        arrays.append(arr)
        return arr.value

    def linear(h, w, dtype, texel):
        """An (h, w, 4) view of rows 512-byte aligned, as an allocator of pitched images gives them."""
        pitch = (w * texel + 511) // 512 * 512
        big = torch.empty((h, pitch // (texel // 4)), dtype=dtype, device="cuda")
        return torch.as_strided(big, (h, w, 4), (pitch // (texel // 4), 4, 1))

    res = {"card": card(), "frames": a.frames, "rounds": a.rounds, "configs": {}}
    configs = [("paris_like_30k_4096_msaa16", lambda: resolve(scenes.paris_like(30000, 4096).encoding), 4096, 4096, AA_MSAA16),
               ("tiger_1920x1080_area", lambda: resolve(scenes.tiger(1920, 1080).encoding), 1920, 1080, AA_AREA)]
    for name, make, w, h, aa in configs:
        r = Renderer(RendererOptions(timing=True))
        r.upload(make())
        p = RenderParams(BLACK, w, h, aa)
        plain = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        dests = {"plain": plain.data_ptr(),
                 "rgba8_linear": r.register_destination(linear(h, w, torch.uint8, 4)),
                 "bgra8_linear": r.register_destination(linear(h, w, torch.uint8, 4), format="bgra8"),
                 "rgba8_array": r.register_destination(array=new_array(w, h, 8, 1)),
                 "bgra8_array": r.register_destination(array=new_array(w, h, 8, 1), format="bgra8")}
        if not a.eight_bit:
            dests.update({
                "rgba8_premultiplied_linear": r.register_destination(linear(h, w, torch.uint8, 4), alpha="premultiplied"),
                "rgba16f_linear": r.register_destination(linear(h, w, torch.float16, 8), format="rgba16f"),
                "rgba32f_linear": r.register_destination(linear(h, w, torch.float32, 16), format="rgba32f"),
                "rgba16f_array": r.register_destination(array=new_array(w, h, 16, 2), format="rgba16f"),
                "rgba32f_array": r.register_destination(array=new_array(w, h, 32, 2), format="rgba32f")})
        fine = {k: [] for k in dests}
        convert = []
        for _ in range(a.rounds):
            for k, out in dests.items():
                for _ in range(a.warmup):
                    r.render_resident(p, out)
                t = [r.render_resident(p, out).stage_ms[FINE] for _ in range(a.frames)]
                fine[k].append(float(np.mean(t)))
            # the old route's extra pass: the RGBA8 frame to float32 in torch
            r.render_resident(p, plain.data_ptr())
            f = plain.float() / 255
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.frames):
                f = plain.float() / 255
            e1.record()
            e1.synchronize()
            convert.append(e0.elapsed_time(e1) / a.frames)
            del f
        res["configs"][name] = {"fine_ms": fine, "fine_ms_median": {k: float(np.median(v)) for k, v in fine.items()},
                                "rgba8_then_torch_float_div_255_ms": convert,
                                "rgba8_then_torch_float_div_255_ms_median": float(np.median(convert))}
        for k, out in dests.items():
            if k != "plain":
                r.unregister_destination(out)
        r.close()
    for arr in arrays:
        rt.cudaFreeArray(arr)

    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
