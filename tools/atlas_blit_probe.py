"""Time k_atlas_blit (k_atlas.cu) against cudaMemcpy2DAsync device-to-device, and a device image refreshed every frame through
override_image against the host round trip it replaces (download, then the device resolve of vb_scene_upload_streams).

    python tools/atlas_blit_probe.py [--reps 50] [--out atlas_blit.json]

Bytes are the copy's algorithmic traffic, 8 * sum(w * h) (read + write), over CUDA-event time of many repetitions. Prints one
JSON document with the card name and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RECT = np.dtype([("src", "<u8"), ("src_pitch", "<u8"), ("unit0", "<u8"), ("w", "<u4"), ("h", "<u4"), ("dst_x", "<u4"), ("dst_y", "<u4"),
                 ("spr", "<u4"), ("pad", "<u4")])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(torch, fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3  # seconds per repetition


def blit_vs_memcpy(torch, lib, cudart, rects_np, srcs, atlas, atlas_w, reps):
    """rects_np: RECT records without spr / unit0; srcs keep the sources alive."""
    units = 0
    for r in rects_np:
        r["spr"] = lib.vb_atlas_blit_units_per_row(int(r["w"]))
        r["unit0"] = units
        units += int(r["h"]) * int(r["spr"])
    d_rects = torch.from_numpy(rects_np.view(np.uint8).copy()).cuda()
    stream = torch.cuda.current_stream().cuda_stream
    n = len(rects_np)
    blit = lambda: lib.vb_launch_atlas_blit(C.c_void_p(d_rects.data_ptr()), n, C.c_uint64(units), C.c_void_p(atlas.data_ptr()), atlas_w,
                                            C.c_void_p(stream))

    def memcpy():
        for r in rects_np:
            dst = atlas.data_ptr() + (int(r["dst_y"]) * atlas_w + int(r["dst_x"])) * 4
            e = cudart.cudaMemcpy2DAsync(C.c_void_p(dst), C.c_size_t(atlas_w * 4), C.c_void_p(int(r["src"])), C.c_size_t(int(r["src_pitch"])),
                                         C.c_size_t(int(r["w"]) * 4), C.c_size_t(int(r["h"])), 3, C.c_void_p(stream))
            assert e == 0, e

    texels = int(sum(int(r["w"]) * int(r["h"]) for r in rects_np))
    atlas.zero_()
    blit()
    got = atlas.clone()
    atlas.zero_()
    memcpy()
    torch.cuda.synchronize()
    assert torch.equal(got, atlas), "k_atlas_blit and cudaMemcpy2DAsync disagree"
    t_blit, t_copy = timed(torch, blit, reps), timed(torch, memcpy, reps)
    gbs = lambda t: 8.0 * texels / t / 1e9
    return {"images": n, "texels": texels, "blit_us": t_blit * 1e6, "memcpy2d_us": t_copy * 1e6, "blit_GBps": gbs(t_blit),
            "memcpy2d_GBps": gbs(t_copy), "blit_share_of_3350GBps": gbs(t_blit) / 3350.0}


def refresh_vs_round_trip(torch, frames):
    """A 4096x4096 device image drawn scaled into a 1024x1024 frame, its contents new every frame."""
    from vello_b200.config import AA_AREA, RenderParams
    from vello_b200.encoding import BLACK, Image
    from vello_b200.renderer import Renderer
    from vello_b200.scene_native import NativeScene
    from vello_b200.shapes import Affine
    S, F = 4096, 1024
    p = RenderParams(BLACK, F, F, AA_AREA)
    t = torch.randint(0, 256, (S, S, 4), dtype=torch.uint8, device="cuda")
    r = Renderer()
    tex = r.register_texture(t)
    s = NativeScene()
    s.draw_image(tex, Affine.scale(F / S))
    s.upload_device(r)
    out = {}

    def new_path():
        t.add_(1)  # the producer writes the image on the device
        torch.cuda.synchronize()
        r.mark_override_image_dirty(tex)
        r.render_resident(p)

    host = torch.empty((S, S, 4), dtype=torch.uint8, pin_memory=True)
    h = NativeScene()
    h.draw_image(Image(host.numpy(), key=host.data_ptr()), Affine.scale(F / S))  # keyed: resolved from `host` itself, not a copy

    def round_trip():
        t.add_(1)
        host.copy_(t)  # download (synchronous)
        h.upload_device(r)  # vb_scene_upload_streams: the image back to the device
        r.render_resident(p)

    for name, fn in (("refresh_ms", new_path), ("round_trip_ms", round_trip)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(frames):
            fn()
        torch.cuda.synchronize()
        out[name] = (time.perf_counter() - t0) / frames * 1e3
    # both paths draw the same pixels
    s.upload_device(r)
    new_path()
    a = r.download_target(p)
    host.copy_(t)
    h.upload_device(r)
    r.render_resident(p)
    assert np.array_equal(a, r.download_target(p))
    out["kernel_launches"] = int(r.last_stats.kernel_launches)
    r.unregister_texture(tex)
    r.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from vello_b200.renderer import load_library
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    torch.zeros(1, device="cuda")
    lib = load_library()
    lib.vb_atlas_blit_units_per_row.restype = C.c_uint32
    lib.vb_atlas_blit_units_per_row.argtypes = [C.c_uint32]
    lib.vb_launch_atlas_blit.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p]
    cudart = C.CDLL("libcudart.so.12")
    cudart.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
    res = {"card": card()}
    S = 4096
    big = torch.randint(0, 256, (S, S, 4), dtype=torch.uint8, device="cuda")
    atlas = torch.zeros((S, S, 4), dtype=torch.uint8, device="cuda")
    one = np.zeros(1, RECT)
    one[0] = (big.data_ptr(), S * 4, 0, S, S, 0, 0, 0, 0)
    res["one_4096"] = blit_vs_memcpy(torch, lib, cudart, one, [big], atlas, S, a.reps)
    wide = torch.randint(0, 256, (S, S + 3, 4), dtype=torch.uint8, device="cuda")  # rows 4 bytes aligned only
    one[0] = (wide.data_ptr() + 4, (S + 3) * 4, 0, S, S, 0, 0, 0, 0)
    res["one_4096_pitched_slice"] = blit_vs_memcpy(torch, lib, cudart, one, [wide], atlas, S, a.reps)
    icons = torch.randint(0, 256, (256, 64, 64, 4), dtype=torch.uint8, device="cuda")
    small_atlas = torch.zeros((8 * 64, 2048, 4), dtype=torch.uint8, device="cuda")
    many = np.zeros(256, RECT)
    for i in range(256):
        many[i] = (icons[i].data_ptr(), 64 * 4, 0, 64, 64, (i % 32) * 64, (i // 32) * 64, 0, 0)
    res["256_of_64"] = blit_vs_memcpy(torch, lib, cudart, many, [icons], small_atlas, 2048, a.reps)
    res["frame_4096_image_1024_frame"] = refresh_vs_round_trip(torch, a.frames)
    res["card_after"] = card()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main()
