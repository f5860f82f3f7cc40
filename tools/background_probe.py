"""What backgrounds (vb_set_background) cost and what they save.

(a) fine's device time (the timing option's stage_ms[FINE], mean over --frames frames after --warmup, in --rounds alternating
    rounds) without a background and over RGBA8 and RGBA32F backgrounds, for paris-like-30k at 4096^2 MSAA16 (bench.py's
    frame) and tiger at 1920x1080 Area.
(b) A layer cache: paris-like-30k rendered once into an RGBA32F premultiplied buffer, then 1,000 markers moved by bound
    transforms every frame over it as background, against the whole scene (paris and the markers) rendered every frame.
    Frame times are host clocks around --frames synchronised frames (render_resident).
(c) Annotating 64 images of 512^2 in place (a batch over an [N, H, W, 4] background that is also the destination), against
    rendering the annotations into a separate buffer and blending them over the images in torch (premultiplied over, u8).
Prints one JSON object, with the card's name, power limit and SM clock read in the same run, and writes it to --out.

    python tools/background_probe.py --out background_probe.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FINE = 10  # VB_STAGE_ID_FINE


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from vello_b200 import scenes
    from vello_b200.config import AA_AREA, AA_MSAA16, RenderParams
    from vello_b200.encoding import BLACK, FILL_NON_ZERO, Color, Scene, resolve
    from vello_b200.renderer import Renderer, RendererOptions
    from vello_b200.shapes import Affine, Circle

    torch.zeros(1, device="cuda")
    res = {"card": card(), "fine_ms": {}, "layer_cache_ms": {}, "annotate_ms": {}}

    # (a) fine with and without a background
    r = Renderer(RendererOptions(timing=True))
    cases = {"paris30k_4096_msaa16": (scenes.paris_like(30000, 4096), 4096, 4096, AA_MSAA16),
             "tiger_1920x1080_area": (scenes.tiger(1920, 1080), 1920, 1080, AA_AREA)}
    for name, (s, w, h, aa) in cases.items():
        r.upload(resolve(s.encoding))
        p = RenderParams(BLACK, w, h, aa)
        out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        bgs = {"none": None, "rgba8": (torch.randint(0, 256, (h, w, 4), dtype=torch.uint8, device="cuda"), "rgba8"),
               "rgba32f": (torch.rand((h, w, 4), device="cuda"), "rgba32f")}
        acc = {k: [] for k in bgs}
        for _ in range(a.rounds):
            for k, bg in bgs.items():
                if bg is None:
                    r.set_background()
                else:
                    r.set_background(bg[0], format=bg[1])
                for i in range(a.warmup + a.frames):
                    st = r.render_resident(p, out.data_ptr())
                    if i >= a.warmup:
                        acc[k].append(float(st.stage_ms[FINE]))
        r.set_background()
        res["fine_ms"][name] = {k: {"mean": float(np.mean(v)), "min": float(np.min(v))} for k, v in acc.items()}
    r.close()

    # (b) a layer cache: the static layer once, the markers over it every frame
    r = Renderer()
    w = h = 4096
    paris = scenes.paris_like(30000, 4096)
    markers = Scene()
    rng = np.random.default_rng(1)
    for k in range(1000):
        markers.fill(FILL_NON_ZERO, Affine.translate(float(rng.uniform(0, w)), float(rng.uniform(0, h))), Color(0.9, 0.2, 0.1, 0.8), None,
                     Circle(0, 0, 6))
    whole = Scene()
    whole.append(paris)
    whole.append(markers)
    p = RenderParams(BLACK, w, h, AA_MSAA16)
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")

    # bound transform rows: NaN keeps a scene's own transform; the markers' entries, the last 1,000, move
    mx = torch.tensor(rng.uniform(0, w, 1000), dtype=torch.float32, device="cuda")
    my = torch.tensor(rng.uniform(0, h, 1000), dtype=torch.float32, device="cuda")

    def moving(n_xf):
        xf = torch.full((n_xf, 6), float("nan"), device="cuda")
        xf[-1000:, 0] = 1.0
        xf[-1000:, 1] = 0.0
        xf[-1000:, 2] = 0.0
        xf[-1000:, 3] = 1.0
        xf[-1000:, 5] = my
        return xf

    def timed(step):
        for _ in range(a.warmup):
            step(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(a.frames):
            step(i + 1)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / a.frames

    r.upload_scene(whole)
    xf_whole = moving(whole.n_transforms)
    r.bind_transforms(xf_whole)

    def step_whole(i):
        xf_whole[-1000:, 4] = mx + float(i % 7)
        r.render_resident(p, out.data_ptr())

    layer = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    r2 = Renderer()
    r2.upload(resolve(paris.encoding))
    key = r2.register_destination(layer, format="rgba32f", alpha="premultiplied")
    r2.render_resident(p, key)
    r2.unregister_destination(key)
    r2.upload_scene(markers)
    xf_m = moving(markers.n_transforms)
    r2.bind_transforms(xf_m)
    r2.set_background(layer, format="rgba32f", alpha="premultiplied")

    def step_cached(i):
        xf_m[-1000:, 4] = mx + float(i % 7)
        r2.render_resident(p, out.data_ptr())

    for _ in range(a.rounds):
        res["layer_cache_ms"].setdefault("whole_scene_every_frame", []).append(timed(step_whole))
        res["layer_cache_ms"].setdefault("markers_over_cached_layer", []).append(timed(step_cached))
    r2.set_background()
    r2.close()
    r.close()

    # (c) annotating a batch of images in place
    n, w, h = 64, 512, 512
    ann = []
    for k in range(n):
        s = Scene()
        for j in range(20):
            s.fill(FILL_NON_ZERO, Affine.IDENTITY, Color(0.1, 0.9, 0.2, 0.6), None, Circle(20 + 24 * j, 30 + 20 * (k % 20), 8))
        ann.append(s)
    imgs = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda")
    imgs[..., 3] = 255
    p = RenderParams(Color(0.0, 0.0, 0.0, 0.0), w, h, AA_MSAA16)
    r = Renderer()
    work = imgs.clone()
    sep = torch.empty_like(imgs)

    def step_in_place(i):
        work.copy_(imgs)
        r.set_background(work)
        r.render_batch(ann, p, out=work)

    def step_blend(i):
        work.copy_(imgs)
        r.set_background()
        r.render_batch(ann, p, out=sep)
        fg = sep.float() / 255.0
        bg = work.float() / 255.0
        a_ = fg[..., 3:]
        rgb = ((fg[..., :3] * a_ + bg[..., :3] * (1 - a_)) * 255.0 + 0.5).clamp(0, 255)
        work.copy_(torch.cat([rgb, torch.full_like(a_, 255.0)], -1).to(torch.uint8))

    # the copy of the images is common to both, and timed apart
    copy_ms = timed(lambda i: work.copy_(imgs))
    for _ in range(a.rounds):
        res["annotate_ms"].setdefault("in_place_background", []).append(timed(step_in_place) - copy_ms)
        res["annotate_ms"].setdefault("separate_buffer_and_torch_blend", []).append(timed(step_blend) - copy_ms)
    r.set_background()
    r.close()
    res["annotate_ms"]["image_copy_subtracted"] = copy_ms

    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
