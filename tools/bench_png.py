"""PNG encoding on the GPU (autovfx_b200.png), measured on one device.

1. Encode time of one 1080p frame's three images (rgba8, depth8 through the TURBO table, normal8) in one call: CUDA events,
   median / p10 / p90 over --reps, and the kernels per frame.
2. File sizes against PIL (torchvision's save_image path) and cv2.imwrite for the same pixels.
3. Wall clock per frame of a --frames trajectory over --gaussians Gaussians written to a temporary directory, two arms:
   FrameLoop(pack8=True, product=True) + FrameFiles, and the reference loop body (render() through FrameLoop's product frame, then
   torchvision save_image, depth2img + cv2.imwrite, np.save and the normal map's cv2.imwrite).

usage: python tools/bench_png.py [--frames 300] [--gaussians 3000000] [--reps 50] [--ref-frames 20]
Prints one JSON line.  Writes only to a temporary directory.
"""
from __future__ import annotations

import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def pct(xs):
    xs = np.asarray(xs)
    return {"median": float(np.median(xs)), "p10": float(np.percentile(xs, 10)), "p90": float(np.percentile(xs, 90))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--ref-frames", type=int, default=20)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_png: needs a CUDA device")
    import cv2
    from PIL import Image
    from autovfx_b200 import png, render_loop as RL, scene
    from autovfx_b200.renderer import TURBO_LUT_BGR
    dev = torch.device("cuda:0")
    W, H = a.width, a.height
    res = {"gpu": torch.cuda.get_device_name(dev), "host_cores": os.cpu_count()}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        res["power_limit"] = "unknown (%s)" % ex
    g = {k: v.to(dev) for k, v in scene.synthetic_gaussians(a.gaussians, seed=4).items()}
    cams = RL.pack_cameras([scene.lookat_camera((3.0 * np.cos(2 * np.pi * i / a.frames), -3.0, 0.4 + 0.2 * np.sin(2 * np.pi * i / a.frames)),
                                                (0, 0, 0), W, H, 60.0) for i in range(a.frames)])
    lut = png.turbo_lut_rgb(dev)

    # 1 + 2: one frame's three images
    loop = RL.FrameLoop(g, 3, W, H, device=dev, to_host=False, pack8=True, product=True)
    held = {}
    loop.render(cams[:1], lambda i, fr, st: held.update({k: v.clone() for k, v in fr.items()}))
    items = [held["rgba8"], (held["depth8"], lut), held["normal8"]]
    for _ in range(5):
        png.encode_pngs(items)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        png.encode_pngs(items)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    res["encode_ms_per_frame_3_images"] = pct(times)
    res["kernels_per_frame"] = 4  # k_png_filter, k_png_match, k_png_deflate, k_png_assemble for up to 16 images per call
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        png.encode_pngs(items)
        torch.cuda.synchronize()
    res["kernel_ms"] = {e.key: round(e.device_time_total / 1000.0 / max(e.count, 1), 4) for e in prof.key_averages() if e.key.startswith("_ZN3gsr") or "png" in e.key}
    buf, spans, sizes = png.encode_pngs(items)
    torch.cuda.synchronize()
    rgba, d8, n8 = held["rgba8"].cpu().numpy(), held["depth8"].cpu().numpy(), held["normal8"].cpu().numpy()
    ours = [int(s) for s in sizes.cpu()]
    pil = []
    for img in (rgba, TURBO_LUT_BGR.numpy()[d8][:, :, ::-1], n8):
        b = io.BytesIO()
        t0 = time.perf_counter()
        Image.fromarray(np.ascontiguousarray(img)).save(b, format="PNG")
        pil.append((len(b.getvalue()), time.perf_counter() - t0))
    cv = []
    for img in (rgba[:, :, [2, 1, 0, 3]], TURBO_LUT_BGR.numpy()[d8], n8[:, :, ::-1]):
        t0 = time.perf_counter()
        ok, enc = cv2.imencode(".png", np.ascontiguousarray(img))
        cv.append((enc.size, time.perf_counter() - t0))
    res["sizes"] = {"ours": ours, "pil": [p[0] for p in pil], "cv2": [c[0] for c in cv],
                    "ratio_vs_pil": [round(o / p[0], 3) for o, p in zip(ours, pil)], "ratio_vs_cv2": [round(o / c[0], 3) for o, c in zip(ours, cv)]}
    res["host_encode_s"] = {"pil": [round(p[1], 4) for p in pil], "cv2": [round(c[1], 4) for c in cv]}

    # 3: trajectories written to disk
    with tempfile.TemporaryDirectory() as tmp:
        ff = png.FrameFiles(os.path.join(tmp, "ours"))
        loop.render(cams[:3], ff)  # warm-up
        ff.flush()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loop.render(cams, ff)
        ff.close()
        torch.cuda.synchronize()
        res["trajectory_ours_ms_per_frame"] = (time.perf_counter() - t0) * 1000.0 / a.frames
        import torchvision
        loop_f = RL.FrameLoop(g, 3, W, H, device=dev, to_host=False, product=True)
        out = os.path.join(tmp, "ref")
        for sub in ("images", "depth", "normal"):
            os.makedirs(os.path.join(out, sub), exist_ok=True)

        def ref_body(i, fr, st):  # scene_representation.py:424-438 on the rendered frame
            f = fr["frame"]
            name = "%05d" % i
            torchvision.utils.save_image(torch.cat([f[0:3], f[4:5]], 0), os.path.join(out, "images", name + ".png"))
            depth_raw = f[3].cpu().numpy().squeeze()
            np.save(os.path.join(out, "depth", name + ".npy"), depth_raw.astype(np.float32))
            d = np.clip(depth_raw / 3.0, 0.0, 1.0)
            cv2.imwrite(os.path.join(out, "depth", name + ".png"), cv2.applyColorMap((d * 255).astype(np.uint8), cv2.COLORMAP_TURBO))
            normal = fr["normal"].cpu().numpy()
            normal = ((normal + 1) / 2 * 255).astype(np.uint8)
            cv2.imwrite(os.path.join(out, "normal", name + ".png"), cv2.cvtColor(normal, cv2.COLOR_RGB2BGR))
        n_ref = min(a.ref_frames, a.frames)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loop_f.render(cams[:n_ref], ref_body)
        torch.cuda.synchronize()
        res["trajectory_reference_body_ms_per_frame"] = (time.perf_counter() - t0) * 1000.0 / n_ref
        res["trajectory_frames"] = {"ours": a.frames, "reference_body": n_ref}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
