"""Time coarse_sdf's depth-map SDF estimate: the torch stretch (coarse_sdf.py:650-712, restated op for op in
tests/sugar_depth_ref.py) against autovfx_b200.sugar_field's close_to_surface_mask + depth_sdf_estimation_loss, forward and
backward, and the whole SDF block on the library, arms alternated in one process.

Scene: config-3 at 3M Gaussians, knn_idx = knn_points(K = 16) (built before timing), a 1080p depth map read as the first channel
of an [H, W, 3] render (a leaf, so the depth gradient is computed), a camera 8 units in front of the scene, 1M samples.
  torch       the restated stretch: the mask over every Gaussian, then the estimate loss on fixed samples, backward
  cuda        the library's two calls on the same inputs, backward
  cuda_det    the same under torch.use_deterministic_algorithms (the fixed-order depth gradient)
  corner, corner_det  the loss alone with every sample projecting beyond the map's corner, so that the border clip sends all of
              them to one texel: the one-thread-per-texel walker's worst case
  block       mask -> sample_points_in_gaussians(mask) -> get_field_values (coarse_sdf's flags) -> depth loss -> better-normal
              loss, backward, all on the library; block_det the same under torch.use_deterministic_algorithms (the torch
              stretch cannot run there: grid_sample's CUDA backward raises)
Per arm: call time (CUDA events; median, p10, p90 after warm-up) and torch.cuda.max_memory_allocated.  --profile counts the
kernels of one call per arm instead of timing.  The card's name and power limit are read in the same run.

    python tools/bench_sugar_depth.py [--calls 20] [--warmup 3] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def stats(ms):
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)),
            "calls": len(ms)}


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sugar_depth needs a GPU"
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    from autovfx_b200 import scene, sugar_field as sf
    from autovfx_b200.knn import knn_points
    from tests import sugar_depth_ref as SD
    from tests import sugar_field_ref as SF
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)

    H, W = 1080, 1920
    g = scene.config3_scene(P=args.gaussians)
    points = g["means3D"].to(dev).contiguous()
    scaling = g["scales"].to(dev).contiguous()
    quats = torch.nn.functional.normalize(g["rotations"].to(dev), dim=-1).contiguous()
    strengths = g["opacities"].reshape(-1, 1).to(dev).contiguous()
    knn = knn_points(points[None], points[None], K=16).idx[0]
    cam = SD.gs_camera((0.0, 0.0, -8.0), (0.0, 0.0, 0.0), W, H, 1.0, device=dev)
    gen = torch.Generator().manual_seed(0)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    d = 8.0 + 0.5 * torch.sin(4 * xx) * torch.cos(3 * yy) + 0.05 * torch.rand(H, W, generator=gen)
    image = torch.stack([d, d, d], -1).to(dev).requires_grad_(True)
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats, strengths)]
    model = SF.Getters(*leaves, knn)
    model.image_height, model.image_width = H, W
    with torch.no_grad():
        mask0 = sf.close_to_surface_mask(model, cam, image[..., 0], 2.0)
        x0, _ = sf.sample_points_in_gaussians(model, args.samples, 1.5, mask=mask0)
    x = x0.clone().requires_grad_(True)
    sdf = (torch.rand(args.samples, generator=gen) * 0.5).to(dev).requires_grad_(True)
    extent = 1.0
    print(json.dumps({"close_to_surface": int(mask0.sum()), "P": points.shape[0], "N": args.samples, "H": H, "W": W}), flush=True)

    def clear():
        for v in leaves + [image, x, sdf]:
            v.grad = None

    def torch_arm():
        clear()
        SD.close_to_surface_mask(model, cam, image[..., 0].detach(), 2.0)
        SD.depth_sdf_estimation_loss(model, cam, image[..., 0], x, sdf, extent / 10., 10. * extent).backward()

    def cuda_arm():
        clear()
        sf.close_to_surface_mask(model, cam, image[..., 0].detach(), 2.0)
        sf.depth_sdf_estimation_loss(model, cam, image[..., 0], x, sdf, extent / 10., 10. * extent).backward()

    def block_arm():
        clear()
        mask = sf.close_to_surface_mask(model, cam, image[..., 0].detach(), 2.0)
        xs, gidx = sf.sample_points_in_gaussians(model, args.samples, 1.5, mask=mask)
        fields = sf.get_field_values(model, xs, gidx, return_sdf=True, density_threshold=1., density_factor=1. / 16.,
                                     return_closest_gaussian_opacities=True)
        loss = 0.2 * sf.depth_sdf_estimation_loss(model, cam, image[..., 0], xs, fields["sdf"], extent / 10., 10. * extent)
        loss = loss + 0.2 * sf.better_normal_loss(model, xs, gidx, fields["closest_gaussian_opacities"]).mean()
        loss.backward()

    # every sample beyond the map's far corner: the border clip sends all of them to one texel, the walker's worst case
    x_corner = (x0 + torch.tensor([-20.0, -20.0, 0.0], device=dev)).requires_grad_(True)

    def corner_arm():
        clear()
        x_corner.grad = None
        sf.depth_sdf_estimation_loss(model, cam, image[..., 0], x_corner, sdf, extent / 10., 10. * extent).backward()

    arms = {"torch": (torch_arm, False), "cuda": (cuda_arm, False), "cuda_det": (cuda_arm, True), "corner": (corner_arm, False),
            "corner_det": (corner_arm, True), "block": (block_arm, False), "block_det": (block_arm, True)}

    def run(name):
        fn, det = arms[name]
        torch.use_deterministic_algorithms(det)
        try:
            fn()
        finally:
            torch.use_deterministic_algorithms(False)

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name in arms:
            run(name)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(name)
                torch.cuda.synchronize()
            n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA")
            print(json.dumps({"arm": name, "kernels_per_call": n}), flush=True)
        return

    base = torch.cuda.memory_allocated()
    times = {a: [] for a in arms}
    peak = {a: 0 for a in arms}
    for _ in range(args.warmup):
        for name in arms:
            run(name)
    torch.cuda.synchronize()
    for _ in range(args.calls):
        for name in arms:  # alternated
            torch.cuda.reset_peak_memory_stats()
            times[name].append(event_ms(lambda: run(name)))
            peak[name] = max(peak[name], torch.cuda.max_memory_allocated())
    for name in arms:
        print(json.dumps({"arm": name, **stats(times[name]), "max_memory_allocated_gb": peak[name] / 1e9,
                          "resident_before_gb": base / 1e9}), flush=True)


if __name__ == "__main__":
    main()
