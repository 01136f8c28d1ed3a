"""Time SuGaR's SDF-regularisation field: the torch method (tests/sugar_field_ref.py, SuGaR's code restated op for op) against
autovfx_b200.sugar_field, forward + backward, alternated in one process.

Scene: config-3 at 3M Gaussians, knn_idx = knn_points(K = 16) (built before timing), 1M samples drawn like
sample_points_in_gaussians (uniform Gaussian choice, scale factor 1.5, fixed seed).  Two configurations:
  density  coarse_density's flags (return_beta, return_closest_gaussian_opacities, density_factor 1) and its density loss
  sdf      coarse_sdf / refine's flags (return_sdf, return_closest_gaussian_opacities, density_factor 1/16) and the sdf loss
Per arm: forward + backward call time (CUDA events; median, p10, p90 after warm-up) and torch.cuda.max_memory_allocated.
Then compute_density under no_grad on one 2,000,000-point pass with the indices given (coarse_mesh.py:653-662), the neighbour
search excluded.  --profile counts the kernels of one call per arm instead of timing.

    python tools/bench_sugar_field.py [--calls 10] [--warmup 3] [--profile]
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
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sugar_field needs a GPU"
    from autovfx_b200 import scene, sugar_field
    from autovfx_b200.knn import knn_points
    from tests import sugar_field_ref as SF
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)

    g = scene.config3_scene(P=args.gaussians)
    points = g["means3D"].to(dev).contiguous()
    scaling = g["scales"].to(dev).contiguous()
    quats = torch.nn.functional.normalize(g["rotations"].to(dev), dim=-1).contiguous()
    strengths = g["opacities"].reshape(-1, 1).to(dev).contiguous()
    knn = knn_points(points[None], points[None], K=16).idx[0]
    gen = torch.Generator().manual_seed(0)
    gidx = torch.randint(0, points.shape[0], (args.samples,), generator=gen).to(dev)
    noise = torch.randn(args.samples, 3, generator=gen).to(dev)
    with torch.no_grad():
        x0 = points[gidx] + (SF.quaternion_to_matrix(quats[gidx]) @ (1.5 * scaling[gidx] * noise)[..., None])[..., 0]
        est = ((x0 - points[gidx]) * SF.quaternion_to_matrix(quats[gidx])[:, :, 2]).sum(-1)  # a fixed sdf estimate
    leaves = [t.clone().requires_grad_(True) for t in (x0, points, scaling, quats, strengths)]
    model = SF.Getters(*leaves[1:], knn)
    arms = {"torch": SF.get_field_values, "cuda": sugar_field.get_field_values}
    configs = {
        "density": dict(return_sdf=False, return_beta=True, return_closest_gaussian_opacities=True, density_factor=1.0),
        "sdf": dict(return_sdf=True, return_beta=False, return_closest_gaussian_opacities=True, density_factor=1.0 / 16),
    }

    def call(arm, cfg):
        for v in leaves:
            v.grad = None
        f = arms[arm](model, leaves[0], gidx, **configs[cfg])
        if cfg == "density":
            loss = (f["density"] - torch.exp(-0.5 * est.pow(2) / f["beta"].pow(2))).abs().mean()
        else:
            loss = (f["sdf"] - est.abs()).abs().mean()
        loss.backward()

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for cfg in configs:
            for arm in arms:
                call(arm, cfg)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(arm, cfg)
                    torch.cuda.synchronize()
                n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA")
                print(json.dumps({"config": cfg, "arm": arm, "kernels_per_call": n}), flush=True)
        return

    base = torch.cuda.memory_allocated()
    for cfg in configs:
        times = {a: [] for a in arms}
        peak = {a: 0 for a in arms}
        for _ in range(args.warmup):
            for arm in arms:
                call(arm, cfg)
        torch.cuda.synchronize()
        for _ in range(args.calls):
            for arm in arms:  # alternated
                torch.cuda.reset_peak_memory_stats()
                times[arm].append(event_ms(lambda: call(arm, cfg)))
                peak[arm] = max(peak[arm], torch.cuda.max_memory_allocated())
        for arm in arms:
            print(json.dumps({"config": cfg, "arm": arm, "N": args.samples, "P": points.shape[0], "K": 16, **stats(times[arm]),
                              "max_memory_allocated_gb": peak[arm] / 1e9, "resident_before_gb": base / 1e9}), flush=True)
    for v in leaves:
        v.grad = None

    # mesh extraction: compute_density on one 2M-point pass, indices given, no grad
    M = 2_000_000
    gen = torch.Generator().manual_seed(1)
    xs = (torch.rand(M, 3, generator=gen).to(dev) * 2 - 1) * torch.tensor([4.0, 4.0, 1.0], device=dev)
    with torch.no_grad():
        idx = knn_points(xs[None], points[None], K=16).idx[0]
        times = {"torch": [], "cuda": []}
        fns = {"torch": SF.compute_density, "cuda": sugar_field.compute_density}
        for _ in range(args.warmup):
            for arm, fn in fns.items():
                fn(model, xs, idx)
        for _ in range(args.calls):
            for arm, fn in fns.items():
                times[arm].append(event_ms(lambda: fn(model, xs, idx)))
    for arm in fns:
        print(json.dumps({"config": "compute_density_no_grad", "arm": arm, "N": M, "P": points.shape[0], "K": 16, **stats(times[arm])}),
              flush=True)


if __name__ == "__main__":
    main()
