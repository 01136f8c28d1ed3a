"""Time coarse_density's SDF-regularisation block (sugar/sugar_trainers/coarse_density.py:683-781 with its default flags; see
tests/sugar_normal_ref.py's density_block), forward + backward, with three arms alternated in one process:
  torch  the field, the projection estimate and the better-normal loss all restated in torch (SuGaR's code op for op)
  field  the field on the library (autovfx_b200.sugar_field.get_field_values), the estimate and the normal loss in torch
  cuda   the field, projection_estimate and better_normal_loss all on the library

Scene: config-3 at 3M Gaussians, knn_idx = knn_points(K = 16) (built before timing), 1M samples drawn like
sample_points_in_gaussians (uniform Gaussian choice, scale factor 1.5, fixed seed), as tools/bench_sugar_field.py draws them.
Per arm: call time (CUDA events; median, p10, p90 after warm-up) and torch.cuda.max_memory_allocated.  --profile counts the
kernels of one call per arm instead of timing.

    python tools/bench_sugar_sdf_block.py [--calls 10] [--warmup 3] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.bench_sugar_field import event_ms, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sugar_sdf_block needs a GPU"
    from autovfx_b200 import scene, sugar_field
    from autovfx_b200.knn import knn_points
    from tests import sugar_normal_ref as SN
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
        x0 = points[gidx] + (SN.sugar_ref.quaternion_to_matrix(quats[gidx]) @ (1.5 * scaling[gidx] * noise)[..., None])[..., 0]
    leaves = [t.clone().requires_grad_(True) for t in (x0, points, scaling, quats, strengths)]
    model = SN.Getters(*leaves[1:], knn)
    lib_field = sugar_field.get_field_values.__get__(model)
    arms = {  # (field on the library, estimate, normal loss)
        "torch": (False, SN.projection_estimate, SN.better_normal_loss),
        "field": (True, SN.projection_estimate, SN.better_normal_loss),
        "cuda": (True, sugar_field.projection_estimate, sugar_field.better_normal_loss),
    }

    def call(arm):
        for v in leaves:
            v.grad = None
        lib, est, nrm = arms[arm]
        if lib:
            model.get_field_values = lib_field
        else:
            model.__dict__.pop("get_field_values", None)
        SN.density_block(model, leaves[0], gidx, estimate=est, normal_loss=nrm).backward()

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for arm in arms:
            call(arm)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(arm)
                torch.cuda.synchronize()
            n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA")
            print(json.dumps({"arm": arm, "kernels_per_call": n}), flush=True)
        return

    base = torch.cuda.memory_allocated()
    times = {a: [] for a in arms}
    peak = {a: 0 for a in arms}
    for _ in range(args.warmup):
        for arm in arms:
            call(arm)
    torch.cuda.synchronize()
    for _ in range(args.calls):
        for arm in arms:  # alternated
            torch.cuda.reset_peak_memory_stats()
            times[arm].append(event_ms(lambda: call(arm)))
            peak[arm] = max(peak[arm], torch.cuda.max_memory_allocated())
    for arm in arms:
        print(json.dumps({"block": "coarse_density", "arm": arm, "N": args.samples, "P": points.shape[0], "K": 16, **stats(times[arm]),
                          "max_memory_allocated_gb": peak[arm] / 1e9, "resident_before_gb": base / 1e9}), flush=True)


if __name__ == "__main__":
    main()
