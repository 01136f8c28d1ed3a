"""Time SuGaR's sample_points_in_gaussians (sugar_model.py:757-799), forward + backward with a loss on the points, and the
coarse trainer's SDF-regularisation block with and without it, all arms alternated in one process:
  sample_torch   SuGaR's method restated op for op in torch (tests/sugar_sample_ref.py: torch.multinomial, pytorch3d's
                 quaternion_apply)
  sample_cuda    autovfx_b200.sugar_field.sample_points_in_gaussians
  block          coarse_density's block on the library (field, projection estimate, better-normal loss), called as
                 tools/bench_sugar_sdf_block.py calls it, on samples drawn before timing
  sample_block   the library's sampler, then that block: the samples carry their gradient back to the model
  sample_block_det  sample_block under torch.use_deterministic_algorithms(True): the sampler's, the field's and the normal
                 terms' backwards sum in a fixed order (gsr_sugar_*_backward_det)

Scene: config-3 at 3M Gaussians, knn_idx = knn_points(K = 16) (built before timing), a mask with about 70 % of the rows set,
1M samples, sampling_scale_factor 1.5, probabilities proportional to volume (the trainers' default).  Per arm: call time (CUDA
events; median, p10, p90 after warm-up) and torch.cuda.max_memory_allocated above the resident scene.  --profile counts the
kernels of one call per arm instead of timing.

    python tools/bench_sugar_sample.py [--calls 10] [--warmup 3] [--profile]
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
    assert torch.cuda.is_available(), "bench_sugar_sample needs a GPU"
    from autovfx_b200 import scene, sugar_field
    from autovfx_b200.knn import knn_points
    from tests import sugar_normal_ref as SN
    from tests import sugar_sample_ref as SR
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)

    g = scene.config3_scene(P=args.gaussians)
    points = g["means3D"].to(dev).contiguous()
    scaling = g["scales"].to(dev).contiguous()
    quats = torch.nn.functional.normalize(g["rotations"].to(dev), dim=-1).contiguous()
    strengths = g["opacities"].reshape(-1, 1).to(dev).contiguous()
    P, N, f = points.shape[0], args.samples, 1.5
    knn = knn_points(points[None], points[None], K=16).idx[0]
    mask = torch.rand(P, generator=torch.Generator().manual_seed(0)).to(dev) < 0.7
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats, strengths)]
    model = SN.Getters(*leaves, knn)
    model.get_field_values = sugar_field.get_field_values.__get__(model)
    torch.manual_seed(0)
    with torch.no_grad():
        x0, gidx0 = sugar_field.sample_points_in_gaussians(model, N, f, mask=mask)
    x0.requires_grad_(True)

    def block(x, gidx):
        return SN.density_block(model, x, gidx, estimate=sugar_field.projection_estimate, normal_loss=sugar_field.better_normal_loss)

    def call(arm):
        for v in leaves + [x0]:
            v.grad = None
        if arm == "sample_torch":
            x, _ = SR.sample_points_in_gaussians(model, N, f, mask=mask)
            (x * x).mean().backward()
        elif arm == "sample_cuda":
            x, _ = sugar_field.sample_points_in_gaussians(model, N, f, mask=mask)
            (x * x).mean().backward()
        elif arm == "block":
            block(x0, gidx0).backward()
        else:
            torch.use_deterministic_algorithms(arm == "sample_block_det")
            try:
                block(*sugar_field.sample_points_in_gaussians(model, N, f, mask=mask)).backward()
            finally:
                torch.use_deterministic_algorithms(False)

    arms = ("sample_torch", "sample_cuda", "block", "sample_block", "sample_block_det")
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

    torch.cuda.synchronize()
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
        print(json.dumps({"arm": arm, "N": N, "P": P, "selected": int(mask.sum()), **stats(times[arm]),
                          "peak_above_resident_gb": (peak[arm] - base) / 1e9, "resident_before_gb": base / 1e9}), flush=True)


if __name__ == "__main__":
    main()
