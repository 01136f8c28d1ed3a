"""The trainers' remaining loss terms: the reference lines in torch against the library's drop-ins, forward + backward, the two
arms alternated call by call in one process (CUDA events around each call; median, p10 and p90 after warm-up):

  depth      loss_utils.depth_loss on a 1080p render depth and an omnidata-like ground truth, half of it missing
  entropy    the coarse trainers' entropy term at 3M Gaussians, 70 % of them visible (radii > 0)
  sparsity   loss_utils.sparsity_loss at 3M Gaussians ([P, 1] opacities)
  density    coarse_density's density-mode SDF estimation loss at 1M samples (proj_mask all true, indexed as the reference does)
  sdf_step   one coarse_density SDF-phase step: render_sugar_raw at 1080p with 3M Gaussians, L1 on the image, the density-mode
             estimation loss on 1M samples, backward; the arms differ only in that term

The torch arm's boolean indexing synchronises with the host, so its time includes the wait for the queued work and the idle
device while Python issues the backward.  --profile instead counts the kernels of one call per arm with torch.profiler.

    python tools/bench_train_terms.py [--calls 20] [--warmup 3] [--profile]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_sugar_field import event_ms, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_terms needs a GPU"
    from autovfx_b200 import losses as L, renderer, scene
    from autovfx_b200.sugar_field import density_estimation_loss
    from tests import sugar_ref as SR
    from tests.test_gpu_loss_terms import torch_density, torch_depth_loss, torch_entropy, torch_sparsity_loss
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)
    gen = torch.Generator().manual_seed(0)
    H, W, P, N = args.height, args.width, args.gaussians, args.samples

    p = (1.0 + 4.0 * torch.rand(H, W, generator=gen)).to(dev)
    gt_depth = 25 * (0.3 * p + 0.2 + 0.05 * torch.randn(H, W, generator=gen).to(dev)).clamp_min(0.01)
    gt_depth[torch.rand(H, W, generator=gen).to(dev) < 0.5] = 0.0
    op = torch.sigmoid(torch.randn(P, 1, generator=gen) * 2).to(dev)
    radii = torch.where(torch.rand(P, generator=gen) < 0.7, 5, 0).to(dev, torch.int32)
    dens = torch.rand(N, generator=gen).to(dev)
    beta = (0.02 + 0.1 * torch.rand(N, generator=gen)).to(dev)
    sdf = (0.1 * torch.randn(N, generator=gen)).to(dev)

    def torch_density_masked(d, b, s):  # coarse_density.py:735-741 with proj_mask = ones_like(..., dtype=bool)
        proj_mask = torch.ones_like(s, dtype=torch.bool)
        return torch_density(d[proj_mask], b[proj_mask], s)

    terms = {
        "depth": ([p], [gt_depth], torch_depth_loss, L.depth_loss),
        "entropy": ([op], [radii], torch_entropy, L.entropy_loss),
        "sparsity": ([op], [], torch_sparsity_loss, L.sparsity_loss),
        "density": ([dens, beta, sdf], [], torch_density_masked, density_estimation_loss),
    }
    leaves = {k: [t.detach().clone().requires_grad_(True) for t in v[0]] for k, v in terms.items()}

    def term_call(name, arm):
        ins, rest, ref, lib = terms[name]
        ls = leaves[name]
        for t in ls:
            t.grad = None
        (ref if arm == "torch" else lib)(*ls, *rest).backward()

    # the SDF-phase step on a SuGaR stand-in
    g = {k: v.to(dev) for k, v in scene.config3_scene(P=P).items()}
    traj = scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=W, h=H, fov_x_deg=60.0)
    eyes = [np.asarray(f["transform_matrix"], dtype=np.float64)[:3, 3] for f in traj["frames"]]
    cams = SR.Cameras(eyes, device=dev)
    model = SR.SugarModel(g, cams, W, H, math.radians(60.0))
    params = list(model.leaves.values())
    gt_image = torch.rand(H, W, 3, generator=gen).to(dev)
    step_i = [0]

    def sdf_step(arm):
        for t in params + leaves["density"]:
            t.grad = None
        ci = step_i[0] % len(cams.p3d_cameras)
        step_i[0] += 1
        out = renderer.render_sugar_raw(model, nerf_cameras=cams, camera_indices=ci, sh_deg=3, compute_color_in_rasterizer=False,
                                        return_2d_radii=True, return_opacities=True)
        loss = (out["image"][..., :3] - gt_image).abs().mean()
        fn = torch_density_masked if arm == "torch" else density_estimation_loss
        loss = loss + 0.2 * fn(*leaves["density"])
        loss.backward()

    calls = {name: (lambda arm, name=name: term_call(name, arm)) for name in terms}
    calls["sdf_step"] = sdf_step
    arms = ("torch", "library")

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name, fn in calls.items():
            for arm in arms:
                fn(arm)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn(arm)
                    torch.cuda.synchronize()
                n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA")
                print(json.dumps({"term": name, "arm": arm, "kernels_per_call": n}), flush=True)
        return

    for name, fn in calls.items():
        for _ in range(args.warmup):
            for arm in arms:
                fn(arm)
        torch.cuda.synchronize()
        times = {a: [] for a in arms}
        for _ in range(args.calls):
            for arm in arms:  # alternated
                times[arm].append(event_ms(lambda: fn(arm)))
        for arm in arms:
            print(json.dumps({"term": name, "arm": arm, "H": H, "W": W, "P": P, "N": N, **stats(times[arm])}), flush=True)


if __name__ == "__main__":
    main()
