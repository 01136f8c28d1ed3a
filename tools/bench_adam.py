"""Time the trainers' optimizer step: torch.optim.Adam(l, lr=0.0, eps=1e-15).step() over a Gaussian model's param groups, three
arms alternated in one process:

  foreach  torch's default (the reference's path): seven list ops, each a pass over every tensor
  fused    torch.optim.Adam(..., fused=True): one pass, the same bytes, but not the same numbers (see autovfx_b200/csrc/gsr_adam.cu)
  library  autovfx_b200.optim.use_cuda_adam: gsr_adam_step, one pass, bit-identical to foreach

Layouts: 3DGS's GaussianModel.training_setup (xyz, f_dc, f_rest, opacity, scaling, rotation) and SuGaR's SuGaROptimizer (points,
sh_coordinates_dc, sh_coordinates_rest, all_densities, scales, quaternions), P = 3M rows, M = 16 SH coefficients per channel:
59 floats per row.  Every arm steps its own copy of the same parameters with the same fixed gradients; the xyz learning rate
changes on every step, as update_learning_rate changes it.  Per arm and layout: step time from CUDA events (median, p10, p90 after
warm-up) and the achieved bandwidth over the 28 bytes per element one pass needs (read param, grad, exp_avg, exp_avg_sq; write
param, exp_avg, exp_avg_sq).  After timing, the library arm's parameters and moments are compared bit for bit with the foreach
arm's.  --profile counts the kernels of one step per arm instead.

    python tools/bench_adam.py [--calls 20] [--warmup 5] [--gaussians 3000000] [--sh 16] [--profile]
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
from torch import nn  # noqa: E402

from tools.bench_sugar_field import event_ms, stats  # noqa: E402

BYTES_PER_ELEMENT = 7 * 4  # one pass: 4 float reads, 3 float writes


def layouts(P, M, spatial_lr_scale=5.0):
    """(name, [(group, shape, lr)]) with the trainers' learning rates."""
    xyz_lr = 0.00016 * spatial_lr_scale
    gs = [("xyz", (P, 3), xyz_lr), ("f_dc", (P, 1, 3), 0.0025), ("f_rest", (P, M - 1, 3), 0.0025 / 20.0), ("opacity", (P, 1), 0.05),
          ("scaling", (P, 3), 0.005), ("rotation", (P, 4), 0.001)]
    sugar = [("points", (P, 3), xyz_lr), ("sh_coordinates_dc", (P, 1, 3), 0.0025), ("sh_coordinates_rest", (P, M - 1, 3), 0.0025 / 20.0),
             ("all_densities", (P, 1), 0.05), ("scales", (P, 3), 0.005), ("quaternions", (P, 4), 0.001)]
    return [("3dgs", gs), ("sugar", sugar)]


def make_arms(layout, dev):
    from autovfx_b200.optim import use_cuda_adam
    g = torch.Generator().manual_seed(0)
    init = [(torch.randn(shape, generator=g)).to(dev) for _, shape, _ in layout]
    grads = [(torch.randn(shape, generator=g) * 1e-3).to(dev) for _, shape, _ in layout]
    arms = {}
    for arm in ("foreach", "fused", "library"):
        ps = [nn.Parameter(x.clone()) for x in init]
        for p, gr in zip(ps, grads):
            p.grad = gr
        opt = torch.optim.Adam([{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(ps, layout)], lr=0.0, eps=1e-15,
                               fused=True if arm == "fused" else None)
        arms[arm] = use_cuda_adam(opt) if arm == "library" else opt
    return arms


def identical(a, b):
    for ga, gb in zip(a.param_groups, b.param_groups):
        pa, pb = ga["params"][0], gb["params"][0]
        for x, y in [(pa, pb)] + [(a.state[pa][k], b.state[pb][k]) for k in ("exp_avg", "exp_avg_sq")]:
            if not torch.equal(x.detach().view(torch.int32), y.detach().view(torch.int32)):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--sh", type=int, default=16)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one step per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_adam needs a GPU"
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)
    for name, layout in layouts(args.gaussians, args.sh):
        arms = make_arms(layout, dev)
        numel = sum(p.numel() for g in arms["foreach"].param_groups for p in g["params"])
        count = {a: 0 for a in arms}

        def step(a):
            count[a] += 1  # a schedule per arm: a new xyz lr on every step, the same sequence in every arm
            arms[a].param_groups[0]["lr"] = layout[0][2] * 0.01 ** ((count[a] % 1000) / 1000.0)
            arms[a].step()

        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for arm in arms:
                step(arm)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    step(arm)
                    torch.cuda.synchronize()
                n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA" and "memcpy" not in e.key.lower()
                        and "memset" not in e.key.lower())
                print(json.dumps({"layout": name, "arm": arm, "kernels_per_step": n}), flush=True)
            del arms
            torch.cuda.empty_cache()
            continue
        times = {a: [] for a in arms}
        for _ in range(args.warmup):
            for a in arms:
                step(a)
        torch.cuda.synchronize()
        for i in range(args.calls):
            order = list(arms) if i % 2 == 0 else list(arms)[::-1]  # alternated
            for a in order:
                times[a].append(event_ms(lambda: step(a)))
        same = identical(arms["foreach"], arms["library"])
        for a, v in times.items():
            s = stats(v)
            print(json.dumps({"layout": name, "arm": a, "P": args.gaussians, "M": args.sh, "elements": numel, **s,
                              "gb_per_s_median": numel * BYTES_PER_ELEMENT / (s["median_ms"] * 1e-3) / 1e9,
                              "bytes_per_step_gb": numel * BYTES_PER_ELEMENT / 1e9,
                              **({"bit_identical_to_foreach": same} if a == "library" else {})}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
