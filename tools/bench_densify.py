"""Time the densification bookkeeping of 3DGS training, the reference's torch lines against the library's drop-ins
(autovfx_b200.densify), alternated in one process:

  stats    the trainer's max-radii line plus GaussianModel.add_densification_stats (train.py:163-164) against
           update_densification_stats, on a viewspace gradient [P,3], int32 radii and a visibility mask of about half the rows
  densify  densify_and_prune (gaussian_model.py:399-413 without its torch.cuda.empty_cache(), restated op for op by
           tests/densify_ref.sequential, which also carries one int64 source tag per row) against densify.densify_and_prune,
           with Adam moments on every group; about 2 % of the rows are cloned, 2 % split and 1 % pruned

Scene: P = 3M Gaussians, M = 16 SH coefficients per channel (59 floats per row), fixed seed.  Per arm: call time (CUDA events;
median, p10, p90 after warm-up) and torch.cuda.max_memory_allocated; --profile counts the kernels of one call per arm instead.

    python tools/bench_densify.py [--calls 10] [--warmup 3] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch import nn  # noqa: E402

from tools.bench_sugar_field import event_ms, stats  # noqa: E402

GROUPS = (("xyz", "_xyz"), ("f_dc", "_features_dc"), ("f_rest", "_features_rest"), ("opacity", "_opacity"), ("scaling", "_scaling"),
          ("rotation", "_rotation"))


def scene(P, M, dev):
    g = torch.Generator().manual_seed(0)
    u = torch.rand(P, generator=g)
    raw = {"xyz": torch.randn(P, 3, generator=g), "f_dc": torch.randn(P, 1, 3, generator=g), "f_rest": torch.randn(P, M - 1, 3, generator=g),
           "opacity": torch.where(u < 0.01, torch.full((P,), -6.0), torch.randn(P, generator=g).clamp(-2, 2))[:, None],
           "rotation": torch.randn(P, 4, generator=g)}
    small = torch.rand(P, generator=g) < 0.5  # percent_dense * extent = 0.01: half below (clone candidates), half above (split)
    raw["scaling"] = torch.where(small[:, None], torch.full((P, 3), -5.5), torch.full((P, 3), -4.0)) + 0.2 * torch.rand(P, 3, generator=g)
    denom = torch.randint(1, 6, (P, 1), generator=g).float()
    hot = torch.rand(P, generator=g) < 0.04  # ~4 % above max_grad: half cloned, half split
    accum = torch.where(hot[:, None], 3e-4, 1e-4) * denom
    return {k: v.to(dev).contiguous() for k, v in raw.items()}, accum.to(dev), denom.to(dev)


def model(raw, accum, denom):
    m = types.SimpleNamespace()
    for n, a in GROUPS:
        setattr(m, a, nn.Parameter(raw[n].clone()))
    m.optimizer = torch.optim.Adam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS], lr=0.0, eps=1e-15)
    for n, a in GROUPS:  # Adam state as after training steps
        p = getattr(m, a)
        m.optimizer.state[p] = {"step": torch.tensor(100.0), "exp_avg": torch.randn_like(p) * 1e-3, "exp_avg_sq": torch.rand_like(p) * 1e-6}
    m.xyz_gradient_accum, m.denom, m.max_radii2D = accum.clone(), denom.clone(), torch.zeros(accum.shape[0], device=accum.device)
    m.percent_dense = 0.01
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--sh", type=int, default=16)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_densify needs a GPU"
    from autovfx_b200 import densify
    from tests import densify_ref as DR
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)
    P = args.gaussians
    raw, accum, denom = scene(P, args.sh, dev)
    gen = torch.Generator().manual_seed(1)
    vs = torch.zeros(P, 3, device=dev, requires_grad=True)
    vs.grad = (torch.randn(P, 3, generator=gen) * 1e-4).to(dev)
    radii = torch.randint(0, 40, (P,), generator=gen, dtype=torch.int32).to(dev)
    vis = radii > 20
    st = types.SimpleNamespace(xyz_gradient_accum=torch.zeros(P, 1, device=dev), denom=torch.zeros(P, 1, device=dev),
                               max_radii2D=torch.zeros(P, device=dev))

    def stats_ref():
        with torch.no_grad():
            st.max_radii2D[vis] = torch.max(st.max_radii2D[vis], radii[vis])
            st.xyz_gradient_accum[vis] += torch.norm(vs.grad[vis, :2], dim=-1, keepdim=True)
            st.denom[vis] += 1

    def stats_lib():
        densify.update_densification_stats(st, vs, radii, vis)

    holder = {}

    def prep(arm):
        holder["m"] = model(raw, accum, denom)
        torch.cuda.synchronize()

    def densify_ref():
        m = holder["m"]
        params = {n: getattr(m, a) for n, a in GROUPS}
        moments = {n: (m.optimizer.state[p]["exp_avg"], m.optimizer.state[p]["exp_avg_sq"]) for n, p in params.items()}
        with torch.no_grad():
            holder["out"] = DR.sequential(params, moments, m.xyz_gradient_accum, m.denom, 2e-4, 0.005, 1.0, 20, 0.01, DR.build_rotation)

    def densify_lib():
        with torch.no_grad():
            densify.densify_and_prune(holder["m"], 2e-4, 0.005, 1.0, 20)
        holder["out"] = holder["m"]._xyz.shape[0]

    arms = {("stats", "reference"): (None, stats_ref), ("stats", "library"): (None, stats_lib),
            ("densify", "reference"): (prep, densify_ref), ("densify", "library"): (prep, densify_lib)}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for (what, arm), (pre, fn) in arms.items():
            for _ in range(2):
                if pre:
                    pre(arm)
                if _ == 0:
                    fn()
                    torch.cuda.synchronize()
                    continue
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn()
                    torch.cuda.synchronize()
            n = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA")
            print(json.dumps({"what": what, "arm": arm, "kernels_per_call": n}), flush=True)
        return

    times = {k: [] for k in arms}
    peak = {k: 0 for k in arms}
    for _ in range(args.warmup):
        for k, (pre, fn) in arms.items():
            if pre:
                pre(k)
            fn()
    torch.cuda.synchronize()
    for _ in range(args.calls):
        for k, (pre, fn) in arms.items():  # alternated
            if pre:
                pre(k)
            holder.pop("out", None)
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            times[k].append(event_ms(fn))
            peak[k] = max(peak[k], torch.cuda.max_memory_allocated() - base)
    for (what, arm) in arms:
        print(json.dumps({"what": what, "arm": arm, "P": P, "M": args.sh, **stats(times[(what, arm)]),
                          "peak_extra_allocated_gb": peak[(what, arm)] / 1e9}), flush=True)


if __name__ == "__main__":
    main()
