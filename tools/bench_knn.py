"""Time knn_points (gsr_knn) on SuGaR's neighbour searches, with distCUDA2 and a torch brute force for context.

Workloads (SuGaR's knn_points calls, sugar_scene/sugar_model.py):
  (a) self K = 16 on config-3 positions at 1M and 3M: the model's neighbour list and every reset_neighbors() (:233, :899);
  (b) self K = 16 on a 3M surface-like cloud: jittered points on four planes and a sphere, 10 % of them exact copies appended
      as clone densification appends them;
  (c) self K = 4 on config-3 at 3M: the initial radii (:47);
  (d) 1M queries near the surface against the 3M surface points, K = 16: get_gaussians_closest_to_samples (:1213).
distCUDA2 runs on the same clouds.  The torch brute force (chunked cdist + topk, a stand-in for pytorch3d's one-thread-per-query
kernel, which is not available here) is timed on a 65,536-query subset against all 3M points and reported per query; it is
not extrapolated to the full cloud.  Every time is CUDA events around one call after warm-up: median, p10, p90.

    python tools/bench_knn.py [--calls 10] [--warmup 3]
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


def surface_cloud(P: int, seed: int, jitter: float = 1e-3, dup_frac: float = 0.1) -> torch.Tensor:
    """[P,3] points on the floor z = 0 and two walls over [-4,4]^2 x [0,2], a tilted plane and a unit sphere, jittered along
    the normal; the last dup_frac of them are exact copies of earlier points."""
    g = torch.Generator().manual_seed(seed)
    n_dup = int(P * dup_frac)
    n = P - n_dup
    u = torch.rand(n, 2, generator=g)
    which = torch.randint(0, 5, (n,), generator=g)
    pts = torch.empty(n, 3)
    a, b = u[:, 0] * 8 - 4, u[:, 1] * 8 - 4
    pts[:] = torch.stack([a, b, torch.zeros(n)], dim=1)                          # floor
    m = which == 1
    pts[m] = torch.stack([torch.full_like(a[m], -4.0), a[m], u[m, 1] * 2], dim=1)   # wall x = -4
    m = which == 2
    pts[m] = torch.stack([a[m], torch.full_like(a[m], 4.0), u[m, 1] * 2], dim=1)    # wall y = 4
    m = which == 3
    pts[m] = torch.stack([a[m] * 0.5, b[m] * 0.5, 0.5 + 0.3 * a[m] * 0.5], dim=1)   # tilted plane
    m = which == 4
    z = u[m, 0] * 2 - 1
    phi = u[m, 1] * 2 * math.pi
    r = torch.sqrt(1 - z * z)
    pts[m] = torch.stack([r * torch.cos(phi) + 1.5, r * torch.sin(phi) - 1.5, z + 1.2], dim=1)  # sphere
    pts += torch.randn(n, 3, generator=g) * jitter
    dup = pts[torch.randint(0, n, (n_dup,), generator=g)]
    return torch.cat([pts, dup]).contiguous()


def timed(fn, calls: int, warmup: int) -> dict:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ms.append(s.elapsed_time(e))
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)),
            "calls": calls}


def brute_topk(q: torch.Tensor, p: torch.Tensor, K: int, chunk: int = 256):
    out = []
    for s in range(0, q.size(0), chunk):
        out.append(torch.cdist(q[s:s + chunk], p).topk(K, dim=1, largest=False).indices)
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_knn needs a GPU"
    from autovfx_b200 import scene
    from autovfx_b200.knn import distCUDA2, knn_points
    from tools.bench_train_render import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps({"card": card()}), flush=True)

    c3 = scene.config3_scene()["means3D"].to(dev)
    c1 = c3[:1_000_000].contiguous()
    surf = surface_cloud(3_000_000, seed=21).to(dev)
    near = surface_cloud(1_000_000, seed=22, jitter=0.02, dup_frac=0.0).to(dev)
    runs = [
        ("a_self_k16_config3_1M", c1, c1, 16),
        ("a_self_k16_config3_3M", c3, c3, 16),
        ("b_self_k16_surface_3M", surf, surf, 16),
        ("c_self_k4_config3_3M", c3, c3, 4),
        ("d_queries1M_k16_surface_3M", near, surf, 16),
    ]
    for name, q, p, K in runs:
        t = timed(lambda: knn_points(q[None], p[None], K=K), args.calls, args.warmup)
        print(json.dumps({"workload": name, "op": "knn_points", "P1": q.size(0), "P2": p.size(0), "K": K, **t}), flush=True)
    for name, p in [("config3_1M", c1), ("config3_3M", c3), ("surface_3M", surf)]:
        t = timed(lambda: distCUDA2(p), args.calls, args.warmup)
        print(json.dumps({"workload": name, "op": "distCUDA2", "P": p.size(0), **t}), flush=True)

    # torch brute-force stand-in: 65,536 queries of config-3 against all 3M points, 16 calls of 4,096 queries
    sub = c3[torch.randperm(c3.size(0), generator=torch.Generator().manual_seed(3))[:65_536].to(dev)]
    calls = [sub[i:i + 4096] for i in range(0, 65_536, 4096)]
    it = iter(range(10 ** 9))
    t = timed(lambda: brute_topk(calls[next(it) % len(calls)], c3, 16), len(calls), 1)
    per_query_us = {k.replace("_ms", "_us_per_query"): v * 1000.0 / 4096 for k, v in t.items() if k.endswith("_ms")}
    print(json.dumps({"workload": "torch_cdist_topk_standin_k16_config3_3M", "op": "cdist+topk (stand-in, measured on a 65,536-query "
                      "subset, 4,096 queries per call, not extrapolated)", "queries_per_call": 4096, "P2": c3.size(0), "K": 16,
                      "calls": len(calls), **per_query_us}), flush=True)
    # the same subset through knn_points against the same 3M points, per query, for a like-for-like rate
    t = timed(lambda: knn_points(sub[None], c3[None], K=16), args.calls, args.warmup)
    print(json.dumps({"workload": "knn_points_queries65536_k16_config3_3M", "op": "knn_points", "P1": 65_536, "P2": c3.size(0), "K": 16,
                      **t, "median_us_per_query": t["median_ms"] * 1000.0 / 65_536}), flush=True)


if __name__ == "__main__":
    main()
