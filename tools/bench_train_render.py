"""Training-step throughput of renderer.render() with gradients: the fused frame against the two-call graph.

One step is what sugar/gaussian_splatting/train.py does per iteration with normals in the loss: render one trajectory camera,
L1 on "render", "depth" and "normal" against "pseudo_normal".detach(), loss.backward().  The fused frame is render() itself
(one rasterize_gaussians_multi call: one forward and one backward for both colour sets); the two-call graph is the same
render() built from two GaussianRasterizer calls (tests/test_gpu_fused_grads._render_two_call).  The two alternate step by
step in one process, each step timed with CUDA events after warm-up.

    python tools/bench_train_render.py --steps 40 --warmup 5 [--gaussians 3000000] [--width 1920 --height 1080]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card() -> dict:
    """Name and power limit of the GPU this process runs on (a read-only nvidia-smi query)."""
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]], capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        pass
    return info


def main():
    from autovfx_b200 import renderer, scene
    from tests.test_gpu_fused_grads import _PC, _cam, _render_two_call
    import types
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="timed steps per path")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = {k: v.to(dev) for k, v in scene.config3_scene(P=args.gaussians).items()}
    pc = _PC(g, 3)
    cams = scene.cameras_from_trajectory(scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=args.width, h=args.height,
                                                               fov_x_deg=60.0))
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    bg = torch.zeros(3, device=dev)
    gen = torch.Generator().manual_seed(0)
    gt_rgb = torch.rand(4, args.height, args.width, generator=gen).to(dev)
    gt_depth = (torch.rand(args.height, args.width, generator=gen) * 4).to(dev)
    paths = {"fused": lambda cam: renderer.render(cam, pc, pipe, bg), "two_call": lambda cam: _render_two_call(cam, pc, pipe, bg)}

    def step(path, i):
        cam = _cam(cams[i % len(cams)], dev)
        for p in (pc._xyz, pc._scales, pc._rot, pc._op, pc._shs):
            p.grad = None
        out = paths[path](cam)
        loss = (out["render"] - gt_rgb).abs().mean() + (out["depth"] - gt_depth).abs().mean() + \
            (out["normal"] - out["pseudo_normal"].detach()).abs().mean()
        loss.backward()

    for i in range(args.warmup):
        for path in paths:
            step(path, i)
    torch.cuda.synchronize()
    ms = {p: [] for p in paths}
    for i in range(args.steps):
        for path in (paths if i % 2 == 0 else list(paths)[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(path, args.warmup + i)
            b.record()
            b.synchronize()
            ms[path].append(a.elapsed_time(b))
    res = {"workload": "render() with gradients, %.1fM Gaussians SH-deg 3, %dx%d, 300-camera trajectory, L1 on render/depth/normal"
                       % (args.gaussians / 1e6, args.width, args.height), "card": card(), "steps": args.steps, "warmup": args.warmup}
    for p, v in ms.items():
        its = 1000.0 / np.asarray(v)
        res[p] = {"it_per_s_median": float(np.median(its)), "it_per_s_p10": float(np.percentile(its, 10)),
                  "it_per_s_p90": float(np.percentile(its, 90)), "ms_median": float(np.median(v))}
    res["speedup_median"] = res["fused"]["it_per_s_median"] / res["two_call"]["it_per_s_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
