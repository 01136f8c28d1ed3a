"""Training-step throughput from a model whose leaves are the RAW parameters: render() through the reference's torch activations
and get_normal, against render_raw() (activations, normals and their backward in CUDA).

One step is the one tools/bench_train_render.py times: render one trajectory camera, L1 on "render", "depth" and "normal" against
"pseudo_normal".detach(), loss.backward().  The two paths alternate step by step in one process, each step timed with CUDA events
after warm-up.  --profile instead counts, with torch.profiler, the kernels each path launches in one step (a separate run: tracing
slows the host).  --optimizer torch|library ends every step with the optimizer step train.py runs after the backward
(torch.optim.Adam(l, lr=0.0, eps=1e-15) over the six param groups with the trainer's learning rates, then the gradients set to
None): torch's default foreach Adam, or the same optimizer switched to the library's CUDA step (autovfx_b200.optim.use_cuda_adam).

    python tools/bench_train_raw.py --steps 40 --warmup 5 [--gaussians 3000000] [--width 1920 --height 1080] [--profile]
                                    [--optimizer none|torch|library]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


class RawModel:
    """The reference GaussianModel's raw leaves and activations (scene/gaussian_model.py:32-128); the getters are its torch ops."""

    def __init__(self, g):
        op = g["opacities"].clamp(1e-4, 1 - 1e-4)
        shs = g["shs"]
        raw = {"_xyz": g["means3D"], "_features_dc": shs[:, :1], "_features_rest": shs[:, 1:], "_opacity": torch.log(op / (1 - op)),
               "_scaling": torch.log(g["scales"]), "_rotation": g["rotations"]}
        for k, v in raw.items():
            setattr(self, k, v.contiguous().clone().requires_grad_(True))
        self.scaling_activation, self.opacity_activation = torch.exp, torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize
        self.active_sh_degree = self.max_sh_degree = 3

    def params(self):
        return [self._xyz, self._features_dc, self._features_rest, self._opacity, self._scaling, self._rotation]

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: s.scaling_activation(s._scaling))
    get_rotation = property(lambda s: s.rotation_activation(s._rotation))
    get_opacity = property(lambda s: s.opacity_activation(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def get_normal(self, dir_pp_normalized=None):
        from tests import wrapper_ref as WR
        n, _ = WR.flip_align_view(WR.get_minimum_axis(self.get_scaling, self.get_rotation), dir_pp_normalized)
        return n / n.norm(dim=1, keepdim=True)


def main():
    from autovfx_b200 import renderer, scene
    from tools.bench_train_render import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="timed steps per path")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one step per path instead of timing")
    ap.add_argument("--optimizer", choices=("none", "torch", "library"), default="none",
                    help="end each step with the trainer's Adam step: torch's foreach Adam or the library's CUDA step")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    pc = RawModel({k: v.to(dev) for k, v in scene.config3_scene(P=args.gaussians).items()})
    optimizer = None
    if args.optimizer != "none":  # GaussianModel.training_setup (gaussian_model.py:164-173), spatial_lr_scale 5
        lrs = (0.00016 * 5.0, 0.0025, 0.0025 / 20.0, 0.05, 0.005, 0.001)
        optimizer = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pc.params(), lrs)], lr=0.0, eps=1e-15)
        if args.optimizer == "library":
            from autovfx_b200.optim import use_cuda_adam
            use_cuda_adam(optimizer)
    cams = scene.cameras_from_trajectory(scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=args.width, h=args.height,
                                                               fov_x_deg=60.0))
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    bg = torch.zeros(3, device=dev)
    gen = torch.Generator().manual_seed(0)
    gt_rgb = torch.rand(4, args.height, args.width, generator=gen).to(dev)
    gt_depth = (torch.rand(args.height, args.width, generator=gen) * 4).to(dev)
    paths = {"render_raw": renderer.render_raw, "render": renderer.render}

    def camera(i):
        c = cams[i % len(cams)]
        return types.SimpleNamespace(FoVx=2 * math.atan(c.tanfovx), FoVy=2 * math.atan(c.tanfovy), image_height=c.image_height,
                                     image_width=c.image_width, world_view_transform=c.world_view_transform.to(dev),
                                     full_proj_transform=c.full_proj_transform.to(dev), camera_center=c.camera_center.to(dev))

    def step(path, i):
        cam = camera(i)
        for p in pc.params():
            p.grad = None
        out = paths[path](cam, pc, pipe, bg)
        loss = (out["render"] - gt_rgb).abs().mean() + (out["depth"] - gt_depth).abs().mean() + \
            (out["normal"] - out["pseudo_normal"].detach()).abs().mean()
        loss.backward()
        if optimizer is not None:
            optimizer.step()
            optimizer.zero_grad(set_to_none=True)

    for i in range(args.warmup):
        for path in paths:
            step(path, i)
    torch.cuda.synchronize()
    res = {"workload": "training step from raw parameters, %.1fM Gaussians SH-deg 3, %dx%d, 300-camera trajectory, L1 on render/depth/normal"
                       % (args.gaussians / 1e6, args.width, args.height), "optimizer": args.optimizer, "card": card()}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for path in paths:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(path, args.warmup)
                torch.cuda.synchronize()
            kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                       and "memset" not in e.name.lower()]
            res[path] = {"kernels_per_step": len(kernels), "kernel_ms": sum(e.device_time for e in kernels) / 1000.0}
        print(json.dumps(res))
        return
    ms = {p: [] for p in paths}
    for i in range(args.steps):
        for path in (paths if i % 2 == 0 else list(paths)[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(path, args.warmup + i)
            b.record()
            b.synchronize()
            ms[path].append(a.elapsed_time(b))
    res.update(steps=args.steps, warmup=args.warmup)
    for p, v in ms.items():
        its = 1000.0 / np.asarray(v)
        res[p] = {"it_per_s_median": float(np.median(its)), "it_per_s_p10": float(np.percentile(its, 10)),
                  "it_per_s_p90": float(np.percentile(its, 90)), "ms_median": float(np.median(v))}
    res["speedup_median"] = res["render_raw"]["it_per_s_median"] / res["render"]["it_per_s_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
