"""SuGaR coarse-training step throughput: SuGaR's render_image_gaussian_rasterizer as the reference writes it (two GaussianRasterizer
calls on the drop-in, the normals as torch ops: tests/sugar_ref.sugar_render_two_pass) against renderer.render_sugar and
renderer.render_sugar_raw (SuGaR's colours and opacities from the raw leaves in CUDA).

One step is a regularised step of sugar/sugar_trainers/coarse_density.py: render one trajectory camera with
compute_color_in_rasterizer=False, return_2d_radii=True, return_opacities=True; loss = L1 on the image + L1 between "normal" and
"pseudo_normal".detach() + the opacity entropy term; then the SDF branch's depth render with gradients (point_colors = view-space
depth, bg = its maximum, channel 0 of the image only) added to the loss; loss.backward().  The three arms alternate step by step in
one process, each step timed with CUDA events after warm-up.  --profile instead counts the kernels of one step per arm with
torch.profiler, and those of the model's colour graph alone (get_points_rgb once and strengths twice, forward and backward: what
render_sugar_raw replaces in a step); --frames times the no-grad frame call of sugar/render.py (return_2d_radii, the normal maps) in
frames/s.  --sh-degree 4 runs SuGaR's own storage, M = 25, at degree 4 (the model's get_points_rgb then evaluates SuGaR's degree-4
eval_sh: tests/sugar_colors_ref.py).

    python tools/bench_train_sugar.py --steps 20 --warmup 3 [--gaussians 3000000] [--width 1920 --height 1080] [--profile] [--frames]
                                      [--sh-degree 4]
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


def main():
    from autovfx_b200 import renderer, scene
    from autovfx_b200.renderer import sugar_camera
    from tests import sugar_ref as SR
    from tools.bench_train_render import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per arm")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one step per arm instead of timing")
    ap.add_argument("--frames", action="store_true", help="time the no-grad frame call instead of the training step")
    ap.add_argument("--sh-degree", type=int, default=3, choices=(3, 4), help="3: M = 16; 4: M = 25 (SuGaR's storage)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    deg = args.sh_degree
    g = {k: v.to(dev) for k, v in scene.config3_scene(P=args.gaussians).items()}  # SH degree 3: M = 16
    if deg == 4:  # nine more coefficients per channel, drawn like the degree-3 ones
        extra = torch.randn(args.gaussians, 9, 3, generator=torch.Generator().manual_seed(1)).to(dev) * 0.1
        g["shs"] = torch.cat([g["shs"], extra], 1).contiguous()
    traj = scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=args.width, h=args.height, fov_x_deg=60.0)
    eyes = [np.asarray(f["transform_matrix"], dtype=np.float64)[:3, 3] for f in traj["frames"]]
    cams = SR.Cameras(eyes, device=dev)
    if deg == 3:
        model = SR.SugarModel(g, cams, args.width, args.height, math.radians(60.0))
    else:
        from tests import sugar_colors_ref as SC
        model = SC.SugarModel4(g, cams, args.width, args.height, math.radians(60.0))
    params = list(model.leaves.values())
    arms = {"render_sugar": renderer.render_sugar, "two_pass": SR.sugar_render_two_pass, "render_sugar_raw": renderer.render_sugar_raw}
    gen = torch.Generator().manual_seed(0)
    gt = torch.rand(args.height, args.width, 3, generator=gen).to(dev)

    def step(arm, i):
        fn = arms[arm]
        for p in params:
            p.grad = None
        ci = i % len(cams.p3d_cameras)
        out = fn(model, nerf_cameras=cams, camera_indices=ci, sh_deg=deg, compute_color_in_rasterizer=False, return_2d_radii=True,
                 return_opacities=True)
        img = out["image"][..., :3]
        loss = (img - gt).abs().mean()
        loss = loss + (out["normal"] - out["pseudo_normal"].detach()).abs().mean()  # normal_loss(normal, pseudo_normal.detach())
        op = out["opacities"]
        loss = loss + 0.1 * (-op * torch.log(op + 1e-10) - (1 - op) * torch.log(1 - op + 1e-10)).mean()  # entropy regulariser
        # the SDF branch's depth render (coarse_density.py:639-648): point_colors = depth in the view, bg = max depth, [..., 0]
        wvt = sugar_camera(cams, ci, model.fov_x, model.fov_y, dev)[0]
        point_depth = (model.points @ wvt[:3, 2:3] + wvt[3, 2]).expand(-1, 3)
        max_depth = point_depth.max()
        depth = fn(model, nerf_cameras=cams, camera_indices=ci, bg_color=max_depth.detach().expand(3), sh_deg=0,
                   point_colors=point_depth)[..., 0]
        loss = loss + 0.01 * (depth / max_depth.detach()).mean()
        loss.backward()

    def frame(arm, i):
        with torch.no_grad():
            arms[arm](model, nerf_cameras=cams, camera_indices=i % len(cams.p3d_cameras), sh_deg=deg, return_2d_radii=True)

    work = frame if args.frames else step
    for i in range(args.warmup):
        for arm in arms:
            work(arm, i)
    torch.cuda.synchronize()
    res = {"workload": ("no-grad frame" if args.frames else "SuGaR coarse-density step with the SDF depth render") +
           ", %.1fM Gaussians SH-deg %d (M=%d), %dx%d, 300-camera trajectory" % (args.gaussians / 1e6, deg, (deg + 1) ** 2, args.width,
                                                                                  args.height),
           "card": card()}
    try:
        res["card"]["clocks_mhz"] = {"sm": torch.cuda.clock_rate()}
    except Exception:  # noqa: BLE001
        pass
    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        def kernels_of(fn):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            return [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                    and "memset" not in e.name.lower()]
        for arm in arms:
            kernels = kernels_of(lambda: work(arm, args.warmup))
            res[arm] = {"kernels_per_step": len(kernels), "kernel_ms": sum(e.device_time for e in kernels) / 1000.0}
            if arm == "render_sugar_raw":
                res[arm]["colour_kernels"] = sorted({e.name for e in kernels if "sugar_colors" in e.name})
        if not args.frames:  # the model's colour graph of one step, forward and backward, with its gradient seeds made beforehand
            camera_center = cams.p3d_cameras[args.warmup % len(cams.p3d_cameras)].get_camera_center()
            seeds = (torch.ones(args.gaussians, 3, device=dev), torch.ones(args.gaussians, 1, device=dev),
                     torch.ones(args.gaussians, 1, device=dev))

            def colour_graph():
                for p in params:
                    p.grad = None
                colors = model.get_points_rgb(positions=model.points, camera_centers=camera_center, sh_levels=deg + 1)
                torch.autograd.backward((colors, model.strengths.view(-1, 1), model.strengths.view(-1, 1)), seeds)
            colour_graph()
            kernels = kernels_of(colour_graph)
            res["colour_graph"] = {"kernels": len(kernels), "kernel_ms": sum(e.device_time for e in kernels) / 1000.0,
                                   "share_of_render_sugar_step": len(kernels) / res["render_sugar"]["kernels_per_step"]}
        print(json.dumps(res))
        return
    ms = {a: [] for a in arms}
    for i in range(args.steps):
        for arm in (arms if i % 2 == 0 else list(arms)[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            work(arm, args.warmup + i)
            b.record()
            b.synchronize()
            ms[arm].append(a.elapsed_time(b))
    unit = "frames_per_s" if args.frames else "it_per_s"
    res.update(steps=args.steps, warmup=args.warmup)
    for arm, v in ms.items():
        rate = 1000.0 / np.asarray(v)
        res[arm] = {unit + "_median": float(np.median(rate)), unit + "_p10": float(np.percentile(rate, 10)),
                    unit + "_p90": float(np.percentile(rate, 90)), "ms_median": float(np.median(v))}
    res["speedup_median"] = res["render_sugar"][unit + "_median"] / res["two_pass"][unit + "_median"]
    res["raw_over_render_sugar_median"] = res["render_sugar_raw"][unit + "_median"] / res["render_sugar"][unit + "_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
