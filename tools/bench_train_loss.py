"""The trainers' per-step objective: torch's loss_utils graph against autovfx_b200.losses, alternated in one process.

The objective is train.py:98-132 with train_3dgs.sh's lambdas: (1 - 0.2) l1_loss + 0.2 (1 - ssim) on the [4,H,W] RGBA render,
0.01 normal_loss(normal, pseudo_normal.detach()) and 0.1 anisotropic_loss(get_scaling).

  default    the objective alone, forward + backward, from a render-shaped leaf, [H,W,3] normal maps and the scales of 3M
             Gaussians (exp of a raw leaf, as get_scaling); median, p10 and p90 of the timed calls, and the peak allocation of
             one call per arm.
  --profile  kernels per call per arm (torch.profiler, a separate run: tracing slows the host).
  --step     a full training step from raw parameters: render_raw + the objective + backward() + the library's Adam step, with
             the objective in torch against the library.

The algorithmic-bytes floor of the library's kernels is printed beside the measurement: a floor from bytes at the H100 SXM's
3.35 TB/s, not a measurement.

    python tools/bench_train_loss.py [--calls 40] [--warmup 5] [--gaussians 3000000] [--width 1920 --height 1080]
                                     [--profile] [--step]
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
import torch.nn.functional as F  # noqa: E402

LAMBDA_DSSIM, LAMBDA_PSEUDO_NORMAL, LAMBDA_ANISOTROPIC = 0.2, 0.01, 0.1
HBM_BYTES_PER_S = 3.35e12


# the reference's loss_utils graph (sugar/gaussian_splatting/utils/loss_utils.py), as the trainers run it
def _gaussian(window_size, sigma):
    gauss = torch.Tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)])
    return gauss / gauss.sum()


def torch_ssim(img1, img2, window_size=11):
    channel = img1.size(-3)
    w1 = _gaussian(window_size, 1.5).unsqueeze(1)
    window = w1.mm(w1.t()).float().unsqueeze(0).unsqueeze(0).expand(channel, 1, window_size, window_size).contiguous()
    window = window.to(img1.device).type_as(img1)
    pad = window_size // 2
    mu1, mu2 = F.conv2d(img1, window, padding=pad, groups=channel), F.conv2d(img2, window, padding=pad, groups=channel)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = F.conv2d(img1 * img1, window, padding=pad, groups=channel) - mu1_sq
    sigma2_sq = F.conv2d(img2 * img2, window, padding=pad, groups=channel) - mu2_sq
    sigma12 = F.conv2d(img1 * img2, window, padding=pad, groups=channel) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))).mean()


def torch_normal_loss(network_output, gt):
    n, g = F.normalize(network_output, p=2, dim=-1), F.normalize(gt, p=2, dim=-1)
    return torch.abs(n - g).mean() + 0.1 * (-torch.sum(n * g, axis=-1).mean())


def torch_anisotropic_loss(s, r=3):
    return torch.mean(torch.clamp(torch.max(s, dim=-1).values / (torch.min(s, dim=-1).values + 1e-6), min=r) - r)


def objective(arm, image, gt, normal, pseudo_normal, scaling):
    if arm == "torch":
        loss = (1.0 - LAMBDA_DSSIM) * torch.abs(image - gt).mean() + LAMBDA_DSSIM * (1.0 - torch_ssim(image, gt))
        return loss + LAMBDA_PSEUDO_NORMAL * torch_normal_loss(normal, pseudo_normal) + \
            LAMBDA_ANISOTROPIC * torch_anisotropic_loss(scaling)
    from autovfx_b200 import losses as L
    return L.photometric_loss(image, gt, LAMBDA_DSSIM) + LAMBDA_PSEUDO_NORMAL * L.normal_loss(normal, pseudo_normal) + \
        LAMBDA_ANISOTROPIC * L.anisotropic_loss(scaling)


def floor_bytes(H, W, P):
    """Algorithmic bytes of the library's objective, forward + backward, from shapes (float32):
    photometric: forward reads both images and writes the three SSIM maps, backward reads the maps and both images and writes dx;
    normal: forward reads both [H,W,3] maps, backward reads them again and writes d normal; anisotropic: forward reads the [P,3]
    scales, backward reads them and writes d scales.  Halo re-reads are assumed to hit L2."""
    img = 4 * H * W * 4
    nrm = H * W * 3 * 4
    sc = P * 3 * 4
    parts = {"photometric": (2 + 3) * img + (3 + 2 + 1) * img, "normal": 2 * nrm + 3 * nrm, "anisotropic": sc + 2 * sc}
    parts["total"] = sum(parts.values())
    return parts


def _stats(ms):
    v = np.asarray(ms)
    return {"ms_median": float(np.median(v)), "ms_p10": float(np.percentile(v, 10)), "ms_p90": float(np.percentile(v, 90))}


def _timed(fn, arms, calls, warmup):
    for i in range(warmup):
        for arm in arms:
            fn(arm, i)
    torch.cuda.synchronize()
    ms = {a: [] for a in arms}
    for i in range(calls):
        for arm in (arms if i % 2 == 0 else arms[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(arm, warmup + i)
            b.record()
            b.synchronize()
            ms[arm].append(a.elapsed_time(b))
    return ms


def _profile(fn, arms, i):
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for arm in arms:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(arm, i)
            torch.cuda.synchronize()
        kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower()]
        res[arm] = {"kernels": len(kernels), "kernel_ms": sum(e.device_time for e in kernels) / 1000.0}
    return res


def main():
    from autovfx_b200 import scene
    from tools.bench_train_render import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40, help="timed calls (or steps) per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one call per arm instead of timing")
    ap.add_argument("--step", action="store_true", help="time a full render_raw training step with each objective")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loss.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    H, W, P = args.height, args.width, args.gaussians
    arms = ["library", "torch"]
    gen = torch.Generator().manual_seed(0)
    gt = torch.rand(4, H, W, generator=gen).to(dev)
    res = {"card": card(), "workload": "train.py:98-132 objective (dssim 0.2, pseudo-normal 0.01, anisotropic 0.1), %.1fM Gaussians "
           "M = 16, %dx%d RGBA" % (P / 1e6, W, H)}
    fb = floor_bytes(H, W, P)
    res["floor_from_bytes_not_measured"] = {"bytes": fb, "ms_at_3.35TB/s": fb["total"] / HBM_BYTES_PER_S * 1e3}
    if not args.step:
        g = scene.config3_scene(P=P)
        scaling_raw = torch.log(g["scales"]).to(dev).requires_grad_(True)
        image = torch.rand(4, H, W, generator=gen).to(dev).requires_grad_(True)
        normal = torch.randn(H, W, 3, generator=gen).to(dev).requires_grad_(True)
        pseudo = torch.randn(3, H, W, generator=gen).to(dev).permute(1, 2, 0)  # an HWC view, as render_raw returns it

        def call(arm, i):
            for t in (image, normal, scaling_raw):
                t.grad = None
            objective(arm, image, gt, normal, pseudo, torch.exp(scaling_raw)).backward()

        res["measure"] = "objective alone, forward + backward"
        if args.profile:
            call("library", 0), call("torch", 0)
            res["profile"] = _profile(call, arms, 0)
            print(json.dumps(res))
            return
        ms = _timed(call, arms, args.calls, args.warmup)
        for arm in arms:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            call(arm, 0)
            torch.cuda.synchronize()
            res[arm] = dict(_stats(ms[arm]), peak_alloc_mb_above_inputs=(torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20)
        res["values"] = {arm: float(objective(arm, image, gt, normal, pseudo, torch.exp(scaling_raw))) for arm in arms}
    else:
        from autovfx_b200 import renderer
        from autovfx_b200.optim import use_cuda_adam
        from tools.bench_train_raw import RawModel
        pc = RawModel({k: v.to(dev) for k, v in scene.config3_scene(P=P).items()})
        lrs = (0.00016 * 5.0, 0.0025, 0.0025 / 20.0, 0.05, 0.005, 0.001)
        optimizer = use_cuda_adam(torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pc.params(), lrs)], lr=0.0, eps=1e-15))
        cams = scene.cameras_from_trajectory(scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=W, h=H, fov_x_deg=60.0))
        pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
        bg = torch.zeros(3, device=dev)

        def call(arm, i):
            c = cams[i % len(cams)]
            cam = types.SimpleNamespace(FoVx=2 * math.atan(c.tanfovx), FoVy=2 * math.atan(c.tanfovy), image_height=c.image_height,
                                        image_width=c.image_width, world_view_transform=c.world_view_transform.to(dev),
                                        full_proj_transform=c.full_proj_transform.to(dev), camera_center=c.camera_center.to(dev))
            out = renderer.render_raw(cam, pc, pipe, bg)
            objective(arm, out["render"], gt, out["normal"], out["pseudo_normal"].detach(), pc.get_scaling).backward()
            optimizer.step()
            optimizer.zero_grad(set_to_none=True)

        res["measure"] = "full step: render_raw + objective + backward + the library's Adam"
        if args.profile:
            res["profile"] = _profile(call, arms, args.warmup)
            print(json.dumps(res))
            return
        ms = _timed(call, arms, args.calls, args.warmup)
        for arm in arms:
            st = _stats(ms[arm])
            res[arm] = dict(st, it_per_s_median=1000.0 / st["ms_median"])
    res.update(calls=args.calls, warmup=args.warmup)
    res["torch_over_library_median"] = res["torch"]["ms_median"] / res["library"]["ms_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
