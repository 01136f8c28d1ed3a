"""Cost of deterministic rasterizer gradients (torch.use_deterministic_algorithms(True) -> gsr_backward_det) in a training step.

The step is tools/bench_train_loss.py --step: render_raw on the 3M-Gaussian config-3 scene at 1920x1080, train.py's objective
(photometric + normal + anisotropic), backward(), the library's Adam.  Three arms alternate step by step in one process:

  default       the flag off: the atomic blend backward;
  det           the flag on with torch's default fill_uninitialized_memory = True (what users get: torch fills every torch.empty
                of the step, the trainer's own tensors included, with NaN; the library's scratch is allocated without the fill);
  det_nofill    the flag on with fill_uninitialized_memory = False, which separates torch's fills from the library's cost.

Printed: median / p10 / p90 of the step and of backward() alone (CUDA events), the peak allocation of one step above the resident
model, the scratch bytes, the (footprint, splat) partials the blend backward visits (counted from the frame's ballot matrix and each
footprint's last contributor) against the 8 R slots, and the card and its power limit.  --profile counts kernels per step per arm
instead (torch.profiler, a separate run).  Needs CUBLAS_WORKSPACE_CONFIG=:4096:8 only when densification runs; this step has none.

    python tools/bench_deterministic.py [--steps 30] [--warmup 5] [--gaussians 3000000] [--width 1920 --height 1080] [--profile]
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
import torch.utils.deterministic  # noqa: E402

ARMS = ("default", "det", "det_nofill")


def _set_arm(arm):
    torch.use_deterministic_algorithms(arm != "default")
    torch.utils.deterministic.fill_uninitialized_memory = arm != "det_nofill"


def _stats(ms):
    v = np.asarray(ms)
    return {"ms_median": float(np.median(v)), "ms_p10": float(np.percentile(v, 10)), "ms_p90": float(np.percentile(v, 90))}


def _raster_node(t):
    """The rasterizer's autograd node behind a render output (its saved tensors hold the frame's workspaces)."""
    seen, todo = set(), [t.grad_fn]
    while todo:
        n = todo.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        if "_RasterizeGaussians" in type(n).__name__:
            return n
        todo.extend(f for f, _ in n.next_functions)
    raise RuntimeError("no rasterizer node behind the render")


def visited_partials(node, P, W, H):
    """(footprint, splat) partials the blend backward visits: list entries whose footprint ballot bit is set and whose position is
    below the footprint's last contributor (max n_contrib over its 8x4 pixels)."""
    from autovfx_b200 import rasterizer as R
    geom, binning, image = node.saved_tensors[7:10]
    v = R.debug_views((geom, binning, image), P, W, H)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = torch.zeros(gy * 16, gx * 16, dtype=torch.int64, device=image.device)
    nc[:H, :W] = v["n_contrib"].long()
    wl = nc.view(gy, 4, 4, gx, 2, 8).amax(dim=(2, 5)).permute(0, 2, 1, 3).reshape(gy * gx, 8)  # [tile][f], f = 2 band + half
    rg = v["ranges"].long()
    n = rg[:, 1] - rg[:, 0]
    tile = torch.repeat_interleave(torch.arange(gx * gy, device=image.device), n)
    j = torch.arange(int(n.sum()), device=image.device) - torch.repeat_interleave(torch.cumsum(n, 0) - n, n)  # position in the tile's list
    fixed = 32 * 131072 + 512  # BinLayout: ballot rows after 12 bytes per instance of capacity, 256-byte aligned
    cap = (binning.numel() - fixed) // 13
    off = -(-12 * cap // 256) * 256
    bal = binning[off:off + 32 * (cap // 32 + 131072 + 2)].view(torch.int32).long() & 0xffffffff
    row = (rg[tile, 0] >> 5) + tile + (j >> 5)
    total = 0
    for f in range(8):
        bit = (bal[row * 8 + f] >> (j & 31)) & 1
        total += int(((bit == 1) & (j < wl[tile, f])).sum())
    return total, int(n.sum())


def main():
    from autovfx_b200 import losses, renderer, scene
    from autovfx_b200 import rasterizer as R
    from autovfx_b200._lib import lib as L
    from autovfx_b200.optim import use_cuda_adam
    from tools.bench_train_loss import LAMBDA_ANISOTROPIC, LAMBDA_DSSIM, LAMBDA_PSEUDO_NORMAL, _profile
    from tools.bench_train_raw import RawModel
    from tools.bench_train_render import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--profile", action="store_true", help="count the kernels of one step per arm instead of timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    H, W, P = args.height, args.width, args.gaussians
    gt = torch.rand(4, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    pc = RawModel({k: v.to(dev) for k, v in scene.config3_scene(P=P).items()})
    lrs = (0.00016 * 5.0, 0.0025, 0.0025 / 20.0, 0.05, 0.005, 0.001)
    optimizer = use_cuda_adam(torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(pc.params(), lrs)], lr=0.0, eps=1e-15))
    cams = scene.cameras_from_trajectory(scene.trajectory_dict(radius=4.0, num_views=300, theta=30.0, w=W, h=H, fov_x_deg=60.0))
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    bg = torch.zeros(3, device=dev)
    res = {"card": card(), "workload": "render_raw training step (train.py objective, library Adam), %.1fM Gaussians M = 16, %dx%d"
           % (P / 1e6, W, H)}

    def camera(i):
        c = cams[i % len(cams)]
        return types.SimpleNamespace(FoVx=2 * math.atan(c.tanfovx), FoVy=2 * math.atan(c.tanfovy), image_height=c.image_height,
                                     image_width=c.image_width, world_view_transform=c.world_view_transform.to(dev),
                                     full_proj_transform=c.full_proj_transform.to(dev), camera_center=c.camera_center.to(dev))

    def step(arm, i, bw=None, keep=None):
        _set_arm(arm)
        out = renderer.render_raw(camera(i), pc, pipe, bg)
        loss = losses.photometric_loss(out["render"], gt, LAMBDA_DSSIM) + \
            LAMBDA_PSEUDO_NORMAL * losses.normal_loss(out["normal"], out["pseudo_normal"].detach()) + \
            LAMBDA_ANISOTROPIC * losses.anisotropic_loss(pc.get_scaling)
        if keep is not None:
            keep.append(visited_partials(_raster_node(out["render"]), P, W, H))
        if bw is not None:
            bw[0].record()
        loss.backward()
        if bw is not None:
            bw[1].record()
        optimizer.step()
        optimizer.zero_grad(set_to_none=True)

    if args.profile:
        for arm in ARMS:
            step(arm, 0)
        res["profile"] = _profile(step, list(ARMS), args.warmup)
        _set_arm("default")
        print(json.dumps(res))
        return
    for i in range(args.warmup):
        for arm in ARMS:
            step(arm, i)
    torch.cuda.synchronize()
    ms = {a: [] for a in ARMS}
    bms = {a: [] for a in ARMS}
    for i in range(args.steps):
        for arm in (ARMS if i % 2 == 0 else ARMS[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            bw = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            a.record()
            step(arm, args.warmup + i, bw)
            b.record()
            b.synchronize()
            ms[arm].append(a.elapsed_time(b))
            bms[arm].append(bw[0].elapsed_time(bw[1]))
    for arm in ARMS:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        step(arm, 0)
        torch.cuda.synchronize()
        res[arm] = {"step": _stats(ms[arm]), "backward": _stats(bms[arm]),
                    "peak_alloc_mb_above_model": (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20}
    counts = []
    step("default", 0, keep=counts)
    visited, rendered = counts[0]
    stats = R.last_frame_stats()
    res["frame0"] = {"num_rendered": rendered, "slots_8R": 8 * rendered, "visited_partials": visited,
                     "visited_share_of_slots": visited / max(1, 8 * rendered),
                     "scratch_bytes": int(L.gsr_backward_det_bytes(rendered, W, H, 1)), "num_rendered_counter": stats["num_rendered"]}
    _set_arm("default")
    res["det_over_default_step_median"] = res["det"]["step"]["ms_median"] / res["default"]["step"]["ms_median"]
    res["det_nofill_over_default_step_median"] = res["det_nofill"]["step"]["ms_median"] / res["default"]["step"]["ms_median"]
    res.update(steps=args.steps, warmup=args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
