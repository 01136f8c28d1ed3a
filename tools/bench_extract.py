"""Time extract_object's subset scoring (extract/extract_object.py:168-224): the reference loop restated on the library's render()
(deepcopy + boolean indexing of six tensors, render() per tracked view, alpha to the host, numpy XOR count) against MaskScorer.

Setup: the 3M-Gaussian config-3 scene, V trajectory views at 1080p with a tracking mask each (a 5 % box subset's render with 2 %
of the pixels flipped), and R box subsets from 0.5 % to 20 % of the scene.  The two arms alternate, one ratio at a time, and
must give the same counts.  Only the rendering and counting are timed: the mesh steps of the function (closest triangles,
ray-cast votes, submesh, convex hull, np.isin) are not.  Prints one JSON line; writes a file only with --out.

    python tools/bench_extract.py [--views 100] [--ratios 22] [--reps 2] [--profile] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _pct(xs):
    a = np.asarray(xs, np.float64)
    return {"median": float(np.median(a)), "p10": float(np.percentile(a, 10)), "p90": float(np.percentile(a, 90))}


def _gpu_info() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--ratios", type=int, default=22)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--profile", action="store_true", help="also count the CUDA kernels of one ratio in each arm (torch.profiler)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_extract: needs a CUDA device")
    from autovfx_b200 import rasterizer as R, scene
    from autovfx_b200.extract import MaskScorer
    from autovfx_b200.renderer import render
    from tests import extract_ref as X
    dev = torch.device("cuda:0")
    R.set_exact_images(True)  # the alpha the threshold reads is the reference CUDA's, bit for bit
    pc = X.model_from(scene.config3_scene(args.gaussians), dev)
    traj = scene.trajectory_dict(radius=6.0, num_views=args.views, theta=35.0)
    views = [X.render_camera(c, dev) for c in scene.cameras_from_trajectory(traj)]
    xyz = pc.get_xyz
    bg = torch.zeros(3, device=dev)
    masks = {}
    obj = X.crop(pc, X.box_subset(xyz, 0.05))
    rng = np.random.default_rng(0)
    for idx, view in enumerate(views):
        with torch.no_grad():
            a = render(view, obj, X.PIPE, bg)["render"][3].cpu().numpy()
        m = np.where(a >= 0.8, 255, 0).astype(np.uint8)
        flip = rng.random(m.shape) < 0.02
        m[flip] = 255 - m[flip]
        masks["{0:05d}.png".format(idx)] = m
    fractions = np.geomspace(0.005, 0.2, args.ratios)
    subsets = [X.box_subset(xyz, float(f)) for f in fractions]
    t0 = time.perf_counter()
    scorer = MaskScorer(pc, views, masks, X.PIPE)
    torch.cuda.synchronize()
    setup_ms = (time.perf_counter() - t0) * 1e3
    scorer.count(subsets[0])  # warm-up: workspaces and binning capacity
    X.missed_pixels(pc, views, masks, subsets[0], bg, deep=True)

    ref_ms = [[] for _ in subsets]
    ours_ms = [[] for _ in subsets]
    for _ in range(args.reps):
        for i, m in enumerate(subsets):
            torch.cuda.synchronize()
            t = time.perf_counter()
            want = X.missed_pixels(pc, views, masks, m, bg, deep=True)
            ref_ms[i].append((time.perf_counter() - t) * 1e3)
            torch.cuda.synchronize()
            t = time.perf_counter()
            got = int(scorer.count(m))  # int() waits for the count
            ours_ms[i].append((time.perf_counter() - t) * 1e3)
            if got != want:
                raise SystemExit("bench_extract: counts differ at ratio %d: %d vs %d" % (i, got, want))
    res = {"bench": "extract_object subset scoring", "gpu": _gpu_info(), "gaussians": args.gaussians, "views": args.views,
           "ratios": args.ratios, "reps": args.reps, "subset_sizes": [int(m.sum()) for m in subsets],
           "scorer_setup_ms": setup_ms, "reference_ms_per_ratio": _pct(sum(ref_ms, [])), "scorer_ms_per_ratio": _pct(sum(ours_ms, [])),
           "speedup_median": float(np.median(sum(ref_ms, [])) / np.median(sum(ours_ms, []))),
           "per_ratio_median_ms": [[float(np.median(r)), float(np.median(o))] for r, o in zip(ref_ms, ours_ms)],
           "rerendered_views": scorer.rerendered, "not_timed": "mesh steps (closest triangles, ray-cast votes, submesh, convex hull, np.isin)"}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        m = subsets[len(subsets) // 2]
        for arm, fn in (("reference", lambda: X.missed_pixels(pc, views, masks, m, bg, deep=True)), ("scorer", lambda: int(scorer.count(m)))):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            res["kernels_per_ratio_" + arm] = len(kernels)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
