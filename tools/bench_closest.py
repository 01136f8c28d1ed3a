"""Times RayMesh.closest (open3d's compute_closest_points on the device LBVH) and the melting-mesh frame on seeded synthetic
scenes: the ray-cast benchmark's height field of 2M triangles with 20 icospheres standing on it (2.41M triangles).

  python tools/bench_closest.py [--reps 20] [--profile]

Measured, each with CUDA events around the call (median, p10, p90 over --reps):
  * 3M near-surface Gaussian-like points (random surface points offset along the normal) in a shuffled order, as densification
    leaves a trained model's rows, and the same points in surface order (the entry point sorts the queries along a Morton curve
    either way, so the two differ by what the sort does not recover);
  * 3M uniform points in the scene's box;
  * the per-ratio mask3d line of extract_object (mask_triangles uploaded and indexed by the closest triangles);
  * one melting frame through ResidentScene.compose: 200k object Gaussians, two melting meshes of 20,480 triangle centres each;
  * the CPU arm: the numpy brute force (tests/closest_ref.py) on a measured subset of points, labelled with its size.  open3d is
    not installed and is not measured.
--profile adds the kernels per call (torch.profiler, a separate run).  Prints one JSON line with the card name and power limit.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_raycast import card, scene, timed  # noqa: E402
from tests import closest_ref as R  # noqa: E402
from tests.test_gpu_raycast import icosphere  # noqa: E402

__all__ = ["scene", "near_surface_points"]


def near_surface_points(v, f, n, seed, device, shuffle=True):
    """float32 [n, 3] on ``device``: points on random triangles (uniform barycentrics) offset along the unit normal by
    N(0, 0.02), in a random row order (``shuffle``) or in triangle order."""
    g = torch.Generator(device=device).manual_seed(seed)
    t = torch.from_numpy(R.triangles(v, f)).to(device)
    tri = torch.randint(0, len(f), (n,), device=device, generator=g)
    if not shuffle:
        tri = torch.sort(tri).values
    w = -torch.log(torch.rand((n, 3), device=device, generator=g, dtype=torch.float64))
    w = w / w.sum(1, keepdim=True)
    nrm = torch.linalg.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    nrm = nrm / nrm.norm(dim=1, keepdim=True)
    p = (t[tri] * w[:, :, None]).sum(1) + nrm[tri] * (0.02 * torch.randn((n, 1), device=device, generator=g, dtype=torch.float64))
    if shuffle:
        p = p[torch.randperm(n, device=device, generator=g)]
    return p.float().contiguous()


def main():
    from autovfx_b200 import edit
    from autovfx_b200.raycast import RayMesh
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_closest needs a CUDA device"
    dev = torch.device("cuda:0")
    out = {"card": card()}
    v, f = scene(1000)
    rm = RayMesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
    out["triangles"] = int(len(f))
    n = 3_000_000
    out["points"] = n

    shuffled = near_surface_points(v, f, n, seed=0, device=dev)
    ordered = near_surface_points(v, f, n, seed=0, device=dev, shuffle=False)
    for name, pts in (("closest_3M_near_surface_shuffled", shuffled), ("closest_3M_near_surface_surface_order", ordered)):
        r = timed(lambda: rm.closest(pts), args.reps)
        r["points_per_s"] = round(n / (r["median_ms"] * 1e-3))
        out[name] = r

    lo, hi = torch.from_numpy(v.min(0)).to(dev), torch.from_numpy(v.max(0)).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    uni = (lo + (hi - lo) * torch.rand((n, 3), device=dev, generator=g, dtype=torch.float64)).float()
    r = timed(lambda: rm.closest(uni), args.reps)
    r["points_per_s"] = round(n / (r["median_ms"] * 1e-3))
    out["closest_3M_uniform_box"] = r

    # extract_object.py:191-192 per ratio: the [F] triangle mask from the host, indexed by the Gaussians' closest triangles
    triangle_ids = rm.compute_closest_points(shuffled)["primitive_ids"]
    mask_triangles = np.random.default_rng(2).random(len(f)) < 0.05
    out["mask3d_line_per_ratio"] = timed(lambda: torch.from_numpy(mask_triangles).cuda()[triangle_ids], args.reps)

    # one melting frame: 200k object Gaussians around a 20,480-triangle icosphere, two melting meshes of 20,480 centres
    ov, of = icosphere(5, radius=1.0)
    rng = np.random.default_rng(3)
    n_obj, M = 200_000, 16

    def raw(k, center):
        u = rng.standard_normal((k, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        return {"xyz": (center + u * (1 + 0.02 * rng.standard_normal((k, 1)))).astype(np.float32),
                "f_dc": rng.standard_normal((k, 1, 3)).astype(np.float32), "f_rest": rng.standard_normal((k, M - 1, 3)).astype(np.float32),
                "opacity": rng.standard_normal((k, 1)).astype(np.float32), "scaling": (rng.standard_normal((k, 3)) - 4).astype(np.float32),
                "rotation": rng.standard_normal((k, 4)).astype(np.float32)}
    rs = edit.ResidentScene(raw(1_000_000, np.zeros(3)), device=dev,
                            melting={"obj": (raw(n_obj, np.zeros(3)), RayMesh(ov.astype(np.float32), of))})
    cen = R.triangles(ov, of).mean(axis=1)
    frame = {"obj": [torch.from_numpy((cen * 0.9).astype(np.float32)).to(dev), torch.from_numpy((cen * 1.1).astype(np.float32)).to(dev)]}
    r = timed(lambda: rs.compose(melting=frame), args.reps)
    r.update(object_gaussians=n_obj, centres_per_mesh=int(len(cen)), meshes=2, rows=int(rs.count - 1_000_000))
    out["melting_frame_compose"] = r

    # CPU arm: the numpy brute force on a measured subset (every triangle of the scene, a few points)
    n_cpu = 8
    sub = shuffled[:n_cpu].cpu().numpy()
    t0 = time.perf_counter()
    rtri, _ = R.closest(sub, v, f, chunk=1)
    cpu_s = time.perf_counter() - t0
    out["cpu_numpy_brute_force"] = {"points": n_cpu, "triangles": int(len(f)), "seconds": round(cpu_s, 3),
                                    "points_per_s": round(n_cpu / cpu_s, 3), "same_ids": bool(np.array_equal(rtri, rm.closest(sub)[0].cpu().numpy())),
                                    "note": "measured on this subset only; open3d is not measured"}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        def kernels(fn):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                fn()
                torch.cuda.synchronize()
            ev = [e for e in p.events() if e.device_type.name == "CUDA"]
            return {"kernels": sum(1 for e in ev if "Memcpy" not in e.name and "Memset" not in e.name),
                    "dtoh_copies": sum(1 for e in ev if "DtoH" in e.name)}
        out["closest_kernels_per_call"] = kernels(lambda: rm.closest(shuffled))
        out["melting_frame_kernels"] = kernels(lambda: rs.compose(melting=frame))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
