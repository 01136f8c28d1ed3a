"""Times RayMesh (first-hit ray casts on an LBVH) on seeded synthetic scenes: a height field of about 2M triangles with
subdivided icospheres placed on it.

  python tools/bench_raycast.py [--reps 20] [--profile]

Measured, each with CUDA events around the call (median, p10, p90 over --reps):
  * the BVH build at 0.5M and 2M triangles;
  * full-frame 1080p first hits from trajectory cameras (coherent rays) and random rays (incoherent), in rays per second;
  * extract_object's vote loop over 100 views with object-sized masks (intersects_first plus the reference's device lines);
  * the inpainting mask of one view (inpaint_mask: two casts, the depth comparison, two counts read back);
  * the CPU arm: the numpy restatement (tests/raycast_ref.py) on a measured subset of rays, labelled with its size.  It is a
    brute force over every triangle, not trimesh; trimesh is not installed and is not measured.
--profile adds the kernels per view of the vote loop and of the inpainting mask (torch.profiler, a separate run).
Prints one JSON line with the card name and power limit.
"""
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

from autovfx_b200.raycast import RayMesh, inpaint_mask  # noqa: E402
from tests import raycast_ref as R  # noqa: E402
from tests.test_gpu_raycast import heightfield, icosphere  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return "unknown (%s)" % ex


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    q = np.percentile(ms, [50, 10, 90])
    return {"median_ms": round(float(q[0]), 4), "p10_ms": round(float(q[1]), 4), "p90_ms": round(float(q[2]), 4)}


def scene(n_cells, n_spheres=20, level=5, seed=0):
    """A height field of 2 n_cells^2 triangles over [0, 100]^2 and n_spheres icospheres standing on it."""
    v, f = heightfield(n_cells, n_cells, seed=seed, size=100.0)
    rng = np.random.default_rng(seed)
    sv0, sf0 = icosphere(level)
    vs, fs = [v], [f]
    base = len(v)
    for _ in range(n_spheres):
        c = np.array([rng.uniform(10, 90), rng.uniform(10, 90), 1.5])
        vs.append(sv0 * rng.uniform(1.0, 3.0) + c)
        fs.append(sf0 + base)
        base += len(sv0)
    return np.concatenate(vs), np.concatenate(fs)


def camera_rays(eye, target, H, W, focal, dev):
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0, 0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = torch.eye(4, device=dev)
    c2w[:3, :3] = torch.tensor(np.stack([right, down, fwd], 1), dtype=torch.float32)
    c2w[:3, 3] = torch.tensor(eye, dtype=torch.float32)
    j, i = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
    dirs = torch.stack([(i - W / 2) / focal, (j - H / 2) / focal, torch.ones_like(i)], -1)
    rays_d = dirs @ c2w[:3, :3].T
    return c2w, c2w[:3, 3].expand_as(rays_d), rays_d


def trajectory(k, n, center=(50, 50, 0), radius=45.0, height=25.0):
    ang = 2 * np.pi * k / n
    return np.array([center[0] + radius * np.cos(ang), center[1] + radius * np.sin(ang), height])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_raycast needs a CUDA device"
    dev = torch.device("cuda:0")
    out = {"card": card()}

    # build at 0.5M and 2M triangles (height fields alone), then the query scene: 2M height-field triangles + 20 x 20480 spheres
    big_v, big_f = scene(1000)
    for name, (v, f) in (("build_0.5M", scene(500, n_spheres=0)), ("build_2M", scene(1000, n_spheres=0))):
        vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
        out[name] = dict(timed(lambda: RayMesh(vt, ft), max(3, args.reps // 2)), triangles=int(len(f)))
    rm = RayMesh(torch.from_numpy(big_v).to(dev), torch.from_numpy(big_f).to(dev))
    out["triangles"] = int(len(big_f))

    # 1080p first hits: coherent (trajectory cameras) and incoherent (random origins and directions in the scene's box)
    H, W = 1080, 1920
    views = [camera_rays(trajectory(k, 8), (50, 50, 0), H, W, 1400.0, dev) for k in range(8)]
    it = iter(range(1 << 30))

    def coherent():
        _, o, d = views[next(it) % len(views)]
        rm.intersects_first(o.reshape(-1, 3), d.reshape(-1, 3))
    r = timed(coherent, args.reps)
    r["rays_per_s"] = round(H * W / (r["median_ms"] * 1e-3))
    out["first_hit_1080p_coherent"] = r
    g = torch.Generator(device=dev).manual_seed(0)
    ro = torch.rand((H * W, 3), device=dev, generator=g) * torch.tensor([100.0, 100.0, 10.0], device=dev)
    rd = torch.randn((H * W, 3), device=dev, generator=g)
    r = timed(lambda: rm.intersects_first(ro, rd), args.reps)
    r["rays_per_s"] = round(H * W / (r["median_ms"] * 1e-3))
    out["first_hit_1080p_random"] = r

    # extract_object's vote loop over 100 views, object-sized masks: the pixels whose ray hits one sphere, dilated
    n_views = 100
    sphere_lo = 2_000_000  # the first sphere's triangles
    sphere_hi = sphere_lo + 20480
    centers = torch.Tensor(R.triangles(big_v, big_f).mean(axis=1)).to(dev)
    Hm, Wm = 540, 960
    K = torch.tensor([[700.0, 0, Wm / 2], [0, 700.0, Hm / 2], [0, 0, 1]], device=dev)
    c0 = big_v[big_f[sphere_lo:sphere_hi]].reshape(-1, 3).mean(0)
    cams, masks = [], []
    for k in range(n_views):
        eye = c0 + np.array([12 * np.cos(2 * np.pi * k / n_views), 12 * np.sin(2 * np.pi * k / n_views), 6.0])
        c2w, o, d = camera_rays(eye, c0, Hm, Wm, 700.0, dev)
        hit = rm.intersects_first(o.reshape(-1, 3), d.reshape(-1, 3)).reshape(Hm, Wm)
        m = (hit >= sphere_lo) & (hit < sphere_hi)
        m = m | torch.roll(m, 3, 0) | torch.roll(m, 3, 1)
        cams.append((c2w, o, d))
        masks.append(m)
    out["vote_mask_pixels_mean"] = round(float(np.mean([int(m.sum()) for m in masks])))

    def vote():
        counter = torch.zeros(len(big_f), dtype=torch.int32, device=dev)
        naive = torch.zeros(len(big_f), dtype=torch.int32, device=dev)
        for (c2w, o, d), mask in zip(cams, masks):
            index_tri = rm.intersects_first(o[mask].reshape(-1, 3), d[mask].reshape(-1, 3))
            naive[index_tri] += 1
            w2c = torch.inverse(c2w)
            xyz = centers[index_tri]
            xyz = torch.cat([xyz, torch.ones(xyz.size(0), 1, device=dev)], dim=1)
            xyz = torch.matmul(xyz, w2c.T)[:, :3]
            xyz = xyz / xyz[:, 2].unsqueeze(1)
            uv = torch.matmul(xyz, K.T)[:, :2].round().long()
            valid_uv = (uv[:, 0] >= 0) & (uv[:, 0] < Wm) & (uv[:, 1] >= 0) & (uv[:, 1] < Hm)
            filtered = uv[valid_uv]
            in_mask_indices = torch.where(mask[filtered[:, 1], filtered[:, 0]])[0]
            in_mask = valid_uv.nonzero().flatten()[in_mask_indices]
            counter[index_tri[in_mask]] += 1
        return counter
    r = timed(vote, max(3, args.reps // 4), warmup=1)
    r["views"] = n_views
    r["per_view_ms"] = round(r["median_ms"] / n_views, 4)
    out["vote_loop_100_views"] = r

    # inpainting mask per view: planar = the height field alone, combined = the whole scene
    planar = RayMesh(torch.from_numpy(big_v).to(dev), torch.from_numpy(big_f[:2_000_000]).to(dev))
    c2w, o, d = views[0]
    w2c = torch.inverse(c2w)
    out["inpaint_mask_1080p"] = timed(lambda: inpaint_mask(planar, rm, o, d, w2c), args.reps)

    # CPU arm: the numpy brute force on a measured subset (every triangle of the 2M scene, a few coherent rays)
    n_cpu = 16
    _, o, d = views[0]
    sel = torch.linspace(0, H * W - 1, n_cpu, device=dev).long()
    oc, dc = o.reshape(-1, 3)[sel].cpu().numpy(), d.reshape(-1, 3)[sel].cpu().numpy()
    t0 = time.perf_counter()
    rtri, _ = R.first_hit(oc, dc, big_v, big_f, chunk=1)
    cpu_s = time.perf_counter() - t0
    ours = rm.intersects_first(oc, dc).cpu().numpy()
    out["cpu_numpy_brute_force"] = {"rays": n_cpu, "triangles": int(len(big_f)), "seconds": round(cpu_s, 3),
                                    "rays_per_s": round(n_cpu / cpu_s, 2), "same_hits": bool(np.array_equal(rtri, ours)),
                                    "note": "measured on this subset only; trimesh is not measured"}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        def kernels(fn):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                fn()
                torch.cuda.synchronize()
            return sum(1 for e in p.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name)
        out["vote_loop_kernels_per_view"] = round(kernels(vote) / n_views, 2)
        out["inpaint_mask_kernels_per_view"] = kernels(lambda: inpaint_mask(planar, rm, views[0][1], views[0][2], w2c))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
