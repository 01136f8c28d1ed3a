"""numpy float64 brute force of gsr_mesh_first_hit: the watertight ray-triangle test (Woop, Benthin and Wald 2013) in exactly
the kernel's operation order (every operation rounded on its own; numpy's elementwise ufuncs do not contract into FMAs), over
every (ray, triangle) pair, the smallest t > 0 winning and ties going to the lower triangle index."""
from __future__ import annotations

import numpy as np


def triangles(vertices, faces) -> np.ndarray:
    """float64 [F, 3, 3] of the mesh's triangles."""
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    return v[f] if len(f) else np.zeros((0, 3, 3))


def valid(tris: np.ndarray) -> np.ndarray:
    """bool [F]: finite vertices and a non-zero (v1 - v0) x (v2 - v0), as the kernel's tri_valid."""
    v0, v1, v2 = tris[:, 0], tris[:, 1], tris[:, 2]
    with np.errstate(all="ignore"):
        e1, e2 = v1 - v0, v2 - v0
        nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
        ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
        nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return np.isfinite(tris).all(axis=(1, 2)) & ((nx != 0) | (ny != 0) | (nz != 0))


def ray_setup(o: np.ndarray, d: np.ndarray):
    """(ok, kx, ky, kz, Sx, Sy, Sz) per ray: kz the axis of largest |d| (ties to the lower axis), kx, ky the next two, swapped
    when d[kz] < 0; the shear coefficients as correctly rounded quotients."""
    ok = np.isfinite(o).all(1) & np.isfinite(d).all(1) & (d != 0).any(1)
    a = np.abs(d)
    kz = np.zeros(len(d), dtype=np.int64)
    kz = np.where(a[:, 1] > a[np.arange(len(d)), kz], 1, kz)
    kz = np.where(a[:, 2] > a[np.arange(len(d)), kz], 2, kz)
    kx = (kz + 1) % 3
    ky = (kx + 1) % 3
    r = np.arange(len(d))
    neg = d[r, kz] < 0
    kx, ky = np.where(neg, ky, kx), np.where(neg, kx, ky)
    with np.errstate(all="ignore"):
        dz = np.where(ok, d[r, kz], 1.0)
        Sx = d[r, kx] / dz
        Sy = d[r, ky] / dz
        Sz = 1.0 / dz
    return ok, kx, ky, kz, Sx, Sy, Sz


def hit_t(o: np.ndarray, d: np.ndarray, tris: np.ndarray) -> np.ndarray:
    """float64 [N, F]: t of every (ray, triangle) pair the test accepts, +inf elsewhere."""
    N, F = len(o), len(tris)
    out = np.full((N, F), np.inf)
    if N == 0 or F == 0:
        return out
    ok, kx, ky, kz, Sx, Sy, Sz = ray_setup(o, d)
    r = np.arange(N)
    ox, oy, oz = o[r, kx][:, None], o[r, ky][:, None], o[r, kz][:, None]
    Sx, Sy, Sz = Sx[:, None], Sy[:, None], Sz[:, None]
    with np.errstate(all="ignore"):
        sh = []
        for k in range(3):
            v = tris[:, k]  # [F, 3]
            akx = v[:, kx].T - ox  # [N, F]
            aky = v[:, ky].T - oy
            akz = v[:, kz].T - oz
            sh.append((akx - Sx * akz, aky - Sy * akz, Sz * akz))
        (Ax, Ay, Az), (Bx, By, Bz), (Cx, Cy, Cz) = sh
        U = Cx * By - Cy * Bx
        V = Ax * Cy - Ay * Cx
        W = Bx * Ay - By * Ax
        mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
        det = (U + V) + W
        T = (U * Az + V * Bz) + W * Cz
        t = T / det
        hit = ~mixed & (det != 0) & (t > 0) & (t < np.inf)
    hit &= ok[:, None] & valid(tris)[None, :]
    out[hit] = t[hit]
    return out


def first_hit(origins, directions, vertices, faces, chunk: int = 256):
    """(tri int64 [N], t float64 [N]): the first hit of every ray, -1 / +inf on a miss."""
    o = np.asarray(origins, dtype=np.float64).reshape(-1, 3)
    d = np.asarray(directions, dtype=np.float64).reshape(-1, 3)
    tris = triangles(vertices, faces)
    N = len(o)
    tri = np.full(N, -1, dtype=np.int64)
    t = np.full(N, np.inf)
    for s in range(0, N, chunk):
        ts = hit_t(o[s:s + chunk], d[s:s + chunk], tris)
        if ts.shape[1] == 0:
            continue
        best = np.argmin(ts, axis=1)  # the first index of the smallest t: ties go to the lower triangle index
        bt = ts[np.arange(len(ts)), best]
        h = bt < np.inf
        tri[s:s + chunk][h] = best[h]
        t[s:s + chunk][h] = bt[h]
    return tri, t


def locations(origins, directions, tri, t):
    """intersects_location's (locations, index_ray, index_tri): o + t d per component for the rays that hit, ascending."""
    o = np.asarray(origins, dtype=np.float64).reshape(-1, 3)
    d = np.asarray(directions, dtype=np.float64).reshape(-1, 3)
    idx = np.nonzero(tri >= 0)[0]
    return o[idx] + t[idx, None] * d[idx], idx, tri[idx]


def depth(loc: np.ndarray, w2c) -> np.ndarray:
    """((x w20 + y w21) + z w22) + w23 in float64, the library's documented order."""
    w = np.asarray(w2c, dtype=np.float64)
    return ((loc[:, 0] * w[2, 0] + loc[:, 1] * w[2, 1]) + loc[:, 2] * w[2, 2]) + w[2, 3]


def inpaint_mask(rays_o, rays_d, planar, combined, w2c):
    """extract_object.py:563-606 for one view with the oracle's hits and the documented depth order: the uint8 mask shaped like
    rays_o[..., 0], or None where the reference continues.  ``planar`` / ``combined``: (vertices, faces)."""
    shape = np.shape(rays_o)[:-1]
    o = np.asarray(rays_o, dtype=np.float64).reshape(-1, 3)
    d = np.asarray(rays_d, dtype=np.float64).reshape(-1, 3)
    tri_p, t_p = first_hit(o, d, *planar)
    loc_p, index_ray_planar, _ = locations(o, d, tri_p, t_p)
    if len(index_ray_planar) == 0:
        return None
    tri_a, t_a = first_hit(o[index_ray_planar], d[index_ray_planar], *combined)
    loc_a, index_ray_all, _ = locations(o[index_ray_planar], d[index_ray_planar], tri_a, t_a)
    if len(index_ray_all) == 0:
        return None
    depth_planar = depth(loc_p, w2c)
    depth_all = np.zeros(depth_planar.shape)
    depth_all[index_ray_all] = depth(loc_a, w2c)
    mask = np.abs(depth_all - depth_planar) < 0.01
    out = np.zeros(int(np.prod(shape)), dtype=np.uint8)
    out[index_ray_planar[mask]] = 255
    return out.reshape(shape)


def first_hit_torch(origins, directions, tris, ok_tri, chunk: int = 8):
    """first_hit restated with torch float64 elementwise ops, one operation per kernel (so no FMA contraction either), for the
    brute force over millions of triangles on the GPU.  ``tris``: float64 [F, 3, 3] tensor; ``ok_tri``: valid(tris) as a bool
    tensor.  tests/test_gpu_raycast.py checks it against the numpy restatement."""
    import torch
    o = torch.as_tensor(np.asarray(origins, dtype=np.float64).reshape(-1, 3), device=tris.device)
    d = torch.as_tensor(np.asarray(directions, dtype=np.float64).reshape(-1, 3), device=tris.device)
    okr, kx, ky, kz, Sx, Sy, Sz = (torch.as_tensor(a, device=tris.device) for a in ray_setup(o.cpu().numpy(), d.cpu().numpy()))
    N = len(o)
    tri = torch.full((N,), -1, dtype=torch.int64, device=tris.device)
    t = torch.full((N,), float("inf"), dtype=torch.float64, device=tris.device)
    for s in range(0, N, chunk):
        e = min(N, s + chunk)
        r = torch.arange(s, e, device=tris.device)
        ox, oy, oz = o[r, kx[r]][:, None], o[r, ky[r]][:, None], o[r, kz[r]][:, None]
        sx, sy, sz = Sx[r][:, None], Sy[r][:, None], Sz[r][:, None]
        sh = []
        for k in range(3):
            v = tris[:, k]
            akx = v[:, kx[r]].T - ox
            aky = v[:, ky[r]].T - oy
            akz = v[:, kz[r]].T - oz
            sh.append((akx - sx * akz, aky - sy * akz, sz * akz))
        (Ax, Ay, Az), (Bx, By, Bz), (Cx, Cy, Cz) = sh
        U = Cx * By - Cy * Bx
        V = Ax * Cy - Ay * Cx
        W = Bx * Ay - By * Ax
        mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
        det = (U + V) + W
        T = (U * Az + V * Bz) + W * Cz
        tt = T / det
        hit = ~mixed & (det != 0) & (tt > 0) & (tt < float("inf")) & okr[r][:, None] & ok_tri[None, :]
        tt = torch.where(hit, tt, torch.full_like(tt, float("inf")))
        bt = tt.min(dim=1).values
        cand = tt == bt[:, None]  # the lowest index among the minima: torch's min does not promise which index it returns
        idx = torch.arange(tt.shape[1], device=tris.device).expand_as(tt)
        best = torch.where(cand, idx, torch.full_like(idx, tt.shape[1])).min(dim=1).values
        h = bt < float("inf")
        tri[s:e] = torch.where(h, best, torch.full_like(best, -1))
        t[s:e] = bt
    return tri, t
