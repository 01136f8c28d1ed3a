"""numpy float64 brute force of gsr_mesh_closest: Ericson's closest-point test (Real-Time Collision Detection §5.1.5) in exactly the
kernel's operation order (every operation rounded on its own; numpy's elementwise ufuncs do not contract into FMAs), over every
(point, triangle) pair, the smallest squared distance winning and ties going to the lower triangle index; and a torch mirror for
meshes of millions of triangles.  Triangles and their validity are those of the ray-cast restatement (tests/raycast_ref.py)."""
from __future__ import annotations

import numpy as np

from tests.raycast_ref import triangles, valid

__all__ = ["closest_d2", "closest", "closest_torch", "triangles", "valid"]


def closest_d2(points, tris, xp=np) -> np.ndarray:
    """float64 [N, F]: the squared distance from every point to its closest point on every triangle, Ericson's
    ClosestPtPointTriangle in exactly gsr_mesh_closest's operation order (gsr_mesh.cu, closest_d2):
      ab = b - a, ac = c - a, ap = p - a, bp = p - b, cp = p - c; dot(u, w) = (ux wx + uy wy) + uz wz
      d1 = dot(ab, ap), d2 = dot(ac, ap); d3 = dot(ab, bp), d4 = dot(ac, bp); d5 = dot(ab, cp), d6 = dot(ac, cp)
      vc = d1 d4 - d3 d2, vb = d5 d2 - d1 d6, va = d3 d6 - d5 d4, e = d4 - d3, f = d5 - d6
      the first region that applies, in this order:
        d1 <= 0 and d2 <= 0                   q = a
        d3 >= 0 and d4 <= d3                  q = b
        vc <= 0 and d1 >= 0 and d3 <= 0       q = a + (d1 / (d1 - d3)) ab
        d6 >= 0 and d5 <= d6                  q = c
        vb <= 0 and d2 >= 0 and d6 <= 0       q = a + (d2 / (d2 - d6)) ac
        va <= 0 and e >= 0 and f >= 0         q = b + (e / (e + f)) (c - b)
        otherwise                             q = (a + (vb / den) ab) + (vc / den) ac, den = (va + vb) + vc
      result ((p - q)x^2 + (p - q)y^2) + (p - q)z^2
    Every operation is one elementwise ufunc (numpy does not contract into FMAs).  Every branch is evaluated and the first
    applicable one is selected, which gives the bits of the kernel's branch.  ``xp``: numpy, or torch for closest_torch."""
    N, F = len(points), len(tris)
    P = [points[:, k][:, None] for k in range(3)]  # [N, 1]
    A = [tris[:, 0, k][None, :] for k in range(3)]  # [1, F]
    B = [tris[:, 1, k][None, :] for k in range(3)]
    Cv = [tris[:, 2, k][None, :] for k in range(3)]

    def dot(u, w):
        return (u[0] * w[0] + u[1] * w[1]) + u[2] * w[2]
    ab = [B[k] - A[k] for k in range(3)]
    ac = [Cv[k] - A[k] for k in range(3)]
    ap = [P[k] - A[k] for k in range(3)]
    bp = [P[k] - B[k] for k in range(3)]
    cp = [P[k] - Cv[k] for k in range(3)]
    d1, d2 = dot(ab, ap), dot(ac, ap)
    d3, d4 = dot(ab, bp), dot(ac, bp)
    d5, d6 = dot(ab, cp), dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e, f = d4 - d3, d5 - d6
    rA = (d1 <= 0) & (d2 <= 0)
    rB = (d3 >= 0) & (d4 <= d3)
    rAB = (vc <= 0) & (d1 >= 0) & (d3 <= 0)
    rC = (d6 >= 0) & (d5 <= d6)
    rAC = (vb <= 0) & (d2 >= 0) & (d6 <= 0)
    rBC = (va <= 0) & (e >= 0) & (f >= 0)
    v_ab = d1 / (d1 - d3)
    w_ac = d2 / (d2 - d6)
    w_bc = e / (e + f)
    den = (va + vb) + vc
    v, w = vb / den, vc / den
    out = None
    for k in range(3):
        q = (A[k] + v * ab[k]) + w * ac[k]
        q = xp.where(rBC, B[k] + w_bc * (Cv[k] - B[k]), q)
        q = xp.where(rAC, A[k] + w_ac * ac[k], q)
        q = xp.where(rC, Cv[k], q)
        q = xp.where(rAB, A[k] + v_ab * ab[k], q)
        q = xp.where(rB, B[k], q)
        q = xp.where(rA, A[k], q)
        ek = P[k] - q
        sq = ek * ek
        out = sq if out is None else out + sq
    return out


def closest(points, vertices, faces, chunk: int = 256):
    """(tri int64 [N], d2 float64 [N]): the brute force of gsr_mesh_closest over every (point, triangle) pair.  Invalid triangles
    (valid() false) never win, nor does a NaN or +inf d2; the smallest d2 wins, ties to the lower index; a point with a non-finite
    coordinate, or no valid triangle, gives -1 and +inf."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    tris = triangles(vertices, faces)
    N = len(p)
    tri = np.full(N, -1, dtype=np.int64)
    d2 = np.full(N, np.inf)
    if len(tris) == 0:
        return tri, d2
    ok_t = valid(tris)
    ok_p = np.isfinite(p).all(1)
    for s in range(0, N, chunk):
        with np.errstate(all="ignore"):
            dd = closest_d2(p[s:s + chunk], tris)
        dd = np.where(ok_t[None, :] & ok_p[s:s + chunk, None] & ~np.isnan(dd), dd, np.inf)
        best = np.argmin(dd, axis=1)  # the first index of the smallest d2: ties go to the lower triangle index
        bd = dd[np.arange(len(dd)), best]
        h = bd < np.inf
        tri[s:s + chunk][h] = best[h]
        d2[s:s + chunk][h] = bd[h]
    return tri, d2


def closest_torch(points, tris, ok_tri, chunk: int = 8):
    """closest restated with torch float64 elementwise ops, one operation per kernel (no FMA contraction), for the brute force
    over millions of triangles on the GPU.  ``tris``: float64 [F, 3, 3] tensor; ``ok_tri``: valid(tris) as a bool tensor.
    tests/test_gpu_closest.py checks it against the numpy restatement."""
    import torch
    p = torch.as_tensor(np.asarray(points, dtype=np.float64).reshape(-1, 3), device=tris.device)
    N, F = len(p), len(tris)
    tri = torch.full((N,), -1, dtype=torch.int64, device=tris.device)
    d2 = torch.full((N,), float("inf"), dtype=torch.float64, device=tris.device)
    if F == 0:
        return tri, d2
    ok_p = torch.isfinite(p).all(1)
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=tris.device)
    for s in range(0, N, chunk):
        e = min(N, s + chunk)
        dd = closest_d2(p[s:e], tris, xp=torch)
        dd = torch.where(ok_tri[None, :] & ok_p[s:e, None] & ~torch.isnan(dd), dd, inf)
        bd = dd.min(dim=1).values
        idx = torch.arange(F, device=tris.device).expand_as(dd)
        best = torch.where(dd == bd[:, None], idx, torch.full_like(idx, F)).min(dim=1).values
        h = bd < float("inf")
        tri[s:e] = torch.where(h, best, torch.full_like(best, -1))
        d2[s:e] = bd
    return tri, d2
