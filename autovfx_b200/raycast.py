"""First-hit ray casts against triangle meshes on the GPU: trimesh's ``mesh.ray.intersects_first`` and
``intersects_location(multiple_hits=False)`` at AutoVFX's call sites (INTEGRATION.md, "Mesh ray casts")::

    rm = RayMesh(mesh.vertices, mesh.faces)               # an LBVH built on the device (gsr_mesh_build)
    index_tri = rm.intersects_first(rays_o, rays_d)       # device int64 [N], -1 on a miss, no readback
    locations, index_ray, index_tri = rm.intersects_location(rays_o, rays_d)

The semantics are fixed (DESIGN.md §4): the watertight test (Woop, Benthin and Wald 2013) in float64, every operation rounded
on its own; both faces; hits with t > 0 along the direction as given; the smallest t, ties to the lower triangle index.
Degenerate triangles, triangles with a non-finite vertex, and zero, NaN or infinite rays never hit.  tests/raycast_ref.py
restates the test in numpy, bit for bit.

The same BVH answers open3d's ``RaycastingScene.compute_closest_points`` (INTEGRATION.md, "Closest triangles")::

    tri, d2 = rm.closest(points)                          # device int64 [N] and float64 [N], no readback
    triangle_ids = rm.compute_closest_points(points)["primitive_ids"]

Ericson's closest-point test in float64, every operation rounded on its own; the smallest squared distance, ties to the lower
triangle index; invalid triangles never win; a non-finite point gives -1.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import lib as _L

__all__ = ["RayMesh", "inpaint_mask"]

_FLOAT = (torch.float32, torch.float64)


def _host_or_cuda(x, name: str) -> torch.Tensor:
    """``x`` as a tensor without copying: a CUDA tensor as it is, a numpy array as a CPU view still to be uploaded; a CPU tensor
    raises RuntimeError."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise RuntimeError("autovfx_b200.raycast: %s must live on a CUDA device (there is no CPU path)" % name)
        return x
    a = np.asarray(x)
    if not (np.issubdtype(a.dtype, np.integer) or np.issubdtype(a.dtype, np.floating)):
        raise ValueError("%s must be a real numeric array, not %s" % (name, a.dtype))
    return torch.from_numpy(np.ascontiguousarray(a))


def _on(t: torch.Tensor, name: str, device: Optional[torch.device]) -> torch.Tensor:
    """Upload a numpy-backed tensor to ``device`` (the current CUDA device if None); a CUDA tensor must already be there."""
    if t.is_cuda:
        if device is not None and t.device != device:
            raise ValueError("%s is on %s, expected %s" % (name, t.device, device))
        return t
    return t.to(device if device is not None else torch.device("cuda", torch.cuda.current_device()))


def _rows3(t: torch.Tensor, name: str) -> None:
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError("%s must have shape [N, 3], got %s" % (name, tuple(t.shape)))


class RayMesh:
    """A triangle mesh prepared for first-hit ray casts and closest-triangle queries on one CUDA device.

    ``vertices``: float32 or float64 ``[V, 3]``; ``faces``: int32 or int64 ``[F, 3]`` with every index in ``[0, V)``, F < 2**31
    (trimesh's ``mesh.vertices`` / ``mesh.faces``).  numpy arrays are uploaded to the current CUDA device (or to the device of
    the other argument when that one is a tensor).  A wrong shape, dtype or index raises ValueError naming the argument; a CPU
    tensor raises RuntimeError.  Building reads nothing back except the face-index range check."""

    def __init__(self, vertices, faces):
        v = _host_or_cuda(vertices, "vertices")
        f = _host_or_cuda(faces, "faces")
        _rows3(v, "vertices")
        _rows3(f, "faces")
        if v.dtype not in _FLOAT:
            raise ValueError("vertices must be float32 or float64, not %s" % v.dtype)
        if f.dtype not in (torch.int32, torch.int64):
            raise ValueError("faces must be int32 or int64, not %s" % f.dtype)
        V, F = int(v.shape[0]), int(f.shape[0])
        if F >= 2 ** 31:
            raise ValueError("faces: %d triangles, at most 2**31 - 1 are supported" % F)
        if F > 0:
            lo, hi = torch.stack(list(torch.aminmax(f))).tolist()
            if lo < 0 or hi >= V:
                raise ValueError("faces: indices must lie in [0, %d), got [%d, %d]" % (V, lo, hi))
        dev = v.device if v.is_cuda else f.device if f.is_cuda else None
        v, f = _on(v, "vertices", dev), _on(f, "faces", dev)
        self.device, self.V, self.F = v.device, V, F
        with torch.no_grad(), torch.cuda.device(self.device):
            v64 = v.detach().to(torch.float64).contiguous()
            f64 = f.detach().to(torch.int64).contiguous()
            self.bvh = torch.zeros(int(_L.gsr_mesh_bvh_bytes(F)), dtype=torch.uint8, device=self.device)
            ws = _lib.scratch_bytes(max(int(_L.gsr_mesh_build_bytes(F)), 256), self.device)
            _lib.check(_L.gsr_mesh_build(V, F, v64.data_ptr(), f64.data_ptr(), self.bvh.data_ptr(), self.bvh.numel(), ws.data_ptr(),
                                         ws.numel(), _lib.stream_ptr(self.device)), "gsr_mesh_build")

    def _rays(self, ray_origins, ray_directions) -> Tuple[torch.Tensor, torch.Tensor, int]:
        o = _host_or_cuda(ray_origins, "ray_origins")
        d = _host_or_cuda(ray_directions, "ray_directions")
        _rows3(o, "ray_origins")
        _rows3(d, "ray_directions")
        if o.shape[0] != d.shape[0]:
            raise ValueError("ray_origins has %d rows, ray_directions %d" % (o.shape[0], d.shape[0]))
        for t, name in ((o, "ray_origins"), (d, "ray_directions")):
            if t.dtype == torch.bool or t.is_complex():
                raise ValueError("%s must be a real array, not %s" % (name, t.dtype))
        o, d = _on(o, "ray_origins", self.device), _on(d, "ray_directions", self.device)
        if o.dtype == torch.float32 and d.dtype == torch.float32:
            return o.contiguous(), d.contiguous(), 0
        # float64 holds every float32 exactly; integer directions (extract_object.py:476-477) are converted as numpy would
        return o.to(torch.float64).contiguous(), d.to(torch.float64).contiguous(), 1

    def first_hit(self, ray_origins, ray_directions, active: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(tri int64 [N], t float64 [N]) on the device: the first triangle each ray hits (-1 on a miss) and its distance in
        units of the direction as given (+inf on a miss).  ``active`` (int64 [N], optional): rays with ``active < 0`` miss."""
        o, d, f64 = self._rays(ray_origins, ray_directions)
        N = int(o.shape[0])
        with torch.no_grad(), torch.cuda.device(self.device):
            tri = torch.empty((N,), dtype=torch.int64, device=self.device)
            t = torch.empty((N,), dtype=torch.float64, device=self.device)
            act = 0
            if active is not None:
                if not isinstance(active, torch.Tensor) or active.dtype != torch.int64 or tuple(active.shape) != (N,) or active.device != self.device:
                    raise ValueError("active must be an int64 tensor of shape (%d,) on %s" % (N, self.device))
                active = active.contiguous()
                act = active.data_ptr()
            _lib.check(_L.gsr_mesh_first_hit(self.F, self.bvh.data_ptr(), N, o.data_ptr(), d.data_ptr(), f64, act, tri.data_ptr(), t.data_ptr(),
                                              _lib.stream_ptr(self.device)), "gsr_mesh_first_hit")
        return tri, t

    def intersects_first(self, ray_origins, ray_directions) -> torch.Tensor:
        """trimesh's ``intersects_first``: the index of the first triangle each ray hits, -1 on a miss (device int64 [N])."""
        return self.first_hit(ray_origins, ray_directions)[0]

    def intersects_location(self, ray_origins, ray_directions, multiple_hits: bool = False):
        """trimesh's ``intersects_location(multiple_hits=False)``: (locations float64 [H,3], index_ray int64 [H], index_tri int64
        [H]) for the rays that hit, in ascending ray order, with ``location = o + t d`` per component (one multiply, one add, in
        float64).  Reads the hit count back once."""
        if multiple_hits:
            raise ValueError("multiple_hits=True is not supported: RayMesh reports the first hit of each ray")
        o, d, _ = self._rays(ray_origins, ray_directions)
        tri, t = self.first_hit(o, d)
        with torch.no_grad(), torch.cuda.device(self.device):
            index_ray = torch.nonzero(tri >= 0).flatten()
            th = t[index_ray].unsqueeze(1)
            locations = o[index_ray].to(torch.float64) + th * d[index_ray].to(torch.float64)
        return locations, index_ray, tri[index_ray]

    def closest(self, points) -> Tuple[torch.Tensor, torch.Tensor]:
        """(tri int64 [N], d2 float64 [N]) on the device, no readback: the valid triangle closest to each point and the squared
        distance to its closest point (Ericson's ClosestPtPointTriangle in float64, every operation rounded on its own), the
        smallest d2 winning and ties going to the lower triangle index.  ``points``: ``[N, 3]`` numpy array or CUDA tensor,
        float32 or float64 (widened exactly), other real dtypes converted to float64.  A point with a non-finite coordinate, or a
        mesh without a valid triangle, gives -1 and +inf.  The kernel visits the points along a Morton curve (N < 2**31)."""
        p = _host_or_cuda(points, "points")
        _rows3(p, "points")
        if p.dtype == torch.bool or p.is_complex():
            raise ValueError("points must be a real array, not %s" % p.dtype)
        p = _on(p, "points", self.device)
        f64 = 0 if p.dtype == torch.float32 else 1
        N = int(p.shape[0])
        if N >= 2 ** 31:
            raise ValueError("points: %d rows, at most 2**31 - 1 are supported" % N)
        with torch.no_grad(), torch.cuda.device(self.device):
            p = p.detach().contiguous() if f64 == 0 else p.detach().to(torch.float64).contiguous()
            tri = torch.empty((N,), dtype=torch.int64, device=self.device)
            d2 = torch.empty((N,), dtype=torch.float64, device=self.device)
            ws = _lib.scratch_bytes(max(int(_L.gsr_mesh_closest_bytes(N)), 256), self.device)
            _lib.check(_L.gsr_mesh_closest(self.F, self.bvh.data_ptr(), N, p.data_ptr(), f64, tri.data_ptr(), d2.data_ptr(), ws.data_ptr(),
                                            ws.numel(), _lib.stream_ptr(self.device)), "gsr_mesh_closest")
        return tri, d2

    def compute_closest_points(self, query_points) -> Dict[str, torch.Tensor]:
        """open3d's ``RaycastingScene.compute_closest_points`` for the one key AutoVFX reads: ``{"primitive_ids": tri}``, a device
        int64 [N] tensor.  Where open3d returns its uint32 ``INVALID_ID`` (no valid triangle, a non-finite point) this returns -1.
        open3d's other keys (``points``, ``geometry_ids``, ``primitive_uvs``, ``primitive_normals``) are not computed."""
        return {"primitive_ids": self.closest(query_points)[0]}


def inpaint_mask(planar: RayMesh, combined: RayMesh, rays_o, rays_d, w2c) -> Optional[torch.Tensor]:
    """One view of extract_object.py:563-606: the uint8 mask (255 where a ray hits ``planar`` and its depth there is within
    0.01 of its depth on ``combined``), shaped like ``rays_o`` without its last axis, on the device.

    ``rays_o``, ``rays_d``: the view's rays ``[..., 3]`` as the reference makes them (its ``.cpu().numpy()`` is not needed);
    ``w2c``: ``torch.inverse(c2w)``, ``[4, 4]``, converted exactly to float64.  Returns None where the reference ``continue``s: no
    ray hits the planar mesh, or none of those rays hits the combined mesh.  Where a planar-hit ray misses the combined mesh its
    combined depth is 0, as the reference's ``np.zeros`` fill.  Depth is ``((x w20 + y w21) + z w22) + w23`` in float64; numpy's
    matmul order is not reproduced (INTEGRATION.md).  Reads two counts back."""
    if not isinstance(planar, RayMesh) or not isinstance(combined, RayMesh):
        raise ValueError("planar and combined must be RayMesh objects")
    if planar.device != combined.device:
        raise ValueError("planar is on %s, combined on %s" % (planar.device, combined.device))
    dev = planar.device
    ro = _host_or_cuda(rays_o, "rays_o")
    rd = _host_or_cuda(rays_d, "rays_d")
    if ro.dim() < 1 or ro.shape[-1] != 3 or tuple(ro.shape) != tuple(rd.shape):
        raise ValueError("rays_o and rays_d must share a shape [..., 3], got %s and %s" % (tuple(ro.shape), tuple(rd.shape)))
    shape = tuple(ro.shape[:-1])
    w = _host_or_cuda(w2c, "w2c")
    if tuple(w.shape) != (4, 4) or not w.dtype.is_floating_point:
        raise ValueError("w2c must be a floating-point [4, 4] matrix, got %s %s" % (w.dtype, tuple(w.shape)))
    w = _on(w, "w2c", dev)
    o, d, f64 = planar._rays(_on(ro, "rays_o", dev).reshape(-1, 3), _on(rd, "rays_d", dev).reshape(-1, 3))
    N = int(o.shape[0])
    tri_p, t_p = planar.first_hit(o, d)
    tri_a, t_a = combined.first_hit(o, d, active=tri_p)
    with torch.no_grad(), torch.cuda.device(dev):
        w64 = w.to(torch.float64).contiguous()
        mask = torch.empty((N,), dtype=torch.uint8, device=dev)
        counts = torch.empty((2,), dtype=torch.int64, device=dev)
        _lib.check(_L.gsr_mesh_inpaint_mask(N, o.data_ptr(), d.data_ptr(), f64, tri_p.data_ptr(), t_p.data_ptr(), tri_a.data_ptr(), t_a.data_ptr(),
                                            w64.data_ptr(), mask.data_ptr(), counts.data_ptr(), _lib.stream_ptr(dev)), "gsr_mesh_inpaint_mask")
        n_planar, n_all = (int(c) for c in counts.tolist())
    if n_planar == 0 or n_all == 0:
        return None
    return mask.reshape(shape)
