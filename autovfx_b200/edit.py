"""Resident, editable Gaussian scene: activation of raw parameters and the per-frame rigid edit of inserted objects.

Replaces, for the render loop of ``scene_representation.py:355-438``:

* ``GaussianModel.get_scaling / get_rotation / get_opacity / get_features`` (``sugar/gaussian_splatting/scene/
  gaussian_model.py:95-115``) — four torch activations + a cat on every render call — by ONE activation pass when the scene
  (or an object) is loaded;
* per frame and per inserted object: ``load_gaussians`` (a .ply read!), ``transform_gaussians`` and ``merge_two_gaussians``
  (``gaussians_utils.py:62-125``) plus a ``copy.deepcopy`` of the whole scene (``scene_representation.py:358``) — by one
  ``gsr_activate_gaussians`` launch per (frame, object) that writes the transformed, activated object into the tail of the
  resident scene arrays;
* per frame and per melting object (``scene_representation.py:372-421``): the mesh and ``.ply`` reloads, open3d's closest
  triangles of the object's Gaussians and of the melting meshes' triangle centres, ``np.isin``, the boolean indexing and the
  merge — by the Gaussians' closest triangles found once, one ``gsr_mesh_closest`` and one ``gsr_mesh_isin_rows`` per melting
  mesh, one readback of the subsets' sizes and one activation per subset.

Raw parameter dict (the reference's ``GaussianModel`` fields, as ``scene.load_ply`` returns them):
``xyz [N,3]``, ``f_dc [N,1,3]``, ``f_rest [N,M-1,3]``, ``opacity [N,1]``, ``scaling [N,3]`` (log), ``rotation [N,4]``.

Reference quirk to be aware of: ``merge_two_gaussians`` builds a fresh ``GaussianModel(4)`` whose ``active_sh_degree`` is 0
(``gaussian_model.py:45``), so the reference renders edited frames with SH degree 0 at the storage stride M; pass
``sh_degree=0`` to the renderer to reproduce that, or the trained degree for what was probably intended.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import lib as _L

__all__ = ["matrix_to_quaternion", "make_xform", "activate_into", "activate", "ResidentScene"]

RAW_KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def matrix_to_quaternion(R) -> np.ndarray:
    """3x3 rotation matrix -> (w,x,y,z), float32 arithmetic; the candidate with the largest denominator wins, like the
    reference's (pytorch3d-derived) ``rotation_utils.py:24-84``.  Host side: it runs once per (frame, object)."""
    m = np.asarray(R, dtype=np.float32).reshape(3, 3)
    f = np.float32
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = (f(v) for v in m.reshape(9))
    one = f(1.0)
    sq = np.array([one + m00 + m11 + m22, one + m00 - m11 - m22, one - m00 + m11 - m22, one - m00 - m11 + m22], dtype=np.float32)
    q_abs = np.sqrt(np.maximum(sq, f(0.0))).astype(np.float32)  # _sqrt_positive_part
    cand = np.array([[q_abs[0] * q_abs[0], m21 - m12, m02 - m20, m10 - m01],
                     [m21 - m12, q_abs[1] * q_abs[1], m10 + m01, m02 + m20],
                     [m02 - m20, m10 + m01, q_abs[2] * q_abs[2], m12 + m21],
                     [m10 - m01, m20 + m02, m21 + m12, q_abs[3] * q_abs[3]]], dtype=np.float32)
    cand = cand / (f(2.0) * np.maximum(q_abs, f(0.1)))[:, None]
    return cand[int(np.argmax(q_abs))].astype(np.float32)


def make_xform(center, rotation, scaling: float, initial_center) -> _lib.gsr_object_xform:
    """The arguments of ``transform_gaussians(gaussians, center, rotation, scaling, initial_center)``
    (gaussians_utils.py:88) packed for the C ABI."""
    x = _lib.gsr_object_xform()
    R = np.asarray(rotation, dtype=np.float32).reshape(3, 3)
    x.rotation[:] = [float(v) for v in R.reshape(9)]
    x.quat[:] = [float(v) for v in matrix_to_quaternion(R)]
    x.center[:] = [float(v) for v in np.asarray(center, dtype=np.float32).reshape(3)]
    x.initial_center[:] = [float(v) for v in np.asarray(initial_center, dtype=np.float32).reshape(3)]
    x.scaling = float(scaling)
    x.log_scaling = float(np.log(scaling))  # np.log(scaling) added to a float32 tensor (gaussians_utils.py:103)
    return x


def _raw_on(raw: Mapping[str, torch.Tensor], device) -> Dict[str, torch.Tensor]:
    out = {}
    alias = {"scaling": "scale", "rotation": "rot"}  # scene.load_ply's names
    for k in RAW_KEYS:
        t = torch.as_tensor(raw[k] if k in raw else raw[alias[k]])
        out[k] = t.to(device=device, dtype=torch.float32).contiguous()
    N = out["xyz"].shape[0]
    if out["f_dc"].numel() != N * 3 or out["opacity"].numel() != N or out["scaling"].shape != (N, 3) or out["rotation"].shape != (N, 4):
        raise ValueError("raw Gaussian parameters have inconsistent shapes")
    if out["f_rest"].numel() % max(N * 3, 1) != 0:
        raise ValueError("f_rest must be [N, M-1, 3]")
    return out


def activate_into(raw: Mapping[str, torch.Tensor], dst: Mapping[str, torch.Tensor], offset: int = 0,
                  xform: Optional[_lib.gsr_object_xform] = None) -> int:
    """Activate (and optionally transform) ``raw`` into rows ``[offset, offset+N)`` of the activated arrays ``dst``
    (``means3D [cap,3]``, ``shs [cap,M,3]``, ``opacities [cap,1]``, ``scales [cap,3]``, ``rotations [cap,4]``).  ``raw`` must
    already live on ``dst``'s device as contiguous float32 (see ``ResidentScene``).  Returns N."""
    means = dst["means3D"]
    device = means.device
    if not means.is_cuda:
        raise RuntimeError("autovfx_b200.edit: CUDA tensors required (there is no CPU path)")
    N = raw["xyz"].shape[0]
    M = dst["shs"].shape[1]
    cap = means.shape[0]
    if offset < 0 or offset + N > cap:
        raise ValueError("activate_into: rows [%d, %d) exceed the capacity %d" % (offset, offset + N, cap))
    rest_coeffs = raw["f_rest"].numel() // max(N * 3, 1) if N else M - 1
    if N and rest_coeffs != M - 1:
        raise ValueError("activate_into: object has %d SH coefficients, the scene stores %d" % (rest_coeffs + 1, M))
    if N == 0:
        return 0
    for k in RAW_KEYS:
        t = raw[k]
        if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("activate_into: raw[%r] must be a contiguous float32 tensor on %s" % (k, device))

    def at(t, row_floats):
        return t.data_ptr() + offset * row_floats * 4
    with torch.cuda.device(device):
        rc = _L.gsr_activate_gaussians(N, M, raw["xyz"].data_ptr(), raw["f_dc"].data_ptr(), raw["f_rest"].data_ptr() if M > 1 else None,
                                       raw["opacity"].data_ptr(), raw["scaling"].data_ptr(), raw["rotation"].data_ptr(),
                                       C.byref(xform) if xform is not None else None, at(means, 3), at(dst["shs"], 3 * M),
                                       at(dst["opacities"], 1), at(dst["scales"], 3), at(dst["rotations"], 4), _lib.stream_ptr(device))
        _lib.check(rc, "gsr_activate_gaussians")
    from . import rasterizer as _R  # the arrays changed behind the version counters the geometry-reuse cache watches
    _R.invalidate_geometry_cache(device)
    return N


def _alloc(cap: int, M: int, device) -> Dict[str, torch.Tensor]:
    f = dict(dtype=torch.float32, device=device)
    return {"means3D": torch.empty((cap, 3), **f), "shs": torch.empty((cap, M, 3), **f), "opacities": torch.empty((cap, 1), **f),
            "scales": torch.empty((cap, 3), **f), "rotations": torch.empty((cap, 4), **f)}


def activate(raw: Mapping[str, torch.Tensor], device=None, xform: Optional[_lib.gsr_object_xform] = None) -> Dict[str, torch.Tensor]:
    """Raw parameters -> the activated tensors a ``GaussianRasterizer`` call takes (one fused pass instead of exp + normalize +
    sigmoid + cat)."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    r = _raw_on(raw, device)
    N = r["xyz"].shape[0]
    M = r["f_rest"].numel() // max(N * 3, 1) + 1 if N else 1
    dst = _alloc(N, M, device)
    activate_into(r, dst, 0, xform)
    return dst


# the melting meshes of one object per frame: ``{idx:03d}_obj.stl`` and ``{idx:03d}_obj_dup.stl``
MELT_SUBSETS = 2


class _Melting:
    """One melting object: its raw Gaussians, its original mesh, their closest triangles, and two compaction buffers."""

    def __init__(self, raw: Dict[str, torch.Tensor], mesh, ids: torch.Tensor):
        self.raw, self.mesh, self.ids = raw, mesh, ids
        self.bufs = [{k: torch.empty_like(v) for k, v in raw.items()} for _ in range(MELT_SUBSETS)]


def _sh_count(raw: Mapping[str, torch.Tensor]) -> Optional[int]:
    """M, the SH coefficients per channel, from the shapes of ``raw`` alone (no copy, no device work); None without rows."""
    n = int(torch.as_tensor(raw["xyz"]).shape[0])
    return int(torch.as_tensor(raw["f_rest"]).numel()) // (n * 3) + 1 if n else None


class ResidentScene:
    """A background scene plus insertable objects, resident on one GPU.

    ``compose({obj_id: (center, rotation, scaling, initial_center), ...})`` returns views of the activated arrays holding
    the scene followed by the transformed objects of this frame, in the order given — what the reference builds per frame with
    ``deepcopy`` + ``load_gaussians`` + ``transform_gaussians`` + ``merge_two_gaussians``
    (scene_representation.py:357-371).  The returned views alias the resident arrays: they are valid until the next
    ``compose`` call on the same stream (frames are rendered in stream order, so a render loop needs no extra synchronisation).

    ``melting={obj_id: (orig_raw, RayMesh(orig_mesh.vertices, orig_mesh.faces))}`` keeps each melting object's original
    Gaussians resident and finds their closest original triangles once.  ``compose(melting={obj_id: [centres, ...]})`` is then
    the melting-mesh branch of the render loop (scene_representation.py:372-421): for each of the frame's melting meshes
    (``triangles_center`` arrays, at most ``_obj`` and ``_obj_dup`` per object, objects in sorted order) the original Gaussians
    whose closest triangle is also the closest triangle of one of the centres (``np.isin``) are activated, in row order, behind
    the scene.  The subsets' sizes are read back once per frame, together.
    """

    def __init__(self, scene_raw: Mapping[str, torch.Tensor], objects: Optional[Mapping[str, Mapping[str, torch.Tensor]]] = None,
                 device=None, melting: Optional[Mapping[str, Tuple[Mapping[str, torch.Tensor], object]]] = None):
        from .raycast import RayMesh
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        melting = dict(melting or {})
        M = _sh_count(scene_raw) or 1
        for k, entry in melting.items():  # checked before anything is uploaded
            if not isinstance(entry, (tuple, list)) or len(entry) != 2:
                raise ValueError("melting[%r] must be a pair (orig_raw, RayMesh)" % (k,))
            if _sh_count(entry[0]) not in (None, M):
                raise ValueError("melting object %r stores %d SH coefficients, the scene %d" % (k, _sh_count(entry[0]), M))
            if not isinstance(entry[1], RayMesh):
                raise ValueError("melting[%r][1] must be a RayMesh of the object's original mesh, not %s" % (k, type(entry[1]).__name__))
            if entry[1].device != self.device:
                raise ValueError("melting[%r][1] is on %s, the scene on %s" % (k, entry[1].device, self.device))
        scene = _raw_on(scene_raw, self.device)
        self.P_scene = scene["xyz"].shape[0]
        self.M = scene["f_rest"].numel() // max(self.P_scene * 3, 1) + 1
        self.objects = {k: _raw_on(v, self.device) for k, v in (objects or {}).items()}
        for k, o in self.objects.items():
            n = o["xyz"].shape[0]
            if n and o["f_rest"].numel() // (n * 3) + 1 != self.M:
                raise ValueError("object %r stores %d SH coefficients, the scene %d" % (k, o["f_rest"].numel() // (n * 3) + 1, self.M))
        self.melting_objects: Dict[str, _Melting] = {}
        with torch.no_grad(), torch.cuda.device(self.device):
            for k, (raw, mesh) in melting.items():
                r = _raw_on(raw, self.device)
                self.melting_objects[k] = _Melting(r, mesh, mesh.closest(r["xyz"])[0])  # once: the same answer on every frame
            ws = max([int(_L.gsr_mesh_isin_rows_bytes(m.ids.shape[0], m.mesh.F)) for m in self.melting_objects.values()], default=0)
            self._isin_ws = torch.empty((max(ws, 4),), dtype=torch.uint8, device=self.device)
            self._isin_count = torch.zeros((max(MELT_SUBSETS * len(melting), 1),), dtype=torch.int64, device=self.device)
        cap = self.P_scene + sum(o["xyz"].shape[0] for o in self.objects.values())
        cap += MELT_SUBSETS * sum(m.ids.shape[0] for m in self.melting_objects.values())
        self.arrays = _alloc(cap, self.M, self.device)
        activate_into(scene, self.arrays, 0, None)  # once; the raw scene tensors are not kept
        self.count = self.P_scene

    def _melting_plan(self, melting: Mapping[str, Sequence]) -> list:
        """(obj_id, slot, centres) of the frame's melting meshes in the reference's order: object ids sorted, then the meshes in
        the order given (``_obj`` before ``_obj_dup``)."""
        plan = []
        for obj_id in sorted(melting):
            if obj_id not in self.melting_objects:
                raise KeyError("unknown melting object %r" % (obj_id,))
            centres = list(melting[obj_id])
            if len(centres) > MELT_SUBSETS:
                raise ValueError("melting[%r]: %d meshes, at most %d per object (_obj and _obj_dup)" % (obj_id, len(centres), MELT_SUBSETS))
            plan += [(obj_id, slot, c) for slot, c in enumerate(centres)]
        return plan

    def compose(self, transforms: Mapping[str, Tuple] = (), melting: Optional[Mapping[str, Sequence]] = None) -> Dict[str, torch.Tensor]:
        if melting is not None and len(dict(transforms)):
            raise ValueError("transforms and melting are exclusive, as the reference's rigid-body and melting-mesh branches are")
        off = self.P_scene
        if melting is not None:
            off += self._compose_melting(self._melting_plan(melting))
        for obj_id, tf in dict(transforms).items():
            if obj_id not in self.objects:
                raise KeyError("unknown object %r" % (obj_id,))
            xf = tf if isinstance(tf, _lib.gsr_object_xform) else make_xform(*tf)
            off += activate_into(self.objects[obj_id], self.arrays, off, xf)
        self.count = off
        return {k: v[:off] for k, v in self.arrays.items()}

    def _compose_melting(self, plan: list) -> int:
        """Select and activate the melting subsets behind the scene; returns the rows written."""
        if not plan:
            return 0
        dev = self.device
        stream = _lib.stream_ptr(dev)
        K = len(RAW_KEYS)
        with torch.no_grad(), torch.cuda.device(dev):
            for j, (obj_id, slot, centres) in enumerate(plan):
                m = self.melting_objects[obj_id]
                tri_c = m.mesh.closest(centres)[0]
                dst = m.bufs[slot]
                src_p = (C.c_void_p * K)(*[m.raw[k].data_ptr() for k in RAW_KEYS])
                dst_p = (C.c_void_p * K)(*[dst[k].data_ptr() for k in RAW_KEYS])
                words = (C.c_int32 * K)(*[m.raw[k].numel() // max(m.ids.shape[0], 1) for k in RAW_KEYS])
                _lib.check(_L.gsr_mesh_isin_rows(m.ids.shape[0], m.ids.data_ptr(), tri_c.shape[0], tri_c.data_ptr(), m.mesh.F, K, src_p, dst_p,
                                                 words, self._isin_count[j:].data_ptr(), self._isin_ws.data_ptr(), self._isin_ws.numel(),
                                                 stream), "gsr_mesh_isin_rows")
            counts = self._isin_count[:len(plan)].tolist()  # the frame's one readback: the views need the row count
        off = self.P_scene
        for (obj_id, slot, _), n in zip(plan, counts):
            sub = {k: v[:n] for k, v in self.melting_objects[obj_id].bufs[slot].items()}
            off += activate_into(sub, self.arrays, off, None)
        return off - self.P_scene
