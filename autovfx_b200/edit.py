"""Resident, editable Gaussian scene: activation of raw parameters and the per-frame rigid edit of inserted objects.

Replaces, for the render loop of ``scene_representation.py:355-438``:

* ``GaussianModel.get_scaling / get_rotation / get_opacity / get_features`` (``sugar/gaussian_splatting/scene/
  gaussian_model.py:95-115``) — four torch activations + a cat on every render call — by ONE activation pass when the scene
  (or an object) is loaded;
* per frame and per inserted object: ``load_gaussians`` (a .ply read!), ``transform_gaussians`` and ``merge_two_gaussians``
  (``gaussians_utils.py:62-125``) plus a ``copy.deepcopy`` of the whole scene (``scene_representation.py:358``) — by one
  ``gsr_activate_gaussians`` launch per (frame, object) that writes the transformed, activated object into the tail of the
  resident scene arrays.

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


class ResidentScene:
    """A background scene plus insertable objects, resident on one GPU.

    ``compose({obj_id: (center, rotation, scaling, initial_center), ...})`` returns views of the activated arrays holding
    the scene followed by the transformed objects of this frame, in the order given — what the reference builds per frame with
    ``deepcopy`` + ``load_gaussians`` + ``transform_gaussians`` + ``merge_two_gaussians``
    (scene_representation.py:357-371).  The returned views alias the resident arrays: they are valid until the next
    ``compose`` call on the same stream (frames are rendered in stream order, so a render loop needs no extra synchronisation).
    """

    def __init__(self, scene_raw: Mapping[str, torch.Tensor], objects: Optional[Mapping[str, Mapping[str, torch.Tensor]]] = None,
                 device=None):
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        scene = _raw_on(scene_raw, self.device)
        self.P_scene = scene["xyz"].shape[0]
        self.M = scene["f_rest"].numel() // max(self.P_scene * 3, 1) + 1
        self.objects = {k: _raw_on(v, self.device) for k, v in (objects or {}).items()}
        for k, o in self.objects.items():
            n = o["xyz"].shape[0]
            if n and o["f_rest"].numel() // (n * 3) + 1 != self.M:
                raise ValueError("object %r stores %d SH coefficients, the scene %d" % (k, o["f_rest"].numel() // (n * 3) + 1, self.M))
        cap = self.P_scene + sum(o["xyz"].shape[0] for o in self.objects.values())
        self.arrays = _alloc(cap, self.M, self.device)
        activate_into(scene, self.arrays, 0, None)  # once; the raw scene tensors are not kept
        self.count = self.P_scene

    def compose(self, transforms: Mapping[str, Tuple] = ()) -> Dict[str, torch.Tensor]:
        off = self.P_scene
        for obj_id, tf in dict(transforms).items():
            if obj_id not in self.objects:
                raise KeyError("unknown object %r" % (obj_id,))
            xf = tf if isinstance(tf, _lib.gsr_object_xform) else make_xform(*tf)
            off += activate_into(self.objects[obj_id], self.arrays, off, xf)
        self.count = off
        return {k: v[:off] for k, v in self.arrays.items()}
