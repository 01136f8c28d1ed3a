"""Densification in CUDA: drop-ins for the per-step statistics and ``densify_and_prune`` of 3DGS's ``GaussianModel``
("GS/" = sugar/gaussian_splatting/scene/gaussian_model.py:268-417) and SuGaR's ``SuGaRDensifier``
("SD/" = sugar/sugar_scene/sugar_densifier.py:48-246), through ``gsr_densify_stats``, ``gsr_densify_plan`` and
``gsr_densify_apply``.

Opt in on the classes (each takes the method's exact signature)::

    from autovfx_b200 import densify
    GaussianModel.add_densification_stats = densify.add_densification_stats
    GaussianModel.update_densification_stats = densify.update_densification_stats
    GaussianModel.densify_and_prune = densify.densify_and_prune
    SuGaRDensifier.update_densification_stats = densify.update_densification_stats
    SuGaRDensifier.densify_and_prune = densify.sugar_densify_and_prune

The statistics run without a host synchronisation.  densify_and_prune reads the two totals {S, P'} back once (they size the new
tensors) and writes every new parameter and both Adam moments in one pass, in the reference's final row order.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from . import _lib

__all__ = ["add_densification_stats", "update_densification_stats", "densify_and_prune", "sugar_densify_and_prune"]

# GaussianModel: (group name, model attribute, role)
_GS_GROUPS = (("xyz", "_xyz", _lib.GSR_DENSIFY_ROLE_XYZ), ("f_dc", "_features_dc", _lib.GSR_DENSIFY_ROLE_COPY),
              ("f_rest", "_features_rest", _lib.GSR_DENSIFY_ROLE_COPY), ("opacity", "_opacity", _lib.GSR_DENSIFY_ROLE_COPY),
              ("scaling", "_scaling", _lib.GSR_DENSIFY_ROLE_SCALING), ("rotation", "_rotation", _lib.GSR_DENSIFY_ROLE_COPY))
# SuGaR (SD/:68-79)
_SUGAR_GROUPS = (("points", "_points", _lib.GSR_DENSIFY_ROLE_XYZ), ("all_densities", "all_densities", _lib.GSR_DENSIFY_ROLE_COPY),
                 ("scales", "_scales", _lib.GSR_DENSIFY_ROLE_SCALING), ("quaternions", "_quaternions", _lib.GSR_DENSIFY_ROLE_COPY),
                 ("sh_coordinates_dc", "_sh_coordinates_dc", _lib.GSR_DENSIFY_ROLE_COPY),
                 ("sh_coordinates_rest", "_sh_coordinates_rest", _lib.GSR_DENSIFY_ROLE_COPY))


def _f32(x) -> float:
    """A threshold as torch compares it with a float32 tensor: a Python number rounded to float, a tensor's float32 value."""
    if isinstance(x, torch.Tensor):
        return float(x.detach().float().cpu())
    return float(np.float32(x))


def _times(a, extent):
    """a * extent as the reference computes it: in double for a Python extent, in float32 for a tensor extent."""
    if isinstance(extent, torch.Tensor):
        return a * extent.detach().float().cpu()
    return a * extent


def _require_cuda(who, *ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("autovfx_b200.%s: every tensor must be a CUDA tensor (there is no CPU path)" % who)
    dev = ts[0].device
    for t in ts:
        if t is not None and t.device != dev:
            raise ValueError("%s: tensors on %s and %s" % (who, dev, t.device))


def _check_leaf(who, name, t, P=None):
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s: %s must be a torch.Tensor, got %s" % (who, name, type(t).__name__))
    if t.dtype != torch.float32:
        raise ValueError("%s: %s must be float32, got %s" % (who, name, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s: %s must be contiguous" % (who, name))
    if t.dim() == 0 or (P is not None and t.shape[0] != P):
        raise ValueError("%s: %s must have %s rows, got shape %s" % (who, name, P, tuple(t.shape)))


# ------------------------------------------------------------------------------------------------------------- statistics
def _stats(who, accum, denom, max_radii, viewspace_point_tensor, mask, radii):
    grad = getattr(viewspace_point_tensor, "grad", None)
    if grad is None:
        raise ValueError("%s: viewspace_point_tensor.grad is missing (call it after loss.backward())" % who)
    _check_leaf(who, "viewspace_point_tensor.grad", grad)
    P = grad.shape[0]
    if grad.dim() != 2 or grad.shape[1] < 2:
        raise ValueError("%s: viewspace_point_tensor.grad must be [P, >=2], got %s" % (who, tuple(grad.shape)))
    for name, t in (("accumulator", accum), ("denom", denom)):
        _check_leaf(who, name, t, P)
        if t.numel() != P:
            raise ValueError("%s: %s must be [P, 1], got %s" % (who, name, tuple(t.shape)))
    if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or mask.shape != (P,):
        raise ValueError("%s: the visibility filter must be a bool tensor [%d]" % (who, P))
    if max_radii is not None:
        _check_leaf(who, "max_radii2D", max_radii, P)
        if not isinstance(radii, torch.Tensor) or radii.dtype != torch.int32 or radii.shape != (P,):
            raise ValueError("%s: radii must be an int32 tensor [%d]" % (who, P))
    _require_cuda(who, grad, accum, denom, mask, max_radii, radii)
    mask = mask.contiguous()
    radii = None if radii is None else radii.contiguous()
    rc = _lib.lib.gsr_densify_stats(P, grad.shape[1], grad.data_ptr(), mask.data_ptr(), None if radii is None else radii.data_ptr(),
                                    accum.data_ptr(), denom.data_ptr(), None if max_radii is None else max_radii.data_ptr(),
                                    _lib.stream_ptr(grad.device))
    _lib.check(rc, "gsr_densify_stats")


def add_densification_stats(self, viewspace_point_tensor, update_filter):
    """GaussianModel.add_densification_stats (GS/:415-417) in one kernel: xyz_gradient_accum[f] += |grad[f, :2]|, denom[f] += 1,
    bit for bit, with no nonzero() and no host synchronisation."""
    _stats("add_densification_stats", self.xyz_gradient_accum, self.denom, None, viewspace_point_tensor, update_filter, None)


def update_densification_stats(self, viewspace_point_tensor, radii, visibility_filter):
    """SuGaRDensifier.update_densification_stats (SD/:156-164) in one kernel; on a GaussianModel it replaces the trainers' pair
    ``max_radii2D[f] = max(max_radii2D[f], radii[f]); add_densification_stats(...)`` (train.py:163-164,
    scene_representation.py:526-527).  The accumulator is ``points_gradient_accum`` or, if absent, ``xyz_gradient_accum``."""
    accum = self.points_gradient_accum if hasattr(self, "points_gradient_accum") else self.xyz_gradient_accum
    _stats("update_densification_stats", accum, self.denom, self.max_radii2D, viewspace_point_tensor, visibility_filter, radii)


# -------------------------------------------------------------------------------------------------------- densify and prune
def _run(who, optimizer, groups, accum, denom, scaling, opacity, xyz, rotation, rotation_mode, max_grad, min_opacity, extent,
         max_screen_size, percent_dense):
    """groups: [(group name, role)] to rebuild.  Returns ({name: new nn.Parameter}, P')."""
    by_name = {}
    for g in optimizer.param_groups:
        by_name.setdefault(g.get("name"), g)
    P = scaling.shape[0]
    found = []
    for name, role in groups:
        g = by_name.get(name)
        if g is None:
            raise ValueError("%s: the optimizer has no param group named %r" % (who, name))
        if len(g["params"]) != 1:
            raise ValueError("%s: param group %r must hold one tensor, got %d" % (who, name, len(g["params"])))
        p = g["params"][0]
        _check_leaf(who, "param group %r" % name, p, P)
        st = optimizer.state.get(p, None)
        if st is not None:
            for k in ("exp_avg", "exp_avg_sq"):
                _check_leaf(who, "%s of param group %r" % (k, name), st.get(k), P)
                if st[k].shape != p.shape:
                    raise ValueError("%s: %s of param group %r has shape %s, the parameter %s" % (who, k, name, tuple(st[k].shape),
                                                                                                 tuple(p.shape)))
        found.append((name, role, g, p, st))
    for name, t, shape in (("accumulator", accum, None), ("denom", denom, None), ("scaling", scaling, (P, 3)),
                           ("opacity", opacity, None), ("xyz", xyz, (P, 3)), ("rotation", rotation, (P, 4))):
        _check_leaf(who, name, t, P)
        if (shape is not None and tuple(t.shape) != shape) or (shape is None and t.numel() != P):
            raise ValueError("%s: %s has shape %s for %d rows" % (who, name, tuple(t.shape), P))
    _require_cuda(who, scaling, accum, denom, opacity, xyz, rotation, *[f[3] for f in found])
    dev = scaling.device
    L = _lib.lib
    stream = _lib.stream_ptr(dev)
    with torch.cuda.device(dev):
        dst = torch.empty((5, P), dtype=torch.int32, device=dev)
        totals = torch.zeros(2, dtype=torch.int32, device=dev)
        nbytes = L.gsr_densify_plan_bytes(P)
        ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        use_screen = bool(max_screen_size)
        rc = L.gsr_densify_plan(P, accum.data_ptr(), denom.data_ptr(), scaling.data_ptr(), opacity.data_ptr(), _f32(max_grad),
                                _f32(_times(percent_dense, extent)), _f32(min_opacity), int(use_screen),
                                _f32(max_screen_size) if use_screen else 0.0, _f32(_times(0.1, extent)), dst.data_ptr(), totals.data_ptr(),
                                ws.data_ptr(), nbytes, stream)
        _lib.check(rc, "gsr_densify_plan")
        S, P2 = totals.tolist()  # the one host synchronisation: P' sizes the new tensors
        # torch.normal(mean=0, std) draws normal_(0, 1) into a [2S, 3] tensor: the same values and the same generator advance
        eps = torch.randn((2 * S, 3), device=dev)
        out, structs = {}, []
        for name, role, g, p, st in found:
            new = torch.empty((P2,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
            m = [None, None]
            if st is not None:
                m = [torch.empty_like(new), torch.empty_like(new)]
            width = int(np.prod(p.shape[1:], dtype=np.int64))
            structs.append(_lib.gsr_densify_group(p.data_ptr(), new.data_ptr(),
                                                  st["exp_avg"].data_ptr() if st is not None else None, _ptr(m[0]),
                                                  st["exp_avg_sq"].data_ptr() if st is not None else None, _ptr(m[1]), width, role))
            out[name] = (g, p, st, new, m)
        arr = (_lib.gsr_densify_group * max(len(structs), 1))(*structs)
        rc = 0 if P2 == 0 else L.gsr_densify_apply(P, S, len(structs), arr, dst.data_ptr(), xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(),
                                 eps.data_ptr(), rotation_mode, stream)
        _lib.check(rc, "gsr_densify_apply")  # P' = 0: every row pruned, nothing to write
    params = {}
    for name, (g, p, st, new, m) in out.items():
        param = nn.Parameter(new.requires_grad_(True))
        if st is not None:
            st["exp_avg"], st["exp_avg_sq"] = m
            del optimizer.state[p]
            optimizer.state[param] = st
        g["params"][0] = param
        params[name] = param
    return params, P2


def _ptr(t):
    return None if t is None else t.data_ptr()


def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size):
    """GaussianModel.densify_and_prune (GS/:399-413) in CUDA: clone, split and the final prune in one pass over every parameter
    and both Adam moments, in the reference's row order, with the same draws from the CUDA generator.  The optimizer's param
    groups hold the new nn.Parameters, its state is re-keyed (the same dict, its ``step`` kept), the model attributes are
    re-assigned and xyz_gradient_accum, denom and max_radii2D are zeros of the new size.  Unlike the reference it does not call
    torch.cuda.empty_cache(): memory the caching allocator keeps is the only observable difference.

    Raises ValueError, naming the argument, for a missing param group or a non-float32 or non-contiguous leaf; RuntimeError for
    CPU tensors (there is no CPU path)."""
    who = "densify_and_prune"
    params, P2 = _run(who, self.optimizer, [(n, r) for n, _, r in _GS_GROUPS], self.xyz_gradient_accum, self.denom, self._scaling,
                      self._opacity, self._xyz, self._rotation, _lib.GSR_DENSIFY_ROTATION_3DGS, max_grad, min_opacity, extent,
                      max_screen_size, self.percent_dense)
    for name, attr, _ in _GS_GROUPS:
        setattr(self, attr, params[name])
    dev = self._xyz.device
    self.xyz_gradient_accum = torch.zeros((P2, 1), device=dev)
    self.denom = torch.zeros((P2, 1), device=dev)
    self.max_radii2D = torch.zeros((P2,), device=dev)


def sugar_densify_and_prune(self, max_grad=None, min_opacity=None, extent=None, max_screen_size=None):
    """SuGaRDensifier.densify_and_prune (SD/:228-244) in CUDA, as densify_and_prune above: the None defaults come from the
    densifier (max_grad, min_opacity, scene_extent), only the groups in ``params_to_densify`` are rebuilt, the prune reads
    ``strengths`` (sigmoid of all_densities) and split children are placed with pytorch3d's quaternion_to_matrix of the normalised
    quaternions.  Raises ValueError for a model bound to a surface mesh."""
    who = "sugar_densify_and_prune"
    model = self.model
    if getattr(model, "binded_to_surface_mesh", False):
        raise ValueError("%s: a model bound to a surface mesh is not supported" % who)
    max_grad = self.max_grad if max_grad is None else max_grad
    min_opacity = self.min_opacity if min_opacity is None else min_opacity
    extent = self.scene_extent if extent is None else extent
    wanted = [(n, r) for n, _, r in _SUGAR_GROUPS if n in self.params_to_densify]
    params, P2 = _run(who, self.optimizer, wanted, self.points_gradient_accum, self.denom, model._scales, model.all_densities,
                      model._points, model._quaternions, _lib.GSR_DENSIFY_ROTATION_SUGAR, max_grad, min_opacity, extent,
                      max_screen_size, self.percent_dense)
    for name, attr, _ in _SUGAR_GROUPS:
        if name in params:
            setattr(model, attr, params[name])
    dev = model._points.device
    self.points_gradient_accum = torch.zeros((P2, 1), device=dev)
    self.denom = torch.zeros((P2, 1), device=dev)
    self.max_radii2D = torch.zeros((P2,), device=dev)
