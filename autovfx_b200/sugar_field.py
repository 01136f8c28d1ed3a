"""SuGaR's SDF-regularisation field in CUDA: drop-ins for ``SuGaR.get_field_values`` and ``SuGaR.compute_density``
("SS/" = sugar/sugar_scene/sugar_model.py:1118-1187 and :1216-1239, with get_covariance :602-608 and get_beta 'average'
:1063-1066), forward and backward through ``gsr_sugar_field`` / ``gsr_sugar_field_backward``.

Opt in on the class (both take the methods' exact signatures and return what they return)::

    from autovfx_b200.sugar_field import get_field_values, compute_density
    SuGaR.get_field_values = get_field_values
    SuGaR.compute_density = compute_density

The coarse trainers' projection estimate and better-normal loss ("CD/" = sugar/sugar_trainers/coarse_density.py:704-707 and
:756-780) run through ``gsr_sugar_sdf_normal`` / ``gsr_sugar_sdf_normal_backward``; the trainer calls them in place of those lines::

    from autovfx_b200.sugar_field import projection_estimate, better_normal_loss
    sdf_estimation = projection_estimate(sugar, sdf_samples, sdf_gaussian_idx)
    sdf_better_normal_loss = better_normal_loss(sugar, sdf_samples, sdf_gaussian_idx, fields['closest_gaussian_opacities'])

SuGaR's sampler of the SDF-regularisation points (SS/:757-799) runs through ``gsr_sugar_sample`` / ``gsr_sugar_sample_backward``::

    from autovfx_b200.sugar_field import sample_points_in_gaussians
    SuGaR.sample_points_in_gaussians = sample_points_in_gaussians

coarse_sdf's depth-map estimate ("CS/" = sugar/sugar_trainers/coarse_sdf.py: the close-to-surface mask :655-665 and the 'sdf'
estimation loss :689-712) runs through ``gsr_sugar_surface_mask`` and ``gsr_sugar_depth_sdf_loss`` / ``..._backward``::

    from autovfx_b200.sugar_field import close_to_surface_mask, depth_sdf_estimation_loss
    gaussians_close_to_surface = close_to_surface_mask(sugar, fov_camera, depth, close_gaussian_threshold)
    loss = loss + sdf_estimation_factor * depth_sdf_estimation_loss(sugar, fov_camera, depth, sdf_samples, fields['sdf'],
                                                                    sdf_sample_std, 10. * sugar.get_cameras_spatial_extent())

coarse_density's 'density' SDF estimation loss ("CD/" :735-741, the same at coarse_sdf.py:714-720) runs through
``gsr_density_estimation_loss`` / ``..._backward`` when ``proj_mask`` is all true (use_projection_as_estimation, the default)::

    from autovfx_b200.sugar_field import density_estimation_loss
    loss = loss + sdf_estimation_factor * density_estimation_loss(fields['density'], fields['beta'], sdf_estimation,
                                                                  squared_sdf_estimation_loss)

The model is read through its getters (``points``, ``scaling``, ``quaternions``, ``strengths``, ``knn_idx``, ``beta_mode``), so
autograd carries the gradients of x and of the getters' outputs back to the raw parameters.  No [N,K,3,3] tensor is built: the
kernels gather one 64-byte record per (sample, neighbour) pair and recompute everything in the backward.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

__all__ = ["get_field_values", "compute_density", "projection_estimate", "better_normal_loss", "sample_points_in_gaussians",
           "close_to_surface_mask", "depth_sdf_estimation_loss", "density_estimation_loss", "FIELD_MAX_K"]

FIELD_MAX_K = 32


def _lib_handle():
    return _lib.lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _check_tensor(who, name, t, shape, dtype):
    """shape: a tuple of ints or None (any size) per dimension."""
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s: %s must be a torch.Tensor, got %s" % (who, name, type(t).__name__))
    if t.dtype != dtype:
        raise ValueError("%s: %s must be %s, got %s" % (who, name, dtype, t.dtype))
    if t.dim() != len(shape) or any(s is not None and s != d for s, d in zip(shape, t.shape)):
        want = "[" + ", ".join("*" if s is None else str(s) for s in shape) + "]"
        raise ValueError("%s: %s must have shape %s, got %s" % (who, name, want, tuple(t.shape)))


def _model_tensors(who, self):
    points, scaling, quaternions, strengths = self.points, self.scaling, self.quaternions, self.strengths
    _check_tensor(who, "self.points", points, (None, 3), torch.float32)
    P = points.shape[0]
    _check_tensor(who, "self.scaling", scaling, (P, 3), torch.float32)
    _check_tensor(who, "self.quaternions", quaternions, (P, 4), torch.float32)
    if not isinstance(strengths, torch.Tensor) or strengths.shape not in ((P, 1), (P,)):
        raise ValueError("%s: self.strengths must have shape [%d, 1], got %s" % (who, P, getattr(strengths, "shape", None)))
    _check_tensor(who, "self.strengths", strengths, tuple(strengths.shape), torch.float32)
    return points, scaling, quaternions, strengths.reshape(P)


def _require_cuda(who, *ts):
    dev = ts[0].device
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("autovfx_b200.%s: every tensor must be a CUDA tensor (there is no CPU path)" % who)
    for t in ts:
        if t is not None and t.device != dev:
            raise ValueError("%s: tensors on %s and %s" % (who, dev, t.device))


class _Cfg:
    __slots__ = ("N", "K", "P", "R", "df", "omc", "offset", "opac", "beta", "sdf")

    def __init__(self, N, K, P, R, df, omc, offset, opac, beta, sdf):
        self.N, self.K, self.P, self.R = N, K, P, R
        self.df, self.omc, self.offset = df, omc, offset
        self.opac, self.beta, self.sdf = opac, beta, sdf


def _forward(cfg, x, rows, row_idx, points, scaling, quaternions, strengths):
    dev = x.device
    N, K = cfg.N, cfg.K
    density = torch.empty(N, dtype=torch.float32, device=dev)
    opac = torch.empty((N, K), dtype=torch.float32, device=dev) if cfg.opac else None
    beta = torch.empty(N, dtype=torch.float32, device=dev) if cfg.beta else None
    sdf = torch.empty(N, dtype=torch.float32, device=dev) if cfg.sdf else None
    if N > 0:
        L = _lib_handle()
        nbytes = L.gsr_sugar_field_bytes(cfg.P)
        ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        rc = L.gsr_sugar_field(N, K, cfg.P, cfg.R, x.data_ptr(), rows.data_ptr(), _ptr(row_idx), points.data_ptr(), scaling.data_ptr(),
                               quaternions.data_ptr(), strengths.data_ptr(), cfg.df, cfg.omc, cfg.offset, density.data_ptr(),
                               _ptr(opac), _ptr(beta), _ptr(sdf), ws.data_ptr(), nbytes, _lib.stream_ptr(dev))
        _lib.check(rc, "gsr_sugar_field")
    return density, opac, beta, sdf


class _SugarField(torch.autograd.Function):
    """Outputs: density, then neighbour opacities, beta and sdf when the configuration asks for them."""

    @staticmethod
    def forward(ctx, x, points, scaling, quaternions, strengths, rows, row_idx, cfg):
        ctx.set_materialize_grads(False)
        ctx.cfg = cfg
        ctx.save_for_backward(x, points, scaling, quaternions, strengths, rows, row_idx)
        density, opac, beta, sdf = _forward(cfg, x, rows, row_idx, points, scaling, quaternions, strengths)
        return tuple(t for t in (density, opac, beta, sdf) if t is not None)

    @staticmethod
    def backward(ctx, *grads):
        cfg = ctx.cfg
        x, points, scaling, quaternions, strengths, rows, row_idx = ctx.saved_tensors
        it = iter(grads)
        g_density = next(it)
        g_opac = next(it) if cfg.opac else None
        g_beta = next(it) if cfg.beta else None
        g_sdf = next(it) if cfg.sdf else None
        g = [None if t is None else t.contiguous() for t in (g_density, g_opac, g_beta, g_sdf)]
        dev = x.device
        P, N = cfg.P, cfg.N
        dx = torch.zeros_like(x) if ctx.needs_input_grad[0] else None
        d_points = torch.zeros_like(points)
        d_scaling = torch.zeros_like(scaling)
        d_quaternions = torch.zeros_like(quaternions)
        d_strengths = torch.zeros_like(strengths)
        if N > 0 and any(t is not None for t in g):
            L = _lib_handle()
            if torch.are_deterministic_algorithms_enabled():  # fixed-order sums (DESIGN §4), no atomics
                fn, what = L.gsr_sugar_field_backward_det, "gsr_sugar_field_backward_det"
                nbytes = L.gsr_sugar_field_backward_det_bytes(N, cfg.K, P)
                ws = _lib.scratch_bytes(nbytes, dev)
            else:
                fn, what = L.gsr_sugar_field_backward, "gsr_sugar_field_backward"
                nbytes = 2 * L.gsr_sugar_field_bytes(P)
                ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
            rc = fn(N, cfg.K, P, cfg.R, x.data_ptr(), rows.data_ptr(), _ptr(row_idx), points.data_ptr(), scaling.data_ptr(),
                    quaternions.data_ptr(), strengths.data_ptr(), cfg.df, cfg.omc, cfg.offset, *[_ptr(t) for t in g], _ptr(dx),
                    d_points.data_ptr(), d_scaling.data_ptr(), d_quaternions.data_ptr(), d_strengths.data_ptr(), ws.data_ptr(), nbytes,
                    _lib.stream_ptr(dev))
            _lib.check(rc, what)
        need = ctx.needs_input_grad
        return (dx, d_points if need[1] else None, d_scaling if need[2] else None, d_quaternions if need[3] else None,
                d_strengths if need[4] else None, None, None, None)


def _field(who, self, x, rows, row_idx, density_factor, opacity_min_clamp, offset, opac, beta, sdf):
    """Validated inputs -> (density, opac or None, beta or None, sdf or None)."""
    points, scaling, quaternions, strengths = _model_tensors(who, self)
    _check_tensor(who, "x", x, (None, 3), torch.float32)
    N, P = x.shape[0], points.shape[0]
    _check_tensor(who, "closest_gaussians_idx" if row_idx is None else "self.knn_idx", rows, (None, None), torch.int64)
    R, K = rows.shape
    if not 1 <= K <= FIELD_MAX_K:
        raise ValueError("%s: K = %d neighbours per sample must be in 1..%d" % (who, K, FIELD_MAX_K))
    if row_idx is None and R != N:
        raise ValueError("%s: closest_gaussians_idx has %d rows for %d samples" % (who, R, N))
    for name, v in (("density_factor", density_factor), ("opacity_min_clamp", opacity_min_clamp)):
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            raise ValueError("%s: %s must be a Python number, got %r" % (who, name, v))
    _require_cuda(who, x, rows, row_idx, points, scaling, quaternions, strengths)
    cfg = _Cfg(N, K, P, R, float(density_factor), float(opacity_min_clamp), offset, opac, beta, sdf)
    rows = rows.contiguous()
    row_idx = None if row_idx is None else row_idx.contiguous()
    ins = [t.contiguous() for t in (x, points, scaling, quaternions, strengths)]
    with torch.cuda.device(x.device):
        if torch.is_grad_enabled() and any(t.requires_grad for t in ins):
            outs = iter(_SugarField.apply(*ins, rows, row_idx, cfg))
            return tuple(next(outs) if want else None for want in (True, opac, beta, sdf))
        return _forward(cfg, ins[0], rows, row_idx, *ins[1:])


def get_field_values(self, x, gaussian_idx=None, closest_gaussians_idx=None, gaussian_strengths=None, gaussian_centers=None,
                     gaussian_inv_scaled_rotation=None, return_sdf=True, density_threshold=1., density_factor=1.,
                     return_sdf_grad=False, sdf_grad_max_value=10., opacity_min_clamp=1e-16, return_closest_gaussian_opacities=False,
                     return_beta=False):
    """SuGaR.get_field_values (SS/:1118-1187) in CUDA.  Returns SuGaR's dict: 'density' (the sum before the d >= 1
    normalisation), then 'closest_gaussian_opacities' [N,K], 'beta' and 'sdf' as requested.  The neighbours are
    closest_gaussians_idx [N,K] or, when it is None, self.knn_idx[gaussian_idx] (read in place, never gathered).

    Raises ValueError, naming the argument, for what no SuGaR caller uses: return_sdf_grad=True, the gaussian_strengths /
    gaussian_centers / gaussian_inv_scaled_rotation overrides, a beta_mode other than 'average' when beta or the sdf is asked for,
    both indices None, bad shapes or dtypes, K outside 1..32.  CPU tensors raise RuntimeError (there is no CPU path)."""
    who = "get_field_values"
    if return_sdf_grad:
        raise ValueError("get_field_values: return_sdf_grad=True is not supported (no SuGaR trainer asks for sdf_grad)")
    for name, v in (("gaussian_strengths", gaussian_strengths), ("gaussian_centers", gaussian_centers),
                    ("gaussian_inv_scaled_rotation", gaussian_inv_scaled_rotation)):
        if v is not None:
            raise ValueError("get_field_values: the %s override is not supported (pass None: the model's getters are used)" % name)
    want_beta = bool(return_sdf or return_beta)
    if want_beta:
        mode = self.beta_mode
        if mode in ("learnable", "weighted_average"):
            raise ValueError("get_field_values: beta_mode = %r is not supported (only 'average')" % (mode,))
        if mode != "average":
            raise ValueError("Unknown beta_mode.")
    if closest_gaussians_idx is not None:
        rows, row_idx = closest_gaussians_idx, None
    elif gaussian_idx is not None:
        rows = self.knn_idx
        _check_tensor(who, "self.knn_idx", rows, (None, None), torch.int64)
        _check_tensor(who, "gaussian_idx", gaussian_idx, (None,), torch.int64)
        row_idx = gaussian_idx
        if isinstance(x, torch.Tensor) and x.dim() == 2 and gaussian_idx.shape[0] != x.shape[0]:
            raise ValueError("get_field_values: gaussian_idx has %d entries for %d samples" % (gaussian_idx.shape[0], x.shape[0]))
    else:
        raise ValueError("get_field_values: gaussian_idx and closest_gaussians_idx are both None")
    offset = float(np.float32(np.sqrt(-2. * np.log(min(density_threshold, 1.))))) if return_sdf else 0.0
    density, opac, beta, sdf = _field(who, self, x, rows, row_idx, density_factor, opacity_min_clamp, offset,
                                      bool(return_closest_gaussian_opacities), want_beta, bool(return_sdf))
    fields = {"density": density}
    if return_closest_gaussian_opacities:
        fields["closest_gaussian_opacities"] = opac
    if return_beta:
        fields["beta"] = beta
    if return_sdf:
        fields["sdf"] = sdf
    return fields


def compute_density(self, x, closest_gaussians_idx=None, density_factor=1., return_closest_gaussian_opacities=False):
    """SuGaR.compute_density (SS/:1216-1239) in CUDA: densities [N] (and the neighbour opacities [N,K]).  Without indices it
    calls self.get_gaussians_closest_to_samples(x), so the model's knn_points binding applies."""
    if closest_gaussians_idx is None:
        closest_gaussians_idx = self.get_gaussians_closest_to_samples(x)
    density, opac, _, _ = _field("compute_density", self, x, closest_gaussians_idx, None, density_factor, 1e-16, 0.0,
                                 bool(return_closest_gaussian_opacities), False, False)
    if return_closest_gaussian_opacities:
        return density, opac
    return density


# ------------------------------------------------------------------------------------------------ better-normal loss, estimate
def _sdf_normal_forward(want_loss, K, x, gidx, knn, points, scaling, quaternions, opac):
    N, P = x.shape[0], points.shape[0]
    out = torch.empty(N, dtype=torch.float32, device=x.device)
    if N > 0:
        L = _lib_handle()
        nbytes = L.gsr_sugar_sdf_normal_bytes(P)
        ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=x.device)
        rc = L.gsr_sugar_sdf_normal(N, K, P, x.data_ptr(), gidx.data_ptr(), _ptr(knn), points.data_ptr(), scaling.data_ptr(),
                                    quaternions.data_ptr(), _ptr(opac), out.data_ptr() if want_loss else None,
                                    None if want_loss else out.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr(x.device))
        _lib.check(rc, "gsr_sugar_sdf_normal")
    return out


class _SugarSdfNormal(torch.autograd.Function):
    """One output: the better-normal loss [N] (want_loss) or the projection estimate [N]."""

    @staticmethod
    def forward(ctx, x, points, quaternions, scaling, gidx, knn, opac, want_loss, K):
        ctx.set_materialize_grads(False)
        ctx.want_loss, ctx.K = want_loss, K
        ctx.save_for_backward(x, points, quaternions, scaling, gidx, knn, opac)
        return _sdf_normal_forward(want_loss, K, x, gidx, knn, points, scaling, quaternions, opac)

    @staticmethod
    def backward(ctx, g):
        x, points, quaternions, scaling, gidx, knn, opac = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx = torch.zeros_like(x) if need[0] else None
        d_points = torch.zeros_like(points)
        d_quaternions = torch.zeros_like(quaternions)
        N, P = x.shape[0], points.shape[0]
        if N > 0 and g is not None:
            g = g.contiguous()
            L = _lib_handle()
            if torch.are_deterministic_algorithms_enabled():  # fixed-order sums (DESIGN §4), no atomics
                fn, what = L.gsr_sugar_sdf_normal_backward_det, "gsr_sugar_sdf_normal_backward_det"
                nbytes = L.gsr_sugar_sdf_normal_backward_det_bytes(N, ctx.K, P, int(ctx.want_loss))
                ws = _lib.scratch_bytes(nbytes, x.device)
            else:
                fn, what = L.gsr_sugar_sdf_normal_backward, "gsr_sugar_sdf_normal_backward"
                nbytes = 2 * L.gsr_sugar_sdf_normal_bytes(P)
                ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=x.device)
            rc = fn(N, ctx.K, P, x.data_ptr(), gidx.data_ptr(), _ptr(knn), points.data_ptr(), scaling.data_ptr(), quaternions.data_ptr(),
                    _ptr(opac), g.data_ptr() if ctx.want_loss else None, None if ctx.want_loss else g.data_ptr(), _ptr(dx),
                    d_points.data_ptr(), d_quaternions.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr(x.device))
            _lib.check(rc, what)
        return (dx, d_points if need[1] else None, d_quaternions if need[2] else None, None, None, None, None, None, None)


def _sdf_normal(who, self, sdf_samples, sdf_gaussian_idx, opacities, want_loss):
    if getattr(self, "binded_to_surface_mesh", False):
        raise ValueError("%s: a model bound to a surface mesh is not supported (its normals are face normals; the refinement runs "
                         "with regularize_sdf = False)" % who)
    points, scaling, quaternions, _ = _model_tensors(who, self)
    P = points.shape[0]
    _check_tensor(who, "sdf_samples", sdf_samples, (None, 3), torch.float32)
    N = sdf_samples.shape[0]
    _check_tensor(who, "sdf_gaussian_idx", sdf_gaussian_idx, (N,), torch.int64)
    knn = opac = None
    K = 1
    if want_loss:
        knn = self.knn_idx
        _check_tensor(who, "self.knn_idx", knn, (P, None), torch.int64)
        K = knn.shape[1]
        if not 1 <= K <= FIELD_MAX_K:
            raise ValueError("%s: K = %d neighbours per Gaussian must be in 1..%d" % (who, K, FIELD_MAX_K))
        _check_tensor(who, "closest_gaussian_opacities", opacities, (N, K), torch.float32)
        knn = knn.contiguous()
        opac = opacities.detach().contiguous()
    _require_cuda(who, sdf_samples, sdf_gaussian_idx, knn, opac, points, scaling, quaternions)
    gidx = sdf_gaussian_idx.contiguous()
    x, points, quaternions = (t.contiguous() for t in (sdf_samples, points, quaternions))
    scaling = scaling.detach().contiguous()
    with torch.cuda.device(x.device):
        diff = (quaternions,) if want_loss else (x, points, quaternions)
        if torch.is_grad_enabled() and any(t.requires_grad for t in diff):
            if want_loss:  # the loss carries no gradient to the samples or the centres
                x, points = x.detach(), points.detach()
            return _SugarSdfNormal.apply(x, points, quaternions, scaling, gidx, knn, opac, want_loss, K)
        return _sdf_normal_forward(want_loss, K, x, gidx, knn, points, scaling, quaternions, opac)


def projection_estimate(self, sdf_samples, sdf_gaussian_idx):
    """The coarse trainers' projection estimate (CD/:706-707) in CUDA: ((sdf_samples - points[i]) * normals[i]).sum(-1) with
    i = sdf_gaussian_idx and normals = self.get_normals() (the smallest axis).  Returns [N], differentiable with respect to the
    samples, ``points`` and ``quaternions``.

    Raises ValueError, naming the argument, for a wrong shape or dtype or a model bound to a surface mesh; RuntimeError for CPU
    tensors (there is no CPU path)."""
    return _sdf_normal("projection_estimate", self, sdf_samples, sdf_gaussian_idx, None, False)


def better_normal_loss(self, sdf_samples, sdf_gaussian_idx, closest_gaussian_opacities):
    """The coarse trainers' better-normal loss per sample (CD/:756-780, before the trainer's ``.mean()``) in CUDA, over the
    neighbours self.knn_idx[sdf_gaussian_idx] (read in place, never gathered) weighted by closest_gaussian_opacities [N,K]
    (read detached).  Returns [N], differentiable with respect to ``quaternions`` only: the trainer's
    sdf_better_normal_gradient_through_normal_only detaches the weights, so the samples, points and scales get nothing.

    Raises ValueError, naming the argument, for wrong shapes, dtypes or widths (the opacities' K must equal knn_idx's), K outside
    1..32 and a model bound to a surface mesh; RuntimeError for CPU tensors (there is no CPU path)."""
    return _sdf_normal("better_normal_loss", self, sdf_samples, sdf_gaussian_idx, closest_gaussian_opacities, True)


# ------------------------------------------------------------------------------------------------ SDF-regularisation samples
def _sample_forward(N, f, volume, mask, strengths, u, z, points, scaling, quaternions):
    dev, P = points.device, points.shape[0]
    out = torch.empty((N, 3), dtype=torch.float32, device=dev)
    idx = torch.empty(N, dtype=torch.int64, device=dev)
    total = torch.empty(1, dtype=torch.float64, device=dev)
    L = _lib_handle()
    nbytes = L.gsr_sugar_sample_bytes(P)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    rc = L.gsr_sugar_sample(N, P, f, int(volume), _ptr(mask), _ptr(strengths), u.data_ptr(), z.data_ptr(), points.data_ptr(),
                            scaling.data_ptr(), quaternions.data_ptr(), out.data_ptr(), idx.data_ptr(), total.data_ptr(),
                            ws.data_ptr(), nbytes, _lib.stream_ptr(dev))
    _lib.check(rc, "gsr_sugar_sample")
    return out, idx, total


class _SugarSample(torch.autograd.Function):
    """Outputs: the samples [N,3] (differentiable with respect to points, scaling and quaternions) and their rows [N]."""

    @staticmethod
    def forward(ctx, points, scaling, quaternions, N, f, volume, mask, strengths, u, z):
        ctx.set_materialize_grads(False)
        out, idx, total = _sample_forward(N, f, volume, mask, strengths, u, z, points, scaling, quaternions)
        ctx.f = f
        ctx.mark_non_differentiable(idx)
        ctx.save_for_backward(scaling, quaternions, z, idx, total)
        return out, idx

    @staticmethod
    def backward(ctx, g, _g_idx):
        scaling, quaternions, z, idx, total = ctx.saved_tensors
        need = ctx.needs_input_grad
        if g is None:
            return (None,) * 10
        g = g.contiguous()
        N, P = idx.shape[0], scaling.shape[0]
        d_points = torch.empty((P, 3), dtype=torch.float32, device=g.device)
        d_scaling = torch.empty((P, 3), dtype=torch.float32, device=g.device)
        d_quaternions = torch.empty((P, 4), dtype=torch.float32, device=g.device)
        L = _lib_handle()
        args = (N, P, ctx.f, idx.data_ptr(), z.data_ptr(), scaling.data_ptr(), quaternions.data_ptr(), total.data_ptr(), g.data_ptr(),
                d_points.data_ptr(), d_scaling.data_ptr(), d_quaternions.data_ptr())
        if torch.are_deterministic_algorithms_enabled():  # fixed-order sums (DESIGN §4), no atomics
            nbytes = L.gsr_sugar_sample_backward_det_bytes(N, P)
            scratch = _lib.scratch_bytes(nbytes, g.device)
            rc = L.gsr_sugar_sample_backward_det(*args, scratch.data_ptr(), nbytes, _lib.stream_ptr(g.device))
            _lib.check(rc, "gsr_sugar_sample_backward_det")
        else:
            rc = L.gsr_sugar_sample_backward(*args, _lib.stream_ptr(g.device))
            _lib.check(rc, "gsr_sugar_sample_backward")
        return (d_points if need[0] else None, d_scaling if need[1] else None, d_quaternions if need[2] else None,
                None, None, None, None, None, None, None)


def sample_points_in_gaussians(self, num_samples, sampling_scale_factor=1., mask=None, probabilities_proportional_to_opacity=False,
                               probabilities_proportional_to_volume=True):
    """SuGaR.sample_points_in_gaussians (SS/:757-799) in CUDA: (random_points [N,3] float32, random_indices [N] int64), the indices
    being rows of the model (as after SuGaR's valid_indices[...]).  Selected rows are mask's True rows (all rows when mask is None);
    a selected row's weight w is |s0 * s1 * s2| (or 1 without probabilities_proportional_to_volume), times strengths with
    probabilities_proportional_to_opacity.  As in SuGaR, whose torch.multinomial is handed cumsum(w) / sum(w) as the weights,
    selected row k is drawn with probability proportional to the cumulative weight C_k = sum of w up to k (float64 here).  Each
    sample is points[i] + quaternion_apply(quaternions[i], (sampling_scale_factor * scaling[i]) * z), z ~ N(0, 1)^3, pytorch3d's
    quaternion_apply op for op.  random_points is differentiable with respect to the getters' points, scaling and quaternions; the
    weights get no gradient.

    The draws come from the CUDA generator of the points' device, in this order: u = torch.rand(N, dtype=float64) (row i is the
    first whose float64 prefix of C over the selected rows exceeds u * total), then z = torch.randn(N, 3).  torch.manual_seed
    controls a run; the samples for a seed differ from SuGaR's (which draws through torch.multinomial), the distribution is the
    same.  Nothing is read back to the host.  An empty selection, or a zero or non-finite total, gives index 0 and NaN samples
    (SuGaR asserts on the device; its trainers call it only when the mask has a True row).

    Raises ValueError, naming the argument, for num_samples < 1, a wrong shape or dtype (float32 getters, a bool mask [P]) or a
    model without rows; RuntimeError for CPU tensors (there is no CPU path)."""
    who = "sample_points_in_gaussians"
    if isinstance(num_samples, bool) or not isinstance(num_samples, (int, np.integer)) or num_samples < 1:
        raise ValueError("%s: num_samples must be an int >= 1, got %r" % (who, num_samples))
    if isinstance(sampling_scale_factor, bool) or not isinstance(sampling_scale_factor, (int, float)):
        raise ValueError("%s: sampling_scale_factor must be a Python number, got %r" % (who, sampling_scale_factor))
    points, scaling, quaternions = self.points, self.scaling, self.quaternions
    _check_tensor(who, "self.points", points, (None, 3), torch.float32)
    P = points.shape[0]
    if P < 1:
        raise ValueError("%s: self.points has no rows" % who)
    _check_tensor(who, "self.scaling", scaling, (P, 3), torch.float32)
    _check_tensor(who, "self.quaternions", quaternions, (P, 4), torch.float32)
    strengths = None
    if probabilities_proportional_to_opacity:
        strengths = self.strengths
        if not isinstance(strengths, torch.Tensor) or strengths.shape not in ((P, 1), (P,)):
            raise ValueError("%s: self.strengths must have shape [%d, 1], got %s" % (who, P, getattr(strengths, "shape", None)))
        _check_tensor(who, "self.strengths", strengths, tuple(strengths.shape), torch.float32)
        strengths = strengths.detach().reshape(P).contiguous()
    if mask is not None:
        _check_tensor(who, "mask", mask, (P,), torch.bool)
    _require_cuda(who, points, scaling, quaternions, strengths, mask)
    N = int(num_samples)
    f = float(sampling_scale_factor)
    dev = points.device
    mask = None if mask is None else mask.contiguous()
    ins = [t.contiguous() for t in (points, scaling, quaternions)]
    with torch.cuda.device(dev):
        u = torch.rand(N, dtype=torch.float64, device=dev)
        z = torch.randn((N, 3), dtype=torch.float32, device=dev)
        if torch.is_grad_enabled() and any(t.requires_grad for t in ins):
            return _SugarSample.apply(*ins, N, f, bool(probabilities_proportional_to_volume), mask, strengths, u, z)
        out, idx, _ = _sample_forward(N, f, probabilities_proportional_to_volume, mask, strengths, u, z, *ins)
        return out, idx


# ------------------------------------------------------------------------------------------------ coarse_sdf's depth-map estimate
def _number(who, name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)):
        raise ValueError("%s: %s must be a Python number, got %r" % (who, name, v))
    return float(v)


def _depth_map(who, self, depth):
    """(H, W, stride_h, stride_w, sx, sy) of the depth view; sx, sy are SuGaR's factor / image_width and factor / image_height
    (SS/:1193-1196), Python doubles rounded to float32 as torch rounds a Python scalar that multiplies a float32 tensor."""
    if not isinstance(depth, torch.Tensor) or depth.dim() != 2 or depth.dtype != torch.float32:
        raise ValueError("%s: depth must be a float32 [H, W] tensor, got %s" % (who, getattr(depth, "shape", type(depth).__name__)))
    H, W = depth.shape
    if H < 1 or W < 1:
        raise ValueError("%s: depth must not be empty, got %s" % (who, tuple(depth.shape)))
    h_img, w_img = getattr(self, "image_height", None), getattr(self, "image_width", None)
    for name, v in (("self.image_height", h_img), ("self.image_width", w_img)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise ValueError("%s: %s must be a positive int, got %r" % (who, name, v))
    factor = -1 * min(h_img, w_img)
    return H, W, depth.stride(0), depth.stride(1), float(np.float32(factor / w_img)), float(np.float32(factor / h_img))


def _camera(who, fov_camera, dev, with_center):
    """[36] float32 on dev: get_world_to_view_transform().get_matrix(), get_projection_transform().get_matrix(), znear and
    get_camera_center(), read through pytorch3d's own methods and concatenated on the device (nothing is read back).  Only the
    mask reads the centre: without with_center its three floats are zeros and get_camera_center() is not called."""
    w2v = fov_camera.get_world_to_view_transform().get_matrix()
    proj = fov_camera.get_projection_transform().get_matrix()
    center = fov_camera.get_camera_center() if with_center else torch.zeros(3, dtype=torch.float32, device=dev)
    znear = fov_camera.znear
    for name, t, n in (("get_world_to_view_transform().get_matrix()", w2v, 16), ("get_projection_transform().get_matrix()", proj, 16),
                       ("get_camera_center()", center, 3)):
        if not isinstance(t, torch.Tensor) or t.numel() != n or t.dtype != torch.float32:
            raise ValueError("%s: fov_camera.%s must be one camera's float32 tensor of %d values, got %s"
                             % (who, name, n, getattr(t, "shape", type(t).__name__)))
    if isinstance(znear, torch.Tensor):
        if znear.numel() != 1 or znear.dtype != torch.float32:
            raise ValueError("%s: fov_camera.znear must be one float32 value, got %s" % (who, tuple(znear.shape)))
        _require_cuda(who, w2v, proj, center, znear)
        znear = znear.detach().reshape(1)
    else:
        _require_cuda(who, w2v, proj, center)
        znear = torch.full((1,), _number(who, "fov_camera.znear", znear), dtype=torch.float32, device=w2v.device)
    if w2v.device != dev:
        raise ValueError("%s: the camera is on %s and the model on %s" % (who, w2v.device, dev))
    return torch.cat([t.detach().reshape(-1) for t in (w2v, proj, znear, center)])


def _surface_mask(self, fov_camera, depth, close_gaussian_threshold, want_map_z):
    who = "close_to_surface_mask"
    thr = _number(who, "close_gaussian_threshold", close_gaussian_threshold)
    points, scaling, quaternions = self.points, self.scaling, self.quaternions
    _check_tensor(who, "self.points", points, (None, 3), torch.float32)
    P = points.shape[0]
    _check_tensor(who, "self.scaling", scaling, (P, 3), torch.float32)
    _check_tensor(who, "self.quaternions", quaternions, (P, 4), torch.float32)
    H, W, sh, sw, sx, sy = _depth_map(who, self, depth)
    _require_cuda(who, points, scaling, quaternions, depth)
    dev = points.device
    with torch.cuda.device(dev):
        cam = _camera(who, fov_camera, dev, True)
        points, scaling, quaternions = (t.detach().contiguous() for t in (points, scaling, quaternions))
        mask = torch.empty(P, dtype=torch.bool, device=dev)
        map_z = torch.empty(P, dtype=torch.float32, device=dev) if want_map_z else None
        rc = _lib_handle().gsr_sugar_surface_mask(P, H, W, sh, sw, depth.data_ptr(), sx, sy, cam.data_ptr(), points.data_ptr(),
                                                  scaling.data_ptr(), quaternions.data_ptr(), float(np.float32(thr)), mask.data_ptr(),
                                                  _ptr(map_z), _lib.stream_ptr(dev))
        _lib.check(rc, "gsr_sugar_surface_mask")
    return mask, map_z


def close_to_surface_mask(self, fov_camera, depth, close_gaussian_threshold=2.):
    """coarse_sdf's gaussians_close_to_surface (CS/:655-666) in CUDA: bool [P], True where |map_z(p) - z| < threshold *
    |scaling * quaternion_apply(quaternion_invert(q), normalize(c - p))|, with z the depth of the centre p in the camera and map_z
    the rendered depth there (SuGaR.get_points_depth_in_depth_map, SS/:1189-1204).  ``depth`` is the [H, W] depth render (a strided
    channel view is read in place); the camera is read through pytorch3d's get_world_to_view_transform(),
    get_projection_transform(), znear and get_camera_center().  No gradient, as under the trainer's torch.no_grad().

    Raises ValueError, naming the argument, for a wrong shape or dtype, a threshold that is not a number or a model without
    image_height / image_width; RuntimeError for CPU tensors (there is no CPU path)."""
    return _surface_mask(self, fov_camera, depth, close_gaussian_threshold, False)[0]


def _depth_loss_forward(cfg, x, depth, sdf, cam):
    N, H, W, sh, sw, sx, sy, inv_std, cmax = cfg
    dev = x.device
    out = torch.empty((), dtype=torch.float32, device=dev)
    count = torch.empty(1, dtype=torch.int64, device=dev)
    L = _lib_handle()
    nbytes = L.gsr_sugar_depth_sdf_loss_bytes(N)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    rc = L.gsr_sugar_depth_sdf_loss(N, H, W, sh, sw, depth.data_ptr(), sx, sy, cam.data_ptr(), _ptr(x) if N else None,
                                    _ptr(sdf) if N else None, inv_std, cmax, out.data_ptr(), count.data_ptr(), ws.data_ptr(), nbytes,
                                    _lib.stream_ptr(dev))
    _lib.check(rc, "gsr_sugar_depth_sdf_loss")
    return out, count


class _DepthSdfLoss(torch.autograd.Function):
    """One output: the 0-dim mean; differentiable with respect to the samples, the depth map and the sdf values."""

    @staticmethod
    def forward(ctx, x, depth, sdf, cam, cfg):
        ctx.set_materialize_grads(False)
        out, count = _depth_loss_forward(cfg, x, depth, sdf, cam)
        ctx.cfg = cfg
        ctx.save_for_backward(x, depth, sdf, cam, count)
        return out

    @staticmethod
    def backward(ctx, g):
        x, depth, sdf, cam, count = ctx.saved_tensors
        N, H, W, sh, sw, sx, sy, inv_std, cmax = ctx.cfg
        need = ctx.needs_input_grad
        if g is None:
            return None, None, None, None, None
        dev = x.device
        g = g.reshape(1).contiguous()
        d_x = torch.empty((N, 3), dtype=torch.float32, device=dev)
        d_sdf = torch.empty(N, dtype=torch.float32, device=dev)
        d_depth = torch.empty((H, W), dtype=torch.float32, device=dev)
        L = _lib_handle()
        args = (N, H, W, sh, sw, depth.data_ptr(), sx, sy, cam.data_ptr(), _ptr(x) if N else None, _ptr(sdf) if N else None, inv_std,
                cmax, count.data_ptr(), g.data_ptr(), _ptr(d_x) if N else None, _ptr(d_sdf) if N else None, d_depth.data_ptr())
        if torch.are_deterministic_algorithms_enabled():  # fixed-order sums (DESIGN §4), no atomics
            nbytes = L.gsr_sugar_depth_sdf_loss_backward_det_bytes(N, H, W)
            scratch = _lib.scratch_bytes(max(nbytes, 16), dev)
            rc = L.gsr_sugar_depth_sdf_loss_backward_det(*args, scratch.data_ptr(), nbytes, _lib.stream_ptr(dev))
            _lib.check(rc, "gsr_sugar_depth_sdf_loss_backward_det")
        else:
            rc = L.gsr_sugar_depth_sdf_loss_backward(*args, _lib.stream_ptr(dev))
            _lib.check(rc, "gsr_sugar_depth_sdf_loss_backward")
        return d_x if need[0] else None, d_depth if need[1] else None, d_sdf if need[2] else None, None, None


def depth_sdf_estimation_loss(self, fov_camera, depth, sdf_samples, sdf_values, sdf_sample_std, clamp_max):
    """coarse_sdf's 'sdf' estimation loss (CS/:689-712 with the trainers' defaults: not squared, normalize_by_sdf_std=False) in
    CUDA, the 0-dim mean before the trainer's sdf_estimation_factor: over the samples in front of the camera (z > znear),
    clamp(|sdf_values - |map_z - z|| / sdf_sample_std, max=clamp_max).mean(), map_z being the depth map's value at the sample's
    projection (SuGaR.get_points_depth_in_depth_map, SS/:1189-1204).  NaN when no sample is in front, as torch's mean of an empty
    tensor.  Differentiable with respect to sdf_samples [N,3], depth [H,W] (a strided channel view is read in place) and
    sdf_values [N]; under torch.use_deterministic_algorithms the depth gradient is summed in a fixed order.  Nothing is read back
    to the host, in the forward or the backward.  sdf_sample_std (the trainer's get_cameras_spatial_extent() / 10) and clamp_max
    (10 * get_cameras_spatial_extent()) are Python numbers; the camera is read as by close_to_surface_mask.

    Raises ValueError, naming the argument, for a wrong shape or dtype or a std or clamp that is not a number; RuntimeError for
    CPU tensors (there is no CPU path)."""
    who = "depth_sdf_estimation_loss"
    std = _number(who, "sdf_sample_std", sdf_sample_std)
    cmax = _number(who, "clamp_max", clamp_max)
    _check_tensor(who, "sdf_samples", sdf_samples, (None, 3), torch.float32)
    N = sdf_samples.shape[0]
    _check_tensor(who, "sdf_values", sdf_values, (N,), torch.float32)
    H, W, sh, sw, sx, sy = _depth_map(who, self, depth)
    _require_cuda(who, sdf_samples, sdf_values, depth)
    dev = sdf_samples.device
    with np.errstate(divide="ignore", over="ignore"):
        inv_std = float(np.float32(1.0) / np.float32(std))  # torch divides a CUDA tensor by a Python number as x * (1 / b)
    cfg = (N, H, W, sh, sw, sx, sy, inv_std, float(np.float32(cmax)))
    with torch.cuda.device(dev):
        cam = _camera(who, fov_camera, dev, False)
        x, sdf = sdf_samples.contiguous(), sdf_values.contiguous()
        if torch.is_grad_enabled() and any(t.requires_grad for t in (x, depth, sdf)):
            return _DepthSdfLoss.apply(x, depth, sdf, cam, cfg)
        return _depth_loss_forward(cfg, x, depth, sdf, cam)[0]


# ------------------------------------------------------------------------------------- coarse_density's density-mode estimation loss
def _density_loss_forward(n, views, squared):
    (d, ds), (b, bs), (e, es) = views
    dev = d.device
    out = torch.empty((), dtype=torch.float32, device=dev)
    ws = torch.empty(_lib.GSR_LOSS_REDUCE_BYTES, dtype=torch.uint8, device=dev)
    rc = _lib_handle().gsr_density_estimation_loss(n, d.data_ptr(), ds, b.data_ptr(), bs, e.data_ptr(), es, int(squared), out.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev))
    _lib.check(rc, "gsr_density_estimation_loss")
    return out


def _flat(t):
    v = t.reshape(-1)
    return v, v.stride(0)


class _DensityLoss(torch.autograd.Function):
    """One output: the 0-dim mean; differentiable with respect to the densities, beta and the SDF estimate."""

    @staticmethod
    def forward(ctx, densities, beta, sdf_estimation, squared):
        ctx.set_materialize_grads(False)
        ctx.squared = squared
        ctx.save_for_backward(densities, beta, sdf_estimation)
        return _density_loss_forward(densities.numel(), [_flat(t) for t in (densities, beta, sdf_estimation)], squared)

    @staticmethod
    def backward(ctx, g):
        if g is None:
            return None, None, None, None
        ins = ctx.saved_tensors
        (d, ds), (b, bs), (e, es) = [_flat(t) for t in ins]
        dev, n = d.device, d.numel()
        grads = [torch.empty(t.shape, dtype=torch.float32, device=dev) for t in ins]
        g = g.detach().reshape(1).to(dtype=torch.float32).contiguous()
        rc = _lib_handle().gsr_density_estimation_loss_backward(n, d.data_ptr(), ds, b.data_ptr(), bs, e.data_ptr(), es, int(ctx.squared),
                                                                g.data_ptr(), *[t.data_ptr() for t in grads], _lib.stream_ptr(dev))
        _lib.check(rc, "gsr_density_estimation_loss_backward")
        return tuple(t if need else None for t, need in zip(grads, ctx.needs_input_grad[:3])) + (None,)


def density_estimation_loss(densities, beta, sdf_estimation, squared=False):
    """coarse_density's 'density' SDF estimation loss (CD/:735-741, coarse_sdf.py:714-720) when proj_mask is all true, before the
    trainer's sdf_estimation_factor: ``mean(|densities - exp(-0.5 * sdf_estimation ** 2 / beta ** 2)|)``, or the mean of its
    square with ``squared`` (squared_sdf_estimation_loss).  ``densities`` and ``beta`` are get_field_values' 'density' and 'beta',
    ``sdf_estimation`` projection_estimate's output: three float32 tensors of one shape, any strides.  The gradient goes to all
    three through torch's own chain, so a sample whose density equals its target gets a zero gradient in all three (torch's
    sign(0)).  Nothing is read back to the host, where the reference's ``[proj_mask]`` indexing synchronises twice per step.  With
    use_projection_as_estimation = False the caller still indexes the three tensors with proj_mask first.

    Raises ValueError, naming the argument, for a wrong dtype, a shape mismatch, an empty input or mixed devices; RuntimeError for
    CPU tensors (there is no CPU path)."""
    who = "density_estimation_loss"
    names = ("densities", "beta", "sdf_estimation")
    ts = (densities, beta, sdf_estimation)
    for name, t in zip(names, ts):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
            raise ValueError("%s: %s must be a float32 tensor, got %s" % (who, name, getattr(t, "dtype", type(t).__name__)))
    for name, t in zip(names[1:], ts[1:]):
        if t.shape != densities.shape:
            raise ValueError("%s: %s has shape %s, densities %s" % (who, name, tuple(t.shape), tuple(densities.shape)))
    if densities.numel() == 0:
        raise ValueError("%s: densities is empty (shape %s)" % (who, tuple(densities.shape)))
    for name, t in zip(names[1:], ts[1:]):
        if t.device != densities.device:
            raise ValueError("%s: %s is on %s, densities on %s" % (who, name, t.device, densities.device))
    _require_cuda(who, *ts)
    with torch.cuda.device(densities.device):
        if torch.is_grad_enabled() and any(t.requires_grad for t in ts):
            return _DensityLoss.apply(densities, beta, sdf_estimation, bool(squared))
        return _density_loss_forward(densities.numel(), [_flat(t) for t in ts], bool(squared))
