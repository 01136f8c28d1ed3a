"""The trainers' per-step objective in CUDA ("LU/" = sugar/gaussian_splatting/utils/loss_utils.py, copied as
sugar/sugar_utils/loss_utils.py): drop-ins for ``ssim`` (LU/:33-62), ``normal_loss`` (LU/:118-132), ``anisotropic_loss``
(LU/:159-168), ``depth_loss`` (LU/:65-111), ``opacity_loss`` and ``sparsity_loss`` (LU/:143-157), ``photometric_loss`` for
train.py's first term ``(1-λ)·l1_loss + λ·(1-ssim)`` (GS/train.py:98-99), and ``entropy_loss`` for the coarse trainers' opacity
entropy term (sugar/sugar_trainers/coarse_density.py:598-606, coarse_sdf.py:582-595).

Each is an ``autograd.Function`` whose value is a 0-dim CUDA tensor (``gsr_photometric_loss``, ``gsr_normal_loss``,
``gsr_anisotropic_loss``, ``gsr_depth_loss``, ``gsr_opacity_loss``, ``gsr_sparsity_loss``, ``gsr_entropy_loss`` and their backwards
in gsr_loss.cu).  Nothing reads the device from the host in the forward or the backward: the masks of ``normal_loss``,
``depth_loss`` and ``entropy_loss``, their counts and depth_loss's scale and shift stay on the device, and the upstream gradients
are read by the kernels.

Gradients flow to the first argument only; a ground truth that requires grad raises ValueError naming it.  Arguments the kernels
do not reproduce (``window_size != 11``, ``size_average=False``, mismatched shapes, non-float32 inputs, mixed devices, empty
inputs, a last dimension other than 3 where one is required) raise ValueError naming the argument; CPU tensors raise RuntimeError.
The window sums are not in cuDNN's order, so values are not bit-identical to torch's (INTEGRATION.md, "Training objective").
"""
from __future__ import annotations

import ctypes as C
from math import exp

import numpy as np
import torch

from . import _lib

__all__ = ["ssim", "photometric_loss", "normal_loss", "anisotropic_loss", "depth_loss", "opacity_loss", "sparsity_loss",
           "entropy_loss", "ssim_window"]

WINDOW_SIZE = 11


def ssim_window() -> torch.Tensor:
    """The 1-D float32 weights of create_window (LU/:24-31), by torch's own expression: σ = 1.5, 11 taps.  create_window's 2-D
    window is the float32 outer product of these; the kernels apply them separably (one row pass, one column pass)."""
    gauss = torch.Tensor([exp(-(x - WINDOW_SIZE // 2) ** 2 / float(2 * 1.5 ** 2)) for x in range(WINDOW_SIZE)])
    return gauss / gauss.sum()


_WINDOW = (C.c_float * WINDOW_SIZE)(*ssim_window().tolist())


def _check_pair(who, names, a, b, image=False):
    """ValueError for what the kernels do not take; RuntimeError for CPU tensors once the pair is otherwise valid."""
    for n, t in zip(names, (a, b)):
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a tensor, got %s" % (who, n, type(t).__name__))
        if t.dtype != torch.float32:
            raise ValueError("%s: %s must be float32, got %s" % (who, n, t.dtype))
    if torch.is_grad_enabled() and b.requires_grad:
        raise ValueError("%s: %s requires grad; only %s is differentiated (detach the ground truth)" % (who, names[1], names[0]))
    if a.shape != b.shape:
        raise ValueError("%s: %s has shape %s, %s %s" % (who, names[1], tuple(b.shape), names[0], tuple(a.shape)))
    if a.device != b.device:
        raise ValueError("%s: %s is on %s, %s on %s" % (who, names[1], b.device, names[0], a.device))
    if a.numel() == 0:
        raise ValueError("%s: %s is empty (shape %s)" % (who, names[0], tuple(a.shape)))
    if image and a.dim() not in (3, 4):
        raise ValueError("%s: %s must be a [C,H,W] or [B,C,H,W] image, got shape %s" % (who, names[0], tuple(a.shape)))
    if not a.is_cuda:
        raise RuntimeError("autovfx_b200.%s: %s must be a CUDA tensor, got one on %s (there is no CPU path)" % (who, names[0], a.device))


def _strides4(t):
    return (C.c_int64 * 4)(*((0,) + tuple(t.stride()) if t.dim() == 3 else tuple(t.stride())))


def _dims4(t):
    return (1,) + tuple(t.shape) if t.dim() == 3 else tuple(t.shape)


class _Photometric(torch.autograd.Function):
    """(mean |x - y| or None, mean SSIM) of two [C,H,W] / [B,C,H,W] images by their own strides; gradients to x."""

    @staticmethod
    def forward(ctx, x, y, with_l1, need_grad):
        ctx.set_materialize_grads(False)
        B, Ch, H, W = _dims4(x)
        dev = x.device
        ws = torch.empty(_lib.lib.gsr_photometric_loss_bytes(B, Ch, H, W, int(need_grad)), dtype=torch.uint8, device=dev)
        l1 = torch.empty((), dtype=torch.float32, device=dev) if with_l1 else None
        s = torch.empty((), dtype=torch.float32, device=dev)
        sx, sy = _strides4(x), _strides4(y)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_photometric_loss(B, Ch, H, W, x.data_ptr(), sx, y.data_ptr(), sy, _WINDOW, int(need_grad),
                                                     l1.data_ptr() if with_l1 else None, s.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     _lib.stream_ptr(dev)), "gsr_photometric_loss")
        if need_grad:
            ctx.save_for_backward(x, y)
            ctx.ws = ws
        return (l1, s) if with_l1 else s

    @staticmethod
    def backward(ctx, *grads):
        x, y = ctx.saved_tensors
        g_l1, g_ssim = grads if len(grads) == 2 else (None, grads[0])
        if g_l1 is None and g_ssim is None:
            return None, None, None, None
        B, Ch, H, W = _dims4(x)
        dev = x.device
        g_l1, g_ssim = (None if g is None else g.detach().to(dtype=torch.float32).contiguous() for g in (g_l1, g_ssim))
        dx = torch.empty((B, Ch, H, W), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_photometric_loss_backward(
                B, Ch, H, W, x.data_ptr(), _strides4(x), y.data_ptr(), _strides4(y), _WINDOW,
                None if g_l1 is None else g_l1.data_ptr(), None if g_ssim is None else g_ssim.data_ptr(), dx.data_ptr(),
                ctx.ws.data_ptr(), ctx.ws.numel(), _lib.stream_ptr(dev)), "gsr_photometric_loss_backward")
        return dx.view(x.shape), None, None, None


def ssim(img1, img2, window_size=11, size_average=True):
    """Drop-in for loss_utils.ssim (LU/:33-41): the mean SSIM of img1 against img2 ([C,H,W] or [B,C,H,W], any strides), a 0-dim
    CUDA tensor differentiable with respect to img1.  Only the trainers' form is reproduced: window_size 11, size_average True."""
    who = "ssim"
    if window_size != WINDOW_SIZE:
        raise ValueError("%s: window_size must be 11 (the trainers' window), got %r" % (who, window_size))
    if size_average is not True:
        raise ValueError("%s: size_average=%r is not reproduced (every trainer takes the mean)" % (who, size_average))
    _check_pair(who, ("img1", "img2"), img1, img2, image=True)
    return _Photometric.apply(img1, img2, False, torch.is_grad_enabled() and img1.requires_grad)


def photometric_loss(image, gt, lambda_dssim):
    """``(1.0 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1.0 - ssim(image, gt))`` (GS/train.py:98-99) with the L1 mean
    and the SSIM mean from one kernel pair; the combination is train.py's own scalar expression."""
    who = "photometric_loss"
    _check_pair(who, ("image", "gt"), image, gt, image=True)
    l1, s = _Photometric.apply(image, gt, True, torch.is_grad_enabled() and image.requires_grad)
    return (1.0 - lambda_dssim) * l1 + lambda_dssim * (1.0 - s)


def _pixels3(t):
    """[n,3] view (a copy only when the leading dims cannot be flattened) and its (pixel, component) strides."""
    v = t.reshape(-1, 3)
    return v, (C.c_int64 * 2)(*v.stride())


class _Normal(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, depth, scene_scale, need_grad):
        dev = pred.device
        p, ps = _pixels3(pred)
        g, gs = _pixels3(gt)
        d = None if depth is None else depth.reshape(-1)
        ws = torch.empty(_lib.GSR_LOSS_REDUCE_BYTES, dtype=torch.uint8, device=dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_normal_loss(p.shape[0], p.data_ptr(), ps, g.data_ptr(), gs, None if d is None else d.data_ptr(),
                                                0 if d is None else d.stride(0), scene_scale, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                _lib.stream_ptr(dev)), "gsr_normal_loss")
        if need_grad:
            ctx.save_for_backward(pred, gt, depth)
            ctx.ws, ctx.scene_scale = ws, scene_scale
        return out

    @staticmethod
    def backward(ctx, g_out):
        pred, gt, depth = ctx.saved_tensors
        dev = pred.device
        p, ps = _pixels3(pred)
        g, gs = _pixels3(gt)
        d = None if depth is None else depth.reshape(-1)
        g_out = g_out.detach().to(dtype=torch.float32).contiguous()
        dp = torch.empty(pred.shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_normal_loss_backward(p.shape[0], p.data_ptr(), ps, g.data_ptr(), gs,
                                                         None if d is None else d.data_ptr(), 0 if d is None else d.stride(0),
                                                         ctx.scene_scale, g_out.data_ptr(), dp.data_ptr(), ctx.ws.data_ptr(),
                                                         ctx.ws.numel(), _lib.stream_ptr(dev)), "gsr_normal_loss_backward")
        return dp, None, None, None, None


def normal_loss(network_output, gt, depth=None, scene_scale=5.0):
    """Drop-in for loss_utils.normal_loss (LU/:118-132): ``mean|n - g| + 0.1 * (-mean n·g)`` of the F.normalize'd [..., 3] maps,
    over the pixels with ``0 < depth < scene_scale`` when depth (shape ``network_output.shape[:-1]``) is given.  The selection and its
    count stay on the device; an empty selection gives NaN, as torch's mean of an empty tensor."""
    who = "normal_loss"
    if isinstance(network_output, torch.Tensor) and (network_output.dim() == 0 or network_output.shape[-1] != 3):
        raise ValueError("%s: network_output must have a last dimension of 3, got shape %s" % (who, tuple(network_output.shape)))
    if depth is not None and isinstance(network_output, torch.Tensor):
        if not isinstance(depth, torch.Tensor) or depth.dtype != torch.float32:
            raise ValueError("%s: depth must be a float32 tensor" % who)
        if depth.shape != network_output.shape[:-1]:
            raise ValueError("%s: depth has shape %s, network_output's pixels %s" % (who, tuple(depth.shape),
                                                                                     tuple(network_output.shape[:-1])))
        if depth.device != network_output.device:
            raise ValueError("%s: depth is on %s, network_output on %s" % (who, depth.device, network_output.device))
    _check_pair(who, ("network_output", "gt"), network_output, gt)
    return _Normal.apply(network_output, gt, depth, float(scene_scale), torch.is_grad_enabled() and network_output.requires_grad)


class _Anisotropic(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scales, r, need_grad):
        dev = scales.device
        s = scales.reshape(-1, 3).contiguous()
        ws = torch.empty(_lib.GSR_LOSS_REDUCE_BYTES, dtype=torch.uint8, device=dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_anisotropic_loss(s.shape[0], s.data_ptr(), r, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     _lib.stream_ptr(dev)), "gsr_anisotropic_loss")
        if need_grad:
            ctx.save_for_backward(s)
            ctx.r, ctx.shape = r, scales.shape
        return out

    @staticmethod
    def backward(ctx, g_out):
        (s,) = ctx.saved_tensors
        dev = s.device
        g_out = g_out.detach().to(dtype=torch.float32).contiguous()
        ds = torch.empty_like(s)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_anisotropic_loss_backward(s.shape[0], s.data_ptr(), ctx.r, g_out.data_ptr(), ds.data_ptr(),
                                                              _lib.stream_ptr(dev)), "gsr_anisotropic_loss_backward")
        return ds.view(ctx.shape), None, None


def anisotropic_loss(gaussians_scale, r=3):
    """Drop-in for loss_utils.anisotropic_loss (LU/:159-168): ``mean(clamp_min(max / (min + 1e-6), r) - r)`` over the rows of
    [..., 3] scales.  The backward sends the max's and the min's gradient to the first extreme index of each row, as torch's
    max(dim) / min(dim) return it on ties, and passes the gradient at ratio == r (clamp_min's rule)."""
    who = "anisotropic_loss"
    if not isinstance(gaussians_scale, torch.Tensor) or gaussians_scale.dtype != torch.float32:
        raise ValueError("%s: gaussians_scale must be a float32 tensor" % who)
    if gaussians_scale.dim() < 1 or gaussians_scale.shape[-1] != 3:
        raise ValueError("%s: gaussians_scale must have a last dimension of 3, got shape %s" % (who, tuple(gaussians_scale.shape)))
    if gaussians_scale.numel() == 0:
        raise ValueError("%s: gaussians_scale is empty (shape %s)" % (who, tuple(gaussians_scale.shape)))
    if not gaussians_scale.is_cuda:
        raise RuntimeError("autovfx_b200.%s: gaussians_scale must be a CUDA tensor, got one on %s (there is no CPU path)"
                           % (who, gaussians_scale.device))
    return _Anisotropic.apply(gaussians_scale, float(r), torch.is_grad_enabled() and gaussians_scale.requires_grad)


def _flat(t):
    """[n] view of t (a copy only when its dims cannot be flattened) and its element stride."""
    v = t.reshape(-1)
    return v, v.stride(0)


def _check_float(who, name, t):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError("%s: %s must be a float32 tensor, got %s" % (who, name, getattr(t, "dtype", type(t).__name__)))
    if t.numel() == 0:
        raise ValueError("%s: %s is empty (shape %s)" % (who, name, tuple(t.shape)))


def _require_cuda(who, name, t):
    if not t.is_cuda:
        raise RuntimeError("autovfx_b200.%s: %s must be a CUDA tensor, got one on %s (there is no CPU path)" % (who, name, t.device))


def _reduce_ws(dev):
    return torch.empty(_lib.GSR_LOSS_REDUCE_BYTES, dtype=torch.uint8, device=dev)


class _Depth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, inv_scale, need_grad):
        dev = pred.device
        p, ps = _flat(pred)
        g, gs = _flat(gt)
        ws = _reduce_ws(dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_depth_loss(p.numel(), p.data_ptr(), ps, g.data_ptr(), gs, inv_scale, out.data_ptr(), ws.data_ptr(),
                                               ws.numel(), _lib.stream_ptr(dev)), "gsr_depth_loss")
        if need_grad:
            ctx.save_for_backward(pred, gt)
            ctx.ws, ctx.inv_scale = ws, inv_scale
        return out

    @staticmethod
    def backward(ctx, g_out):
        pred, gt = ctx.saved_tensors
        dev = pred.device
        p, ps = _flat(pred)
        g, gs = _flat(gt)
        g_out = g_out.detach().to(dtype=torch.float32).contiguous()
        dp = torch.empty(pred.shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_depth_loss_backward(p.numel(), p.data_ptr(), ps, g.data_ptr(), gs, ctx.inv_scale, g_out.data_ptr(),
                                                        dp.data_ptr(), ctx.ws.data_ptr(), ctx.ws.numel(), _lib.stream_ptr(dev)),
                       "gsr_depth_loss_backward")
        return dp, None, None, None


def depth_loss(network_output, gt, scene_scale=5.0):
    """Drop-in for loss_utils.depth_loss (LU/:94-111): ``mean(w * exp(-p / scene_scale) * (scale * p + shift - d) ** 2)`` over every
    pixel of the flattened rendered depth p, with d = gt / 25, w = 1 where d > 0 and (scale, shift) the least-squares fit of p to d
    on that mask (compute_scale_and_shift, LU/:65-92).  The five masked sums are accumulated in double in a fixed order and rounded
    to float32; the 2x2 solve runs in one device thread with torch's operation order, so the mask, its count, the scale and the
    shift never reach the host.  The gradient goes to network_output only: the scale, the shift and the exp factor are constants,
    as the reference detaches them.

    One deviation: where the reference's ``det == 0`` (an empty mask included) builds 0-element tensors and then fails with a
    broadcast error, this returns NaN for the value and every gradient element (INTEGRATION.md, "Training objective")."""
    who = "depth_loss"
    _check_float(who, "network_output", network_output)
    _check_float(who, "gt", gt)
    if torch.is_grad_enabled() and gt.requires_grad:
        raise ValueError("%s: gt requires grad; only network_output is differentiated (detach the ground truth)" % who)
    if gt.numel() != network_output.numel():
        raise ValueError("%s: gt has %d elements (shape %s), network_output %d (shape %s)" % (
            who, gt.numel(), tuple(gt.shape), network_output.numel(), tuple(network_output.shape)))
    if gt.device != network_output.device:
        raise ValueError("%s: gt is on %s, network_output on %s" % (who, gt.device, network_output.device))
    if isinstance(scene_scale, bool) or not isinstance(scene_scale, (int, float, np.floating, np.integer)):
        raise ValueError("%s: scene_scale must be a Python number, got %r" % (who, scene_scale))
    _require_cuda(who, "network_output", network_output)
    with np.errstate(divide="ignore", over="ignore"):
        inv_scale = float(np.float32(1.0) / np.float32(scene_scale))  # torch divides a CUDA tensor by a Python number as x * (1 / b)
    return _Depth.apply(network_output, gt, inv_scale, torch.is_grad_enabled() and network_output.requires_grad)


class _Opacity(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, sparse, need_grad):
        dev = x.device
        v, vs = _flat(x)
        ws = _reduce_ws(dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        fn, what = (_lib.lib.gsr_sparsity_loss, "gsr_sparsity_loss") if sparse else (_lib.lib.gsr_opacity_loss, "gsr_opacity_loss")
        with torch.cuda.device(dev):
            _lib.check(fn(v.numel(), v.data_ptr(), vs, out.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), what)
        if need_grad:
            ctx.save_for_backward(x)
            ctx.sparse = sparse
        return out

    @staticmethod
    def backward(ctx, g_out):
        (x,) = ctx.saved_tensors
        dev = x.device
        v, vs = _flat(x)
        g_out = g_out.detach().to(dtype=torch.float32).contiguous()
        dx = torch.empty(x.shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if ctx.sparse:
                _lib.check(_lib.lib.gsr_sparsity_loss_backward(v.numel(), v.data_ptr(), vs, g_out.data_ptr(), dx.data_ptr(),
                                                               _lib.stream_ptr(dev)), "gsr_sparsity_loss_backward")
            else:
                _lib.check(_lib.lib.gsr_opacity_loss_backward(v.numel(), g_out.data_ptr(), dx.data_ptr(), _lib.stream_ptr(dev)),
                           "gsr_opacity_loss_backward")
        return dx, None, None


def _opacity_term(who, x, sparse):
    _check_float(who, "network_output", x)
    _require_cuda(who, "network_output", x)
    return _Opacity.apply(x, sparse, torch.is_grad_enabled() and x.requires_grad)


def opacity_loss(network_output):
    """Drop-in for loss_utils.opacity_loss (LU/:143-147): ``mean(network_output)`` over any shape and strides."""
    return _opacity_term("opacity_loss", network_output, False)


def sparsity_loss(network_output):
    """Drop-in for loss_utils.sparsity_loss (LU/:149-157): ``mean(log(c) + log(1 - c))`` with ``c = clamp(x, 1e-3, 1 - 1e-3)``,
    the bounds rounded to float32 as torch compares against them.  The gradient passes where ``1e-3 <= x <= 1 - 1e-3``, both bounds
    included, as torch's clamp backward does."""
    return _opacity_term("sparsity_loss", network_output, True)


class _Entropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, o, radii, need_grad):
        dev = o.device
        v, vs = _flat(o)
        r = radii.reshape(-1)
        ws = _reduce_ws(dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_entropy_loss(v.numel(), v.data_ptr(), vs, r.data_ptr(), r.stride(0), out.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _lib.stream_ptr(dev)), "gsr_entropy_loss")
        if need_grad:
            ctx.save_for_backward(o, radii)
            ctx.ws = ws
        return out

    @staticmethod
    def backward(ctx, g_out):
        o, radii = ctx.saved_tensors
        dev = o.device
        v, vs = _flat(o)
        r = radii.reshape(-1)
        g_out = g_out.detach().to(dtype=torch.float32).contiguous()
        do = torch.empty(o.shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_entropy_loss_backward(v.numel(), v.data_ptr(), vs, r.data_ptr(), r.stride(0), g_out.data_ptr(),
                                                          do.data_ptr(), ctx.ws.data_ptr(), ctx.ws.numel(), _lib.stream_ptr(dev)),
                       "gsr_entropy_loss_backward")
        return do, None, None


def entropy_loss(opacities, radii):
    """The coarse trainers' opacity entropy term (coarse_density.py:598-606, coarse_sdf.py:582-595) without its
    entropy_regularization_factor: the mean over the Gaussians with ``radii > 0`` of
    ``-o * log(o + 1e-10) - (1 - o) * log(1 - o + 1e-10)``.  ``opacities`` is [P] or [P, 1] (as render_sugar / render_sugar_raw
    return them) and ``radii`` the render's int32 [P].  The visibility filter and its count stay on the device, where the
    reference's boolean indexing synchronises with the host; no visible Gaussian gives NaN, as torch's mean of an empty tensor."""
    who = "entropy_loss"
    _check_float(who, "opacities", opacities)
    if opacities.dim() not in (1, 2) or (opacities.dim() == 2 and opacities.shape[1] != 1):
        raise ValueError("%s: opacities must be [P] or [P, 1], got shape %s" % (who, tuple(opacities.shape)))
    P = opacities.shape[0]
    if not isinstance(radii, torch.Tensor) or radii.dtype != torch.int32:
        raise ValueError("%s: radii must be an int32 tensor, got %s" % (who, getattr(radii, "dtype", type(radii).__name__)))
    if tuple(radii.shape) != (P,):
        raise ValueError("%s: radii must have shape [%d], got %s" % (who, P, tuple(radii.shape)))
    if radii.device != opacities.device:
        raise ValueError("%s: radii is on %s, opacities on %s" % (who, radii.device, opacities.device))
    _require_cuda(who, "opacities", opacities)
    return _Entropy.apply(opacities, radii, torch.is_grad_enabled() and opacities.requires_grad)
