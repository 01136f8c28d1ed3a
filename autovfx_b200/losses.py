"""The trainers' per-step objective in CUDA ("LU/" = sugar/gaussian_splatting/utils/loss_utils.py, copied as
sugar/sugar_utils/loss_utils.py): drop-ins for ``ssim`` (LU/:33-62), ``normal_loss`` (LU/:118-132) and ``anisotropic_loss``
(LU/:159-168), and ``photometric_loss`` for train.py's first term ``(1-λ)·l1_loss + λ·(1-ssim)`` (GS/train.py:98-99).

Each is an ``autograd.Function`` whose value is a 0-dim CUDA tensor (``gsr_photometric_loss``, ``gsr_normal_loss``,
``gsr_anisotropic_loss`` and their backwards in gsr_loss.cu).  Nothing reads the device from the host in the forward or the backward:
the depth mask of ``normal_loss`` and its pixel count stay on the device, and the upstream gradients are read by the kernels.

Gradients flow to the first argument only; a ground truth that requires grad raises ValueError naming it.  Arguments the kernels
do not reproduce (``window_size != 11``, ``size_average=False``, mismatched shapes, non-float32 inputs, mixed devices, empty
inputs, a last dimension other than 3 where one is required) raise ValueError naming the argument; CPU tensors raise RuntimeError.
The window sums are not in cuDNN's order, so values are not bit-identical to torch's (INTEGRATION.md, "Training objective").
"""
from __future__ import annotations

import ctypes as C
from math import exp

import torch

from . import _lib

__all__ = ["ssim", "photometric_loss", "normal_loss", "anisotropic_loss", "ssim_window"]

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
