"""fp64 restatement of the trainers' remaining loss terms with closed-form gradients, and the per-element float32 error bounds the
GPU tests hold the library (and torch's own float32 graph) to:

  depth_loss, opacity_loss, sparsity_loss   sugar/gaussian_splatting/utils/loss_utils.py:65-157
  entropy                                  sugar/sugar_trainers/coarse_density.py:598-606 (coarse_sdf.py:582-595)
  density-mode SDF estimation              coarse_density.py:735-741 (coarse_sdf.py:714-720), proj_mask all true

Every function returns a dict with the value ``val``, the gradient(s) and their bounds.  A sum of n float32 terms is within
``k_sum * U32 * sum |terms|`` of its exact value: the library sums in double (its error is one rounding), torch's float32 reduction
sums in blocks of a tree, whose error in practice stays far below the default k_sum.  Each elementwise float32 operation adds one
rounding of its own magnitude.  Written for the tests; tests/test_loss_terms_cpu.py pins the values and gradients against fp64
autograd of the reference lines.
"""
from __future__ import annotations

import numpy as np
import torch

U32 = 2.0 ** -24  # unit roundoff of float32
TINY = 2.0 ** -149  # the spacing of float32 subnormals
K_SUM = 128.0
SPARSE_LO, SPARSE_HI = float(np.float32(1e-3)), float(np.float32(1 - 1e-3))
ENTROPY_EPS = 1e-10


def depth64(network_output, gt, scene_scale=5.0, g_out=1.0, k_sum=K_SUM):
    """depth_loss: value, d value / d network_output, and bounds.  The bound of the scale x0 and the shift x1 carries the
    conditioning of the 2x2 fit: det = a00 a11 - a01^2 cancels, so the sums' errors are amplified by |a00 a11| / |det|.
    ``cond`` is the first-order relative error bound of det; the bounds are valid (and returned finite) for cond <= 0.5."""
    p = network_output.double().reshape(-1)
    d = gt.double().reshape(-1) / 25
    n = p.numel()
    m = d > 0
    w = m.double()
    pm, dm = p[m], d[m]
    a00, a01, a11, b0, b1 = (pm * pm).sum(), pm.sum(), m.sum().double(), (pm * dm).sum(), dm.sum()
    det = a00 * a11 - a01 * a01
    out = dict(count=int(m.sum()), det=float(det))
    if float(det) == 0.0:
        nan = float("nan")
        return dict(out, val=torch.tensor(nan, dtype=torch.float64), grad=torch.full_like(p, nan).reshape(network_output.shape),
                    cond=float("inf"))
    x0 = (a11 * b0 - a01 * b1) / det
    x1 = (-a01 * b0 + a00 * b1) / det
    e = torch.exp(-p / scene_scale)
    r = x0 * p + x1 - d
    v = w * e * r * r
    grad = 2 * w * e * r * x0 * g_out / n
    # the sums (d's own rounding, 2 u relative, is inside k_sum) and the float32 solve
    ku = k_sum * U32
    e00, e01, eb0, eb1 = ku * a00, ku * pm.abs().sum(), ku * (pm * dm).abs().sum(), ku * dm.abs().sum()
    ddet = a11 * e00 + 2 * a01.abs() * e01 + 4 * U32 * (a00 * a11 + a01 * a01)
    dn0 = a11 * eb0 + e01 * b1.abs() + a01.abs() * eb1 + 4 * U32 * ((a11 * b0).abs() + (a01 * b1).abs())
    dn1 = e01 * b0.abs() + a01.abs() * eb0 + e00 * b1.abs() + a00 * eb1 + 4 * U32 * ((a01 * b0).abs() + (a00 * b1).abs())
    cond = float(ddet / det.abs())
    if cond > 0.5:
        inf = float("inf")
        return dict(out, val=v.mean(), grad=grad.reshape(network_output.shape), x0=float(x0), x1=float(x1), cond=cond, vb=inf,
                    gb=torch.full_like(p, inf).reshape(network_output.shape))
    # |x' - x| <= (|dn| + |x| |ddet|) / (|det| (1 - cond)) <= 2 (...) / |det|, plus the division's rounding
    bx0 = float(2 * (dn0 + x0.abs() * ddet) / det.abs() + 2 * U32 * x0.abs())
    bx1 = float(2 * (dn1 + x1.abs() * ddet) / det.abs() + 2 * U32 * x1.abs())
    re = 4 * U32 * (p.abs() / scene_scale + 1)  # exp's relative error: the rounded argument and exp itself
    dr = p.abs() * bx0 + bx1 + 4 * U32 * ((x0 * p).abs() + abs(float(x1)) + d.abs() + r.abs())
    we = w * e
    vb = (we * (2 * r.abs() * dr + dr * dr) + (re + 4 * U32) * v.abs()).mean() + ku * v.abs().mean()
    gb = 2 * we * abs(g_out) / n * (dr * abs(float(x0)) + r.abs() * bx0 + dr * bx0) + (re + 8 * U32) * grad.abs()
    return dict(out, val=v.mean(), grad=grad.reshape(network_output.shape), x0=float(x0), x1=float(x1), bx0=bx0, bx1=bx1, cond=cond,
                vb=float(vb), gb=gb.reshape(network_output.shape))


def opacity64(x, g_out=1.0, k_sum=K_SUM):
    """opacity_loss: mean(x); the gradient g_out / n everywhere."""
    v = x.double()
    n = v.numel()
    return dict(val=v.mean(), grad=torch.full_like(v, g_out / n), vb=k_sum * U32 * float(v.abs().mean()),
                gb=torch.full_like(v, 4 * U32 * abs(g_out) / n))


def sparsity64(x, g_out=1.0, k_sum=K_SUM):
    """sparsity_loss: mean(log c + log(1 - c)), c = clamp(x, float32(1e-3), float32(1 - 1e-3)); the gradient passes where
    lo <= x <= hi (both bounds included)."""
    v = x.double()
    n = v.numel()
    c = v.clamp(SPARSE_LO, SPARSE_HI)
    t = torch.log(c) + torch.log(1 - c)
    on = ((v >= SPARSE_LO) & (v <= SPARSE_HI)).double()
    grad = on * g_out / n * (1 / c - 1 / (1 - c))
    tb = 8 * U32 * (torch.log(c).abs() + torch.log(1 - c).abs() + 1)
    gb = on * abs(g_out) / n * 8 * U32 * (1 / c + 1 / (1 - c))
    return dict(val=t.mean(), grad=grad, vb=float(tb.mean() + k_sum * U32 * t.abs().mean()), gb=gb)


def entropy64(opacities, radii, g_out=1.0, k_sum=K_SUM):
    """The coarse trainers' entropy term over radii > 0: value (NaN with no visible Gaussian), gradient (0 off the filter)."""
    o = opacities.double()
    vis = (radii.reshape(o.shape[0]) > 0)
    if o.dim() == 2:
        vis = vis.unsqueeze(1)
    cnt = int(vis.sum())
    u = 1 - o
    L1, L2 = torch.log(o + ENTROPY_EPS), torch.log(u + ENTROPY_EPS)
    t = -o * L1 - u * L2
    visd = vis.double()
    val = t[vis].mean() if cnt else torch.tensor(float("nan"), dtype=torch.float64)
    g = g_out / max(cnt, 1)
    grad = visd * g * (-L1 - o / (o + ENTROPY_EPS) + L2 + u / (u + ENTROPY_EPS))
    tb = 8 * U32 * ((o * L1).abs() + (u * L2).abs() + o.abs() + u.abs())
    vb = float(tb[vis].mean() + k_sum * U32 * t[vis].abs().mean()) if cnt else 0.0
    gb = visd * abs(g) * 16 * U32 * (L1.abs() + L2.abs() + 4)
    return dict(val=val, grad=grad, vb=vb, gb=gb, count=cnt)


def density64(densities, beta, sdf_estimation, squared=False, g_out=1.0, k_sum=K_SUM):
    """Density-mode SDF estimation: value, the gradients with respect to densities, beta and sdf_estimation, and their bounds.
    With the absolute value, a sample whose error |d - t| is within rounding of 0 may take any sign of abs's gradient."""
    d, b, s = densities.double(), beta.double(), sdf_estimation.double()
    n = d.numel()
    q = -0.5 * s * s / (b * b)
    t = torch.exp(q)
    e = d - t
    v = e * e if squared else e.abs()
    g = g_out / n
    ge = g * (2 * e if squared else torch.sign(e))
    g_d = ge
    g_s = ge * t * s / (b * b)
    g_b = -ge * t * s * s / (b * b * b)
    rel = 12 * U32 * (1 + q.abs())         # the chain's roundings and exp's error through q
    de = U32 * e.abs() + t * rel + TINY     # the float32 error of e
    if squared:
        vbe = 2 * e.abs() * de + de * de + 2 * U32 * v
        dge = 2 * abs(g) * de + 4 * U32 * ge.abs()
    else:
        vbe = de
        dge = torch.where(e.abs() <= de, torch.full_like(e, 2 * abs(g)), 2 * U32 * ge.abs())
    gb_d = dge
    # below q = -87 exp(q) is a float32 subnormal or 0: t, -ge t and the quotients after it lose their relative precision, so each
    # carries up to one subnormal spacing (TINY) of absolute error through the rest of the chain
    dgq = 2 * TINY
    gb_s = dge * t * s.abs() / (b * b) + rel * g_s.abs() + (dgq / (b * b) + TINY) * 2 * s.abs() + TINY
    gb_b = dge * t * s * s / (b * b * b).abs() + rel * g_b.abs() + (dgq * q.abs() / (b * b) + TINY) * 2 * b.abs() + TINY
    vb = float(vbe.mean() + k_sum * U32 * v.mean())
    return dict(val=v.mean(), grads=(g_d, g_b, g_s), vb=vb, gbs=(gb_d, gb_b, gb_s))
