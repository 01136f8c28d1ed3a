"""fp64 restatement of the trainers' loss terms (sugar/gaussian_splatting/utils/loss_utils.py: l1_loss, ssim, normal_loss,
anisotropic_loss) with closed-form gradients, and the per-element error bounds the GPU tests hold autovfx_b200.losses (and torch's
own float32 graph) to.  Written for the tests; tests/test_losses_cpu.py pins it against fp64 autograd of the reference formulas.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24  # unit roundoff of float32
C1, C2 = 0.01 ** 2, 0.03 ** 2


def window64():
    """The exact (fp64) 11-tap Gaussian, sigma 1.5, normalised to sum 1."""
    g = torch.tensor([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)], dtype=torch.float64)
    return g / g.sum()


def conv_sep(img, w):
    """Zero-padded 11x11 correlation of every plane of img [..., H, W] with outer(w, w), as a row then a column pass."""
    shape = img.shape
    p = img.reshape(-1, 1, shape[-2], shape[-1])
    p = F.conv2d(p, w.view(1, 1, 1, 11).to(p), padding=(0, 5))
    p = F.conv2d(p, w.view(1, 1, 11, 1).to(p), padding=(5, 0))
    return p.reshape(shape)


def _b4(t):
    return t.unsqueeze(0) if t.dim() == 3 else t


def ssim_parts(x, y, w=None):
    """Every per-pixel quantity of ssim(x, y) in fp64 ([B,C,H,W] or [C,H,W] inputs, any dtype): the moments, A = 2 mu1 mu2 + C1,
    Bv = 2 s12 + C2, Cv = mu1^2 + mu2^2 + C1, D = s1 + s2 + C2, the map S = A Bv / (Cv D) and its partials g_mu, g_xx, g_xy with
    respect to mu_x, E[x^2], E[xy]."""
    w = window64() if w is None else w.double()
    x, y = _b4(x).double(), _b4(y).double()
    mu1, mu2 = conv_sep(x, w), conv_sep(y, w)
    exx, eyy, exy = conv_sep(x * x, w), conv_sep(y * y, w), conv_sep(x * y, w)
    s1, s2, s12 = exx - mu1 ** 2, eyy - mu2 ** 2, exy - mu1 * mu2
    A, Bv = 2 * mu1 * mu2 + C1, 2 * s12 + C2
    Cv, D = mu1 ** 2 + mu2 ** 2 + C1, s1 + s2 + C2
    S = A * Bv / (Cv * D)
    g_mu = 2 * mu2 * (Bv - A) / (Cv * D) + 2 * mu1 * S * (1 / D - 1 / Cv)
    g_xx = -S / D
    g_xy = 2 * A / (Cv * D)
    return dict(x=x, y=y, w=w, mu1=mu1, mu2=mu2, exx=exx, eyy=eyy, exy=exy, A=A, Bv=Bv, Cv=Cv, D=D, S=S, g_mu=g_mu, g_xx=g_xx,
                g_xy=g_xy)


def photometric64(x, y, g_l1=1.0, g_ssim=1.0, w=None):
    """(mean |x - y|, mean SSIM, d(g_l1 * l1 + g_ssim * ssim)/dx) in fp64; the abs's gradient is 0 where x == y."""
    p = ssim_parts(x, y, w)
    n = p["S"].numel()
    grad = g_ssim / n * (conv_sep(p["g_mu"], p["w"]) + 2 * p["x"] * conv_sep(p["g_xx"], p["w"]) + p["y"] * conv_sep(p["g_xy"], p["w"]))
    grad = grad + g_l1 / n * torch.sign(p["x"] - p["y"])
    return (p["x"] - p["y"]).abs().mean(), p["S"].mean(), grad.reshape(x.shape), p


def _map_fns(mu1, mu2, A, Bv, Cv, D):
    S = A * Bv / (Cv * D)
    return dict(S=S, g_mu=2 * mu2 * (Bv - A) / (Cv * D) + 2 * mu1 * S * (1 / D - 1 / Cv), g_xx=-S / D, g_xy=2 * A / (Cv * D))


def photometric_bounds(p, g_l1=1.0, g_ssim=1.0, k=64.0):
    """Per-element float32 error bounds derived from the operand magnitudes.  A window sum of 11 x 11 products, in any order and
    with float32 weights, is within k u of its sum of absolute terms (ax, ay, axx, ayy, axy below); each such error moves A, Bv, Cv,
    D, mu1 and mu2 by at most that much, and the maps S, g_mu, g_xx, g_xy by their first-order partials times it, plus k u of their
    own magnitude for the elementwise roundings.  The image gradient bound is the same correlation over the maps' bounds, plus k u
    of its sum of absolute terms.  Returns (bound on mean SSIM, bound on every element of the gradient)."""
    w = p["w"]
    ax, ay = conv_sep(p["x"].abs(), w), conv_sep(p["y"].abs(), w)
    axx, ayy, axy = conv_sep(p["x"] ** 2, w), conv_sep(p["y"] ** 2, w), conv_sep((p["x"] * p["y"]).abs(), w)
    e_mom = axx + ayy + 2 * axy + (ax + ay) ** 2  # magnitude of every second-moment combination and of the mu products
    err = {"mu1": ax, "mu2": ay, "A": 2 * ax * ay, "Bv": 2 * (axy + ax * ay), "Cv": ax ** 2 + ay ** 2, "D": e_mom}
    eb = {}
    for name in ("S", "g_mu", "g_xx", "g_xy"):
        v = {n: p[n].detach().clone().requires_grad_(True) for n in err}
        with torch.enable_grad():
            m = _map_fns(v["mu1"], v["mu2"], v["A"], v["Bv"], v["Cv"], v["D"])[name]
            parts = torch.autograd.grad(m.sum(), [v[n] for n in err], allow_unused=True)
        m = m.detach()
        tot = k * U32 * m.abs()
        for n, d in zip(err, parts):
            if d is not None:
                tot = tot + k * U32 * d.abs() * err[n]
        eb[name] = tot
    n = p["S"].numel()
    gs = abs(g_ssim) / n
    cabs = conv_sep(p["g_mu"].abs(), w) + 2 * p["x"].abs() * conv_sep(p["g_xx"].abs(), w) + p["y"].abs() * conv_sep(p["g_xy"].abs(), w)
    gb = gs * (conv_sep(eb["g_mu"], w) + 2 * p["x"].abs() * conv_sep(eb["g_xx"], w) + p["y"].abs() * conv_sep(eb["g_xy"], w))
    gb = gb + gs * k * U32 * cabs + abs(g_l1) / n * k * U32
    sb = eb["S"].mean() + k * U32 * p["S"].abs().mean()
    return float(sb), gb


def _normalize64(v):
    return v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def normal64(pred, gt, depth=None, scene_scale=5.0, g_out=1.0):
    """(normal_loss value, d value/d pred) in fp64, and the float32 error bound of each gradient element (an element whose
    |n - g| is within rounding of 0 may take either sign of the L1 term)."""
    v, g0 = pred.double().reshape(-1, 3), gt.double().reshape(-1, 3)
    sel = torch.ones(v.shape[0], dtype=torch.bool, device=v.device) if depth is None else \
        ((depth.reshape(-1) > 0) & (depth.reshape(-1) < scene_scale))
    cnt = int(sel.sum())
    n, g = _normalize64(v), _normalize64(g0)
    diff = n - g
    val = diff[sel].abs().mean() + 0.1 * (-(n[sel] * g[sel]).sum(-1).mean()) if cnt else torch.tensor(float("nan"), dtype=torch.float64)
    grad = torch.zeros_like(v)
    bound = torch.zeros_like(v)
    if cnt:
        len_ = v.norm(dim=-1, keepdim=True)
        c = len_.clamp_min(1e-12)
        gl, gc = g_out / (3 * cnt), 0.1 * g_out / cnt
        dn = gl * torch.sign(diff) - gc * g
        s = (dn * v).sum(-1, keepdim=True) / c ** 2
        pas = (len_ >= 1e-12).double()
        gv = dn / c - pas * s * v / len_.clamp_min(1e-300)
        grad[sel] = gv[sel]
        mag = dn.abs() / c + pas * ((dn.abs() * v.abs()).sum(-1, keepdim=True) / c ** 2) * v.abs() / len_.clamp_min(1e-300)
        amb = (diff.abs() <= 16 * U32).double() * 2 * abs(gl) / c  # the L1 sign is ambiguous within rounding of n == g
        bound[sel] = (64 * U32 * (mag + abs(gl) / c) + amb * (1 + pas * 1.0))[sel]
    return val, grad.reshape(pred.shape), bound.reshape(pred.shape)


def first_extremes(s):
    """Per row of s [P,3]: the first maximal and the first minimal index (NaN first), the rule torch's max(dim) / min(dim) follow."""
    s = s.double()
    imax = torch.zeros(s.shape[0], dtype=torch.long, device=s.device)
    imin = torch.zeros_like(imax)
    rows = torch.arange(s.shape[0], device=s.device)
    for k in (1, 2):
        bm, bn, sk = s[rows, imax], s[rows, imin], s[:, k]
        imax = torch.where(~bm.isnan() & ((sk > bm) | sk.isnan()), torch.full_like(imax, k), imax)
        imin = torch.where(~bn.isnan() & ((sk < bn) | sk.isnan()), torch.full_like(imin, k), imin)
    return imax, imin


def anisotropic64(scales, r=3.0, g_out=1.0):
    """(anisotropic_loss value, d value/d scales, per-element float32 error bound) in fp64 on the float32 scales.  The clamp's
    decision is ambiguous within rounding of ratio == r, so an element there may take either branch."""
    s = scales.double().reshape(-1, 3)
    P = s.shape[0]
    imax, imin = first_extremes(s)
    rows = torch.arange(P, device=s.device)
    mx, mn = s[rows, imax], s[rows, imin]
    den = mn + 1e-6
    q = mx / den
    val = (torch.clamp(q, min=r) - r).mean()
    g = g_out / P
    on = (q >= r).double()
    grad = torch.zeros_like(s)
    grad[rows, imax] += on * g / den
    grad[rows, imin] += on * (-g * mx / den ** 2)
    mag = torch.zeros_like(s)
    mag[rows, imax] += abs(g) / den
    mag[rows, imin] += abs(g) * mx.abs() / den ** 2
    amb = ((q - r).abs() <= 8 * U32 * q.abs()).double().unsqueeze(-1)
    bound = 16 * U32 * mag + amb * mag
    return val, grad.reshape(scales.shape), bound.reshape(scales.shape)
