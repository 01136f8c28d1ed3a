"""Differentiable fp64 PyTorch restatement of the rasterizer at tiny sizes (test infrastructure).

Purpose: pin the CPU oracle's forward AND backward independently of any CUDA code: the continuous part of the
forward (reference forward.cu:74-256 preprocess math, forward.cu:330-366 blend recurrence) is restated in torch
fp64 and differentiated by autograd, while the discrete decisions (tile lists, skip / terminate per pixel) are
taken from the oracle's forward and treated as constants — exactly what the reference's hand-written backward
does (backward.cu:415-599 replays the forward's decisions).
"""
from __future__ import annotations

import numpy as np
import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
         -0.5900435899266435]


def eval_sh(deg, sh, dirs):
    """sh [P,M,3], dirs [P,3] unit.  Same polynomials as forward.cu:20-71 / utils/sh_utils.py:57-112."""
    x, y, z = dirs[:, 0:1], dirs[:, 1:2], dirs[:, 2:3]
    res = SH_C0 * sh[:, 0]
    if deg > 0:
        res = res - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            res = res + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * sh[:, 6] + \
                SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8]
            if deg > 2:
                res = res + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10] + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + \
                    SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12] + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + \
                    SH_C3[5] * z * (xx - yy) * sh[:, 14] + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15]
    return res


def preprocess(means3D, scales, rotations, opacities, shs, view, proj, campos, W, H, tanfovx, tanfovy, sh_degree, scale_modifier,
               colors_precomp=None, cov3D_precomp=None, reference_clamp_grad=False):
    """Continuous per-Gaussian quantities in fp64: means2D [P,2], conic [P,3], rgb [P,3] (SH colours clamped at 0, precomputed
    colours as given), depth [P].  cov3D_precomp [P,6] (upper triangle, row by row) replaces scales / rotations.
    reference_clamp_grad: differentiate the +-1.3 tan(fov) clamp of the view-space position as the reference does (the values
    are the same either way)."""
    P = means3D.shape[0]
    hom = torch.cat([means3D, torch.ones(P, 1, dtype=means3D.dtype)], dim=1)
    p_hom = hom @ proj  # row-vector convention on the row-major buffer (auxiliary.h:58-77)
    p_w = 1.0 / (p_hom[:, 3] + 0.0000001)
    p_proj = p_hom[:, :3] * p_w[:, None]
    t = (hom @ view)[:, :3]
    depth = t[:, 2]
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    if cov3D_precomp is None:
        r, x, y, z = rotations.unbind(-1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z), 1 - 2 * (x * x + z * z),
                         2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).view(P, 3, 3)
        L = R * (scales * scale_modifier).unsqueeze(1)
        Sigma = L @ L.transpose(1, 2)
    else:
        c = cov3D_precomp
        Sigma = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], dim=-1).view(P, 3, 3)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    tx = torch.clamp(t[:, 0] / t[:, 2], -limx, limx) * t[:, 2]
    ty = torch.clamp(t[:, 1] / t[:, 2], -limy, limy) * t[:, 2]
    if reference_clamp_grad:
        # the reference's backward (backward.cu:175-176, 262-264) treats a clamped t.x (t.y) as a constant: no gradient to t.x and
        # none through the clamped value's dependence on t.z
        cx = (t[:, 0] / t[:, 2]).abs() > limx
        cy = (t[:, 1] / t[:, 2]).abs() > limy
        tx = torch.where(cx, tx.detach(), tx)
        ty = torch.where(cy, ty.detach(), ty)
    tz = t[:, 2]
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -(fx * tx) / (tz * tz), zero, fy / tz, -(fy * ty) / (tz * tz)], dim=-1).view(P, 2, 3)
    Wr = view[:3, :3].T  # world -> camera rotation (the buffer holds the transpose)
    T = J @ Wr
    cov = T @ Sigma @ T.transpose(1, 2)
    a = cov[:, 0, 0] + 0.3
    b = cov[:, 0, 1]
    c = cov[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c / det, -b / det, a / det], dim=-1)
    px = ((p_proj[:, 0] + 1.0) * W - 1.0) * 0.5
    py = ((p_proj[:, 1] + 1.0) * H - 1.0) * 0.5
    if colors_precomp is not None:
        rgb = colors_precomp
    else:
        d = means3D - campos[None]
        d = d / d.norm(dim=1, keepdim=True)
        rgb = torch.clamp_min(eval_sh(sh_degree, shs, d) + 0.5, 0.0)
    return torch.stack([px, py], dim=-1), conic, rgb, depth


def oracle_hits(fw, ranges, point_list, tile, xx, yy):
    """[entries, pixels] mask of the list entries of one tile that the oracle's forward blends at each pixel: power <= 0 and
    alpha >= 1/255 in fp32 (the oracle's rounding sequence, expf correctly rounded), up to the pixel's n_contrib."""
    from tests.helpers import oracle_power
    r0, r1 = int(ranges[tile, 0]), int(ranges[tile, 1])
    g = point_list[r0:r1].numpy()
    pix = np.stack([xx.reshape(-1).numpy(), yy.reshape(-1).numpy()], axis=-1).astype(np.float32)[None]
    co = fw["conic_opacity"][g][:, None]
    power = oracle_power(fw["means2D"][g][:, None], co, pix)
    alpha = np.minimum(np.float32(0.99), co[..., 3] * np.exp(power.astype(np.float64)).astype(np.float32))
    last = fw["n_contrib"][yy.reshape(-1).numpy(), xx.reshape(-1).numpy()].astype(np.int64)
    pos = np.arange(1, r1 - r0 + 1)[:, None]
    return torch.from_numpy((power <= 0) & (alpha >= np.float32(1.0 / 255.0)) & (pos <= last[None]))


def blend(means2D, conic, opac, rgb, depth, ranges, point_list, W, H, bg, decisions=None):
    """Blend with the oracle's tile lists; decisions (skip / terminate) are evaluated on detached values, or, with decisions (the
    oracle's forward), taken from the oracle's fp32 evaluation and its n_contrib."""
    color = torch.zeros(3, H, W, dtype=means2D.dtype)
    dimg = torch.zeros(1, H, W, dtype=means2D.dtype)
    aimg = torch.zeros(1, H, W, dtype=means2D.dtype)
    gx = (W + 15) // 16
    for tile in range(ranges.shape[0]):
        ty, tx = divmod(tile, gx)
        ys = torch.arange(ty * 16, min(ty * 16 + 16, H))
        xs = torch.arange(tx * 16, min(tx * 16 + 16, W))
        if len(ys) == 0 or len(xs) == 0:
            continue
        yy, xx = torch.meshgrid(ys, xs, indexing="ij")
        pxf, pyf = xx.reshape(-1).to(means2D.dtype), yy.reshape(-1).to(means2D.dtype)
        n = pxf.shape[0]
        T = torch.ones(n, dtype=means2D.dtype)
        C = torch.zeros(n, 3, dtype=means2D.dtype)
        D = torch.zeros(n, dtype=means2D.dtype)
        done = torch.zeros(n, dtype=torch.bool)
        hits = None if decisions is None else oracle_hits(decisions, ranges, point_list, tile, xx, yy)
        for j in range(int(ranges[tile, 0]), int(ranges[tile, 1])):
            if hits is not None and not bool(hits[j - int(ranges[tile, 0])].any()):
                continue  # blended nowhere in the tile: contributes nothing
            if bool(done.all()):
                break  # every pixel has terminated: the rest of the list contributes nothing
            g = int(point_list[j])
            dx, dy = means2D[g, 0] - pxf, means2D[g, 1] - pyf
            power = -0.5 * (conic[g, 0] * dx * dx + conic[g, 2] * dy * dy) - conic[g, 1] * dx * dy
            alpha = torch.clamp_max(opac[g] * torch.exp(power), 0.99)
            with torch.no_grad():
                if hits is not None:
                    active = hits[j - int(ranges[tile, 0])]
                else:
                    active = (~done) & (power <= 0) & (alpha >= 1.0 / 255.0)
                    term = active & (T * (1 - alpha) < 0.0001)
                    done = done | term
                    active = active & ~term
            w = torch.where(active, alpha * T, torch.zeros_like(T))
            C = C + w[:, None] * rgb[g][None]
            D = D + w * depth[g]
            T = torch.where(active, T * (1 - alpha), T)
        hh, ww = len(ys), len(xs)
        color[:, ys[0]:ys[0] + hh, xs[0]:xs[0] + ww] = (C + T[:, None] * bg[None]).T.reshape(3, hh, ww)
        dimg[0, ys[0]:ys[0] + hh, xs[0]:xs[0] + ww] = D.reshape(hh, ww)
        aimg[0, ys[0]:ys[0] + hh, xs[0]:xs[0] + ww] = (1 - T).reshape(hh, ww)
    return color, dimg, aimg


def render(a, oracle_fw, reference_clamp_grad=False, oracle_decisions=False):
    """a: resolved case (tests/helpers.resolve): shs or colors_precomp, scales/rotations or cov3D_precomp.  Returns the images and
    the fp64 leaf tensors (one per input the case provides; the absent ones are None).  oracle_decisions: every skip / terminate
    decision is the oracle's fp32 one (else each is taken on the fp64 values)."""
    f64 = lambda t: None if t is None else t.detach().cpu().double().clone().requires_grad_(True)  # noqa: E731
    leaves = {k: f64(a[k]) for k in ("means3D", "scales", "rotations", "opacities", "shs", "colors_precomp", "cov3D_precomp")}
    view, proj, campos = a["view"].cpu().double(), a["proj"].cpu().double(), a["campos"].cpu().double()
    m2d, conic, rgb, depth = preprocess(leaves["means3D"], leaves["scales"], leaves["rotations"], leaves["opacities"], leaves["shs"], view, proj,
                                        campos, a["W"], a["H"], a["tanfovx"], a["tanfovy"], a["sh_degree"], a["scale_modifier"],
                                        colors_precomp=leaves["colors_precomp"], cov3D_precomp=leaves["cov3D_precomp"],
                                        reference_clamp_grad=reference_clamp_grad)
    m2d.retain_grad()
    ranges = torch.from_numpy(oracle_fw["ranges"].astype(np.int64))
    plist = torch.from_numpy(oracle_fw["point_list"].astype(np.int64))
    color, dimg, aimg = blend(m2d, conic, leaves["opacities"].reshape(-1), rgb, depth, ranges, plist, a["W"], a["H"], a["bg"].cpu().double(),
                              decisions=oracle_fw if oracle_decisions else None)
    return color, dimg, aimg, leaves, m2d
