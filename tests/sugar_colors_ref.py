"""SuGaR's per-Gaussian colours restated for the tests of render_sugar_raw() — test infrastructure.

"SH/" = sugar/sugar_utils/spherical_harmonics.py, "SS/" = sugar/sugar_scene/sugar_model.py.  tests/sugar_ref.py states SuGaR's
eval_sh for degrees 0-3; SuGaR stores degree-4 coefficients (M = 25) and its eval_sh evaluates them, so this module states:

  * ``eval_sh`` for degrees 0-4 in torch, op for op as SH/:117-172 writes it, and a SuGaR stand-in whose get_points_rgb uses it;
  * ``basis``: SH/'s basis factors for any array module and float type, in SH/'s operation order (float32: one rounding per op);
  * ``colors_np``: get_points_rgb in numpy float32, one rounding per torch op (the arithmetic gsr_sugar_colors implements);
  * ``colors_vjp``: the closed-form backward gsr_sugar_colors_backward implements, in float64;
  * ``colors_forced``: the same colours in torch with the clamp decisions fixed, for fp64 autograd;
  * a mesh-bound stand-in whose points, scaling and quaternions are torch functions of other leaves.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import sugar_ref as SR

C0, C1, C2, C3 = SR.C0, SR.C1, SR.C2, SR.C3
C4 = (2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892, 0.10578554691520431, -0.6690465435572892,
      0.47308734787878004, -1.7701307697799304, 0.6258357354491761)
SIGN = np.ones(25)
SIGN[[1, 3]] = -1.0  # result - C1 y sh1 + C1 z sh2 - C1 x sh3


def eval_sh(deg, sh, dirs):
    """SH/:117-172 for degrees 0-4: sh [..., C, >= (deg+1)^2], dirs [..., 3]."""
    assert 0 <= deg <= 4
    assert sh.shape[-1] >= (deg + 1) ** 2
    result = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            result = (result + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] + C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] +
                      C2[3] * xz * sh[..., 7] + C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10] +
                          C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12] +
                          C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14] +
                          C3[6] * x * (xx - 3 * yy) * sh[..., 15])
                if deg > 3:
                    result = (result + C4[0] * xy * (xx - yy) * sh[..., 16] + C4[1] * yz * (3 * xx - yy) * sh[..., 17] +
                              C4[2] * xy * (7 * zz - 1) * sh[..., 18] + C4[3] * yz * (7 * zz - 3) * sh[..., 19] +
                              C4[4] * (zz * (35 * zz - 30) + 3) * sh[..., 20] + C4[5] * xz * (7 * zz - 3) * sh[..., 21] +
                              C4[6] * (xx - yy) * (7 * zz - 1) * sh[..., 22] + C4[7] * xz * (xx - 3 * yy) * sh[..., 23] +
                              C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy)) * sh[..., 24])
    return result


def basis(deg, x, y, z, dtype=np.float32):
    """SH/'s factor of each coefficient, (deg+1)^2 arrays, without the signs of terms 1 and 3 (SIGN): in ``dtype`` every product
    and sum rounds once, in SH/'s order; constants and integer literals are rounded to ``dtype`` once, as torch does."""
    f = lambda v: dtype(v)  # noqa: E731
    b = [np.full_like(x, f(C0))]
    if deg > 0:
        b += [f(C1) * y, f(C1) * z, f(C1) * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [f(C2[0]) * xy, f(C2[1]) * yz, f(C2[2]) * ((f(2) * zz - xx) - yy), f(C2[3]) * xz, f(C2[4]) * (xx - yy)]
        if deg > 2:
            b += [(f(C3[0]) * y) * (f(3) * xx - yy), (f(C3[1]) * xy) * z, (f(C3[2]) * y) * ((f(4) * zz - xx) - yy),
                  (f(C3[3]) * z) * ((f(2) * zz - f(3) * xx) - f(3) * yy), (f(C3[4]) * x) * ((f(4) * zz - xx) - yy),
                  (f(C3[5]) * z) * (xx - yy), (f(C3[6]) * x) * (xx - f(3) * yy)]
            if deg > 3:
                b += [(f(C4[0]) * xy) * (xx - yy), (f(C4[1]) * yz) * (f(3) * xx - yy), (f(C4[2]) * xy) * (f(7) * zz - f(1)),
                      (f(C4[3]) * yz) * (f(7) * zz - f(3)), f(C4[4]) * (zz * (f(35) * zz - f(30)) + f(3)),
                      (f(C4[5]) * xz) * (f(7) * zz - f(3)), (f(C4[6]) * (xx - yy)) * (f(7) * zz - f(1)),
                      (f(C4[7]) * xz) * (xx - f(3) * yy), f(C4[8]) * (xx * (xx - f(3) * yy) - yy * (f(3) * xx - yy))]
    return b


def view_dirs_np(positions, campos):
    """F.normalize(positions - campos, dim=-1) in float32: sqrt of the left-to-right sum of squares, clamped at 1e-12."""
    f = np.float32
    d = np.asarray(positions, dtype=f) - np.asarray(campos, dtype=f).reshape(1, 3)
    n = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return d / np.maximum(n, f(1e-12))[:, None]


def colors_np(deg, sh, dirs):
    """get_points_rgb in float32: sh [P, >= (deg+1)^2, 3] (cat(dc, rest)), dirs [P,3] -> (colours [P,3], pre-clamp values [P,3])."""
    f = np.float32
    sh = np.asarray(sh, dtype=f)
    d = np.asarray(dirs, dtype=f)
    b = basis(deg, d[:, 0:1], d[:, 1:2], d[:, 2:3], f)
    r = b[0] * sh[:, 0]
    if deg > 0:
        r = ((r - b[1] * sh[:, 1]) + b[2] * sh[:, 2]) - b[3] * sh[:, 3]
        for k in range(4, (deg + 1) ** 2):
            r = r + b[k] * sh[:, k]
    pre = r + f(0.5)
    return np.where(pre < 0, f(0), pre).astype(f), pre


def _grad_basis(deg, x, y, z):
    """Gradients (d/dx, d/dy, d/dz) of the unsigned basis polynomials, float64."""
    o = np.zeros_like(x)
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    g = [(o, o, o)]
    if deg > 0:
        g += [(o, C1 + o, o), (o, o, C1 + o), (C1 + o, o, o)]
    if deg > 1:
        g += [(C2[0] * y, C2[0] * x, o), (o, C2[1] * z, C2[1] * y), (-2 * C2[2] * x, -2 * C2[2] * y, 4 * C2[2] * z),
              (C2[3] * z, o, C2[3] * x), (2 * C2[4] * x, -2 * C2[4] * y, o)]
    if deg > 2:
        g += [(6 * C3[0] * xy, C3[0] * (3 * xx - 3 * yy), o), (C3[1] * yz, C3[1] * xz, C3[1] * xy),
              (-2 * C3[2] * xy, C3[2] * (4 * zz - xx - 3 * yy), 8 * C3[2] * yz),
              (-6 * C3[3] * xz, -6 * C3[3] * yz, C3[3] * (6 * zz - 3 * xx - 3 * yy)),
              (C3[4] * (4 * zz - 3 * xx - yy), -2 * C3[4] * xy, 8 * C3[4] * xz), (2 * C3[5] * xz, -2 * C3[5] * yz, C3[5] * (xx - yy)),
              (C3[6] * (3 * xx - 3 * yy), -6 * C3[6] * xy, o)]
    if deg > 3:
        xyz = xy * z
        g += [(C4[0] * (3 * xx * y - yy * y), C4[0] * (xx * x - 3 * x * yy), o),
              (6 * C4[1] * xyz, C4[1] * (3 * xx * z - 3 * yy * z), C4[1] * (3 * xx * y - yy * y)),
              (C4[2] * y * (7 * zz - 1), C4[2] * x * (7 * zz - 1), 14 * C4[2] * xyz),
              (o, C4[3] * z * (7 * zz - 3), C4[3] * y * (21 * zz - 3)),
              (o, o, C4[4] * (140 * zz * z - 60 * z)),
              (C4[5] * z * (7 * zz - 3), o, C4[5] * x * (21 * zz - 3)),
              (2 * C4[6] * x * (7 * zz - 1), -2 * C4[6] * y * (7 * zz - 1), 14 * C4[6] * z * (xx - yy)),
              (C4[7] * z * (3 * xx - 3 * yy), -6 * C4[7] * xyz, C4[7] * x * (xx - 3 * yy)),
              (C4[8] * (4 * xx * x - 12 * x * yy), C4[8] * (4 * yy * y - 12 * xx * y), o)]
    return g


def colors_vjp(deg, sh, g, passed, directions=None, positions=None, campos=None):
    """The closed form of gsr_sugar_colors_backward in float64: dL/dcolors g [P,3], the clamp's pass mask [P,3] (pre >= 0) ->
    (dL/dsh [P, (deg+1)^2, 3], dL/ddirections or dL/dpositions [P,3])."""
    sh = np.asarray(sh, dtype=np.float64)
    gp = np.asarray(g, dtype=np.float64) * passed
    if directions is not None:
        v = np.asarray(directions, dtype=np.float64)
    else:
        d = np.asarray(positions, dtype=np.float64) - np.asarray(campos, dtype=np.float64).reshape(1, 3)
        n = np.linalg.norm(d, axis=1)
        v = d / np.maximum(n, 1e-12)[:, None]
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    K = (deg + 1) ** 2
    b = basis(deg, x, y, z, np.float64)
    dsh = np.stack([SIGN[k] * b[k][:, None] * gp for k in range(K)], 1)
    w = [SIGN[k] * (gp * sh[:, k]).sum(1) for k in range(K)]
    gb = _grad_basis(deg, x, y, z)
    dv = np.stack([sum(w[k] * gb[k][a] for k in range(K)) for a in range(3)], 1)
    if directions is not None:
        return dsh, dv
    big = n >= 1e-12
    u = d / np.where(big, n, 1.0)[:, None]
    dd = np.where(big[:, None], (dv - u * (u * dv).sum(1, keepdims=True)) / np.where(big, n, 1.0)[:, None], dv / 1e-12)
    return dsh, dd


def colors_forced(deg, sh, passed, directions=None, positions=None, campos=None):
    """get_points_rgb in torch with the clamp replaced by the fixed mask ``passed`` (the decisions are piecewise constant; this is
    what autograd differentiates).  sh [P, >= (deg+1)^2, 3]."""
    if directions is None:
        directions = torch.nn.functional.normalize(positions - campos, dim=-1)
    n = (deg + 1) ** 2
    return (eval_sh(deg, sh[:, :n].transpose(-1, -2), directions) + 0.5) * passed


class SugarModel4(SR.SugarModel):
    """tests/sugar_ref.SugarModel with SuGaR's eval_sh up to degree 4 in get_points_rgb (SS/:711-755)."""

    def get_points_rgb(self, positions=None, camera_centers=None, directions=None, sh_levels=None, sh_coordinates=None):
        if positions is None:
            positions = self.points
        if camera_centers is not None:
            render_directions = torch.nn.functional.normalize(positions - camera_centers, dim=-1)
        elif directions is not None:
            render_directions = directions
        else:
            raise ValueError("Either camera_centers or directions must be provided.")
        if sh_coordinates is None:
            sh_coordinates = self.sh_coordinates
        if sh_levels is not None:
            sh_coordinates = sh_coordinates[:, :sh_levels ** 2]
        shs_view = sh_coordinates.transpose(-1, -2).view(-1, 3, sh_levels ** 2)
        sh2rgb = eval_sh(sh_levels - 1, shs_view, render_directions)
        return torch.clamp_min(sh2rgb + 0.5, 0.0).view(-1, 3)


class MeshBoundModel(SugarModel4):
    """A mesh-bound SuGaR stand-in (SS/:365-392 with one Gaussian per face): points are the barycentres of triangles whose vertices
    are the leaf ``_vertices`` [3P,3]; scaling = exp(_scales) * exp(_scale_shift); quaternions = _quaternions * _quat_gain.  The
    leaves _points, _scales and _quaternions of the unbound model stay for construction only and are not read by the getters
    except _scales and _quaternions."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        grad = self._points.requires_grad
        P = self._points.shape[0]
        gen = torch.Generator().manual_seed(17)
        off = (0.01 * torch.randn(P, 3, 3, generator=gen)).to(self._points.device)
        off = off - off.mean(1, keepdim=True)
        verts = (self._points.detach()[:, None, :] + off).reshape(-1, 3)
        self._vertices = verts.contiguous().requires_grad_(grad)
        self._scale_shift = torch.zeros(1, 3, device=self._points.device, requires_grad=grad)
        self._quat_gain = torch.ones(1, 1, device=self._points.device, requires_grad=grad)
        del self.leaves["_points"]
        self.leaves.update(_vertices=self._vertices, _scale_shift=self._scale_shift, _quat_gain=self._quat_gain)

    points = property(lambda s: s._vertices.view(-1, 3, 3).mean(dim=1))
    n_points = property(lambda s: s._vertices.shape[0] // 3)
    scaling = property(lambda s: torch.exp(s._scales) * torch.exp(s._scale_shift))
    quaternions = property(lambda s: s._quaternions * s._quat_gain)
