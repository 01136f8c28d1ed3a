"""Restatements of SuGaR's sample_points_in_gaussians ("SS/" = sugar/sugar_scene/sugar_model.py:757-799) for the tests of
autovfx_b200.sugar_field.sample_points_in_gaussians:

  sample_points_in_gaussians  SuGaR's method as written: torch.multinomial on cumsum(w) / sum(w), then pytorch3d's quaternion_apply
  select_rows                 the drop-in's choice of rows given u: float64 prefix over all P rows and the inverse-CDF search
  place                       the drop-in's placement given rows and z: the kernel's float32 op order, one torch op per rounding

pytorch3d is not a dependency: its quaternion ops (pytorch3d/transforms/rotation_conversions.py) are restated below.
"""
from __future__ import annotations

import torch


def quaternion_raw_multiply(a, b):  # pytorch3d
    aw, ax, ay, az = torch.unbind(a, -1)
    bw, bx, by, bz = torch.unbind(b, -1)
    ow = aw * bw - ax * bx - ay * by - az * bz
    ox = aw * bx + ax * bw + ay * bz - az * by
    oy = aw * by - ax * bz + ay * bw + az * bx
    oz = aw * bz + ax * by - ay * bx + az * bw
    return torch.stack((ow, ox, oy, oz), -1)


def quaternion_invert(quaternion):  # pytorch3d: the conjugate, not the inverse
    scaling = torch.tensor([1, -1, -1, -1], device=quaternion.device)
    return quaternion * scaling


def quaternion_apply(quaternion, point):  # pytorch3d
    real_parts = point.new_zeros(point.shape[:-1] + (1,))
    point_as_quaternion = torch.cat((real_parts, point), -1)
    out = quaternion_raw_multiply(quaternion_raw_multiply(quaternion, point_as_quaternion), quaternion_invert(quaternion))
    return out[..., 1:]


def sample_points_in_gaussians(self, num_samples, sampling_scale_factor=1., mask=None, probabilities_proportional_to_opacity=False,
                               probabilities_proportional_to_volume=True, generator=None):
    """SS/:772-799 as written (``generator`` feeds both draws; None: the default generator of the points' device)."""
    if mask is None:
        scaling = self.scaling
    else:
        scaling = self.scaling[mask]
    if probabilities_proportional_to_volume:
        areas = scaling[..., 0] * scaling[..., 1] * scaling[..., 2]
    else:
        areas = torch.ones_like(scaling[..., 0])
    if probabilities_proportional_to_opacity:
        if mask is None:
            areas = areas * self.strengths.view(-1)
        else:
            areas = areas * self.strengths[mask].view(-1)
    areas = areas.abs()
    cum_probs = areas.cumsum(dim=-1) / areas.sum(dim=-1, keepdim=True)
    random_indices = torch.multinomial(cum_probs, num_samples=num_samples, replacement=True, generator=generator)
    if mask is not None:
        valid_indices = torch.arange(self.points.shape[0], device=self.points.device)[mask]
        random_indices = valid_indices[random_indices]
    noise = torch.randn(self.points[random_indices].shape, generator=generator, device=self.points.device, dtype=self.points.dtype)
    random_points = self.points[random_indices] + quaternion_apply(
        self.quaternions[random_indices],
        sampling_scale_factor * self.scaling[random_indices] * noise)
    return random_points, random_indices


def weights(scaling, strengths=None, mask=None, volume=True):
    """SuGaR's areas over all P rows (float32 as SuGaR evaluates them), 0 on unselected rows."""
    w = scaling[:, 0] * scaling[:, 1] * scaling[:, 2] if volume else torch.ones_like(scaling[:, 0])
    if strengths is not None:
        w = w * strengths.reshape(-1)
    w = w.abs()
    return w if mask is None else torch.where(mask, w, torch.zeros_like(w))


def prefix(w, mask=None):
    """T [P] (float64): the prefix over all rows of t_i = mask_i C_i, C_i = the float64 prefix of w."""
    c = w.double().cumsum(0)
    t = c if mask is None else torch.where(mask, c, torch.zeros_like(c))
    return t.cumsum(0)


def select_rows(T, u):
    """The first row whose prefix exceeds u * total, u * total capped below the total; (rows, total)."""
    total = T[-1]
    x = torch.minimum(u * total, torch.nextafter(total, torch.zeros_like(total)))
    return torch.searchsorted(T, x, right=True), total


def place(points, scaling, quaternions, rows, z, f):
    """points[rows] + quaternion_apply(q[rows], (f * s[rows]) * z), written component by component in the kernel's order."""
    p, s, q = points[rows], scaling[rows], quaternions[rows]
    v0, v1, v2 = ((f * s) * z).unbind(-1)
    qw, qx, qy, qz = q.unbind(-1)
    zero = torch.zeros_like(qw)
    aw = qw * zero - qx * v0 - qy * v1 - qz * v2
    ax = qw * v0 + qx * zero + qy * v2 - qz * v1
    ay = qw * v1 - qx * v2 + qy * zero + qz * v0
    az = qw * v2 + qx * v1 - qy * v0 + qz * zero
    bw, bx, by, bz = qw, -qx, -qy, -qz
    rx = aw * bx + ax * bw + ay * bz - az * by
    ry = aw * by - ax * bz + ay * bw + az * bx
    rz = aw * bz + ax * by - ay * bx + az * bw
    return p + torch.stack((rx, ry, rz), -1)


def place_pytorch3d(points, scaling, quaternions, rows, z, f):
    """The same placement through the pytorch3d restatement (SS/:795-797 with the rows and the noise given)."""
    return points[rows] + quaternion_apply(quaternions[rows], f * scaling[rows] * z)


def draws(N, device, seed):
    """The drop-in's draws for torch.manual_seed(seed): u = rand(N, float64), then z = randn(N, 3)."""
    torch.manual_seed(seed)
    u = torch.rand(N, dtype=torch.float64, device=device)
    z = torch.randn((N, 3), dtype=torch.float32, device=device)
    return u, z


class Getters:
    """A model whose getters return given tensors."""

    def __init__(self, points, scaling, quaternions, strengths=None):
        self.points, self.scaling, self.quaternions, self.strengths = points, scaling, quaternions, strengths


class RawModel:
    """SuGaR-like getters over raw leaves: scaling = exp(raw), quaternions = normalize(raw), strengths = sigmoid(raw)."""

    def __init__(self, points, log_scaling, raw_quaternions, raw_densities):
        self._points, self._scales, self._quaternions, self.all_densities = points, log_scaling, raw_quaternions, raw_densities

    points = property(lambda s: s._points)
    scaling = property(lambda s: torch.exp(s._scales))
    quaternions = property(lambda s: torch.nn.functional.normalize(s._quaternions, dim=-1))
    strengths = property(lambda s: torch.sigmoid(s.all_densities))
