"""The coarse trainers' projection estimate and better-normal loss restated op for op in torch — test infrastructure.

"SS/" = sugar/sugar_scene/sugar_model.py, "CD/" = sugar/sugar_trainers/coarse_density.py (coarse_sdf.py :732-760 is the same code).
``get_normals`` is SS/:817-839 without a surface mesh (get_smallest_axis, SS/:801-815).  ``projection_estimate`` is CD/:704-707,
``better_normal_loss`` CD/:756-780 before the trainer's ``.mean()``, and ``density_block`` the whole regularisation block
CD/:683-781 with the trainer's default flags: density mode, projection estimate, density_factor 1, factors 0.2 and 0.2.  It
reuses the field's restatement (tests/sugar_field_ref.py) for get_field_values.

Run in float64 they are the oracle; in float32 they are torch's own graph.  torch fixes no order for the 3-term sums, so the
sign decisions sigma = sign(n_j . n_i) of a float32 evaluation come from ``pinned_signs``: the normals from a quaternion_to_matrix
whose |q|^2 is summed left to right, and the dot as (a0 b0 + a1 b1) + a2 b2, one rounding per op.  ``better_normal_loss`` takes
those decisions through ``sign`` so that the float64 oracle uses the same ones.
"""
from __future__ import annotations

import torch

from tests import sugar_field_ref as SF
from tests import sugar_ref


def quaternion_to_matrix_pinned(q):
    """pytorch3d's quaternion_to_matrix with |q|^2 = ((r r + i i) + j j) + k k."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (((r * r + i * i) + j * j) + k * k)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def get_normals(self, pinned=False):  # SS/:817-839, estimate_from_points=False, no surface mesh -> get_smallest_axis
    rotation_matrices = (quaternion_to_matrix_pinned if pinned else sugar_ref.quaternion_to_matrix)(self.quaternions)
    smallest_axis_idx = self.scaling.min(dim=-1)[1][..., None, None].expand(-1, 3, -1)
    return rotation_matrices.gather(2, smallest_axis_idx).squeeze(dim=2)


def projection_estimate(self, sdf_samples, sdf_gaussian_idx):  # CD/:706-707
    samples_gaussian_normals = get_normals(self)[sdf_gaussian_idx]
    return ((sdf_samples - self.points[sdf_gaussian_idx]) * samples_gaussian_normals).sum(dim=-1)


def pinned_signs(self, sdf_gaussian_idx):
    """sigma [N,K] of CD/:763-765 in the model's dtype with the pinned roundings (see the module docstring)."""
    with torch.no_grad():
        n = get_normals(self, pinned=True)
        idx = self.knn_idx[sdf_gaussian_idx]
        return torch.sign(dot3(n[idx], n[sdf_gaussian_idx][:, None]))


def better_normal_loss(self, sdf_samples, sdf_gaussian_idx, closest_gaussian_opacities, sign=None):
    """CD/:756-780 with sdf_better_normal_gradient_through_normal_only = True -> [N].  ``sign`` [N,K], when given, replaces
    torch.sign(...) of CD/:763-765 (it is detached there anyway)."""
    closest_gaussians_idx = self.knn_idx[sdf_gaussian_idx]
    closest_min_scaling = self.scaling.min(dim=-1)[0][closest_gaussians_idx].detach().view(len(sdf_samples), -1)
    closest_gaussian_normals = get_normals(self)[closest_gaussians_idx]
    samples_gaussian_normals = get_normals(self)[sdf_gaussian_idx]
    if sign is None:
        sign = torch.sign((closest_gaussian_normals * samples_gaussian_normals[:, None]).sum(dim=-1, keepdim=True))
    else:
        sign = sign[..., None].to(closest_gaussian_normals.dtype)
    closest_gaussian_normals = closest_gaussian_normals * sign.detach()
    closest_gaussian_opacities = closest_gaussian_opacities.detach()
    normal_weights = ((sdf_samples[:, None] - self.points[closest_gaussians_idx]) * closest_gaussian_normals).sum(dim=-1).abs()
    normal_weights = normal_weights.detach()
    normal_weights = closest_gaussian_opacities * normal_weights / closest_min_scaling.clamp(min=1e-6) ** 2
    normal_weights_sum = normal_weights.sum(dim=-1).detach()
    normal_weights = normal_weights / normal_weights_sum.unsqueeze(-1).clamp(min=1e-6)
    return (samples_gaussian_normals - (normal_weights[..., None] * closest_gaussian_normals).sum(dim=-2)).pow(2).sum(dim=-1)


def density_block(self, sdf_samples, sdf_gaussian_idx, estimate=projection_estimate, normal_loss=better_normal_loss, sign=None,
                  sdf_estimation_factor=0.2, sdf_better_normal_factor=0.2):
    """coarse_density's regularisation block (CD/:692-781) with its default flags over a fixed sample set -> loss.  The field is
    self.get_field_values (bind the library's to run it in CUDA); ``estimate`` and ``normal_loss`` are the two computations
    (the restatements above, or the library's).  ``sign`` goes to the restated normal loss only."""
    fields = self.get_field_values(sdf_samples, sdf_gaussian_idx, return_sdf=False, density_threshold=1., density_factor=1.,
                                   return_sdf_grad=False, sdf_grad_max_value=10., return_closest_gaussian_opacities=True,
                                   return_beta=True)
    sdf_estimation = estimate(self, sdf_samples, sdf_gaussian_idx)
    beta = fields['beta']
    densities = fields['density']
    target_densities = torch.exp(-0.5 * sdf_estimation.pow(2) / beta.pow(2))
    sdf_estimation_loss = (densities - target_densities).abs()
    loss = sdf_estimation_factor * sdf_estimation_loss.mean()
    kw = {} if sign is None else {"sign": sign}
    sdf_better_normal_loss = normal_loss(self, sdf_samples, sdf_gaussian_idx, fields['closest_gaussian_opacities'], **kw)
    return loss + sdf_better_normal_factor * sdf_better_normal_loss.mean()


FieldModel = SF.FieldModel
Getters = SF.Getters
sample_points_in_gaussians = SF.sample_points_in_gaussians
