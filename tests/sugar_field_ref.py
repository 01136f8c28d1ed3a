"""SuGaR's SDF-regularisation field restated op for op in torch — test infrastructure.

"SS/" = sugar/sugar_scene/sugar_model.py, "CD/" = sugar/sugar_trainers/coarse_density.py, "CS/" = sugar/sugar_trainers/coarse_sdf.py.
The model module imports pytorch3d, so the methods are restated here and bound to a stand-in model: ``get_covariance``
(SS/:602-622), ``get_beta`` 'average' (SS/:1043-1116), ``get_field_values`` (SS/:1118-1187), ``get_gaussians_closest_to_samples``
(SS/:1206-1214, pytorch3d's knn_points as a brute force) and ``compute_density`` (SS/:1216-1239).  Run in float64 they are the
oracle; in float32 they are torch's own graph, which the CUDA path must match as well as it does.  ``density_block`` and
``sdf_block`` are the trainers' SDF-regularisation blocks (CD/:683-742, CS/:671-721) with their default flags, over a fixed
sample set, with the projection estimate (``use_projection_as_estimation``) so that no camera is needed.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import sugar_ref


def quaternion_to_matrix(q):
    return sugar_ref.quaternion_to_matrix(q)


# ------------------------------------------------------------------------------------------------ the methods
def get_covariance(self, return_full_matrix=False, return_sqrt=False, inverse_scales=False):  # SS/:602-622
    scaling = self.scaling
    if inverse_scales:
        scaling = 1. / scaling.clamp(min=1e-8)
    scaled_rotation = quaternion_to_matrix(self.quaternions) * scaling[:, None]
    if return_sqrt:
        return scaled_rotation
    cov3Dmatrix = scaled_rotation @ scaled_rotation.transpose(-1, -2)
    if return_full_matrix:
        return cov3Dmatrix
    raise NotImplementedError("the packed covariance is not used by the field")


def get_beta(self, x, closest_gaussians_idx=None, closest_gaussians_opacities=None, densities=None, opacity_min_clamp=1e-32):
    if self.beta_mode == 'average':  # SS/:1063-1066
        if closest_gaussians_idx is None:
            raise ValueError("closest_gaussians_idx must be provided when using beta_mode='average'.")
        return self.scaling.min(dim=-1)[0][closest_gaussians_idx].mean(dim=1)
    raise ValueError("Unknown beta_mode.")  # 'learnable' and 'weighted_average' are not restated


def get_field_values(self, x, gaussian_idx=None, closest_gaussians_idx=None, gaussian_strengths=None, gaussian_centers=None,
                     gaussian_inv_scaled_rotation=None, return_sdf=True, density_threshold=1., density_factor=1., return_sdf_grad=False,
                     sdf_grad_max_value=10., opacity_min_clamp=1e-16, return_closest_gaussian_opacities=False, return_beta=False):
    """SS/:1118-1187 (without the sdf_grad branch, which is not restated)."""
    assert not return_sdf_grad
    if gaussian_strengths is None:
        gaussian_strengths = self.strengths
    if gaussian_centers is None:
        gaussian_centers = self.points
    if gaussian_inv_scaled_rotation is None:
        gaussian_inv_scaled_rotation = self.get_covariance(return_full_matrix=True, return_sqrt=True, inverse_scales=True)
    if closest_gaussians_idx is None:
        closest_gaussians_idx = self.knn_idx[gaussian_idx]
    closest_gaussian_centers = gaussian_centers[closest_gaussians_idx]
    closest_gaussian_inv_scaled_rotation = gaussian_inv_scaled_rotation[closest_gaussians_idx]
    closest_gaussian_strengths = gaussian_strengths[closest_gaussians_idx]
    fields = {}
    shift = (x[:, None] - closest_gaussian_centers)
    warped_shift = closest_gaussian_inv_scaled_rotation.transpose(-1, -2) @ shift[..., None]
    neighbor_opacities = (warped_shift[..., 0] * warped_shift[..., 0]).sum(dim=-1).clamp(min=0., max=1e8)
    neighbor_opacities = density_factor * closest_gaussian_strengths[..., 0] * torch.exp(-1. / 2 * neighbor_opacities)
    densities = neighbor_opacities.sum(dim=-1)
    fields['density'] = densities.clone()
    density_mask = densities >= 1.
    densities[density_mask] = densities[density_mask] / (densities[density_mask].detach() + 1e-12)
    if return_closest_gaussian_opacities:
        fields['closest_gaussian_opacities'] = neighbor_opacities
    if return_sdf or return_sdf_grad or return_beta:
        beta = self.get_beta(x, closest_gaussians_idx=closest_gaussians_idx, closest_gaussians_opacities=neighbor_opacities,
                             densities=densities, opacity_min_clamp=opacity_min_clamp)
        clamped_densities = densities.clamp(min=opacity_min_clamp)
    if return_beta:
        fields['beta'] = beta
    if return_sdf:
        sdf_values = beta * (torch.sqrt(-2. * torch.log(clamped_densities)) - np.sqrt(-2. * np.log(min(density_threshold, 1.))))
        fields['sdf'] = sdf_values
    return fields


def get_gaussians_closest_to_samples(self, x, n_closest_gaussian=None):  # SS/:1206-1214, knn_points as a brute force
    if n_closest_gaussian is None:
        n_closest_gaussian = self.knn_to_track
    p = self.points.detach()
    out = []
    for s in range(0, x.shape[0], 4096):
        d = ((x.detach()[s:s + 4096, None, :] - p[None]) ** 2).sum(-1)
        out.append(d.topk(n_closest_gaussian, dim=1, largest=False).indices)
    return torch.cat(out) if out else torch.empty((0, n_closest_gaussian), dtype=torch.int64, device=x.device)


def compute_density(self, x, closest_gaussians_idx=None, density_factor=1., return_closest_gaussian_opacities=False):  # SS/:1216-1239
    if closest_gaussians_idx is None:
        closest_gaussians_idx = self.get_gaussians_closest_to_samples(x)
    close_gaussian_centers = self.points[closest_gaussians_idx]
    close_gaussian_inv_scaled_rotation = self.get_covariance(return_full_matrix=True, return_sqrt=True, inverse_scales=True)[closest_gaussians_idx]
    close_gaussian_strengths = self.strengths[closest_gaussians_idx]
    shift = (x[:, None] - close_gaussian_centers)
    warped_shift = close_gaussian_inv_scaled_rotation.transpose(-1, -2) @ shift[..., None]
    neighbor_opacities = (warped_shift[..., 0] * warped_shift[..., 0]).sum(dim=-1).clamp(min=0., max=1e8)
    neighbor_opacities = density_factor * close_gaussian_strengths[..., 0] * torch.exp(-1. / 2 * neighbor_opacities)
    densities = neighbor_opacities.sum(dim=-1)
    if return_closest_gaussian_opacities:
        return densities, neighbor_opacities
    return densities


# ------------------------------------------------------------------------------------------------ the stand-in model
class FieldModel(sugar_ref.SugarModel):
    """sugar_ref.SugarModel with SuGaR's normalising quaternions getter (SS/:426-452: F.normalize(_quaternions, dim=-1)), a
    neighbour table knn_idx [P,K] int64, knn_to_track and beta_mode, and the restated methods bound.  ``dtype`` float64 casts
    the raw leaves, which makes every getter and method float64."""

    get_covariance = get_covariance
    get_beta = get_beta
    get_field_values = get_field_values
    compute_density = compute_density
    get_gaussians_closest_to_samples = get_gaussians_closest_to_samples

    def __init__(self, g, knn_idx, beta_mode="average", dtype=torch.float32, grad=True):
        super().__init__(g, None, 64, 64, 1.0, grad=False)
        for k in list(self.leaves):
            v = self.leaves[k].detach().to(dtype).contiguous().clone().requires_grad_(grad)
            self.leaves[k] = v
            setattr(self, k, v)
        self.knn_idx = knn_idx
        self.knn_to_track = knn_idx.shape[1]
        self.beta_mode = beta_mode

    quaternions = property(lambda s: torch.nn.functional.normalize(s._quaternions, dim=-1))


class Getters:
    """A model whose getters return given tensors (leaves of the test's own choosing), for gradients with respect to the five
    inputs of the field: points, scaling, quaternions, strengths [P,1] (and x, passed to the method)."""

    get_covariance = get_covariance
    get_beta = get_beta
    get_field_values = get_field_values
    compute_density = compute_density
    get_gaussians_closest_to_samples = get_gaussians_closest_to_samples

    def __init__(self, points, scaling, quaternions, strengths, knn_idx=None, beta_mode="average"):
        self.points, self.scaling, self.quaternions, self.strengths = points, scaling, quaternions, strengths
        self.knn_idx = knn_idx
        self.knn_to_track = None if knn_idx is None else knn_idx.shape[1]
        self.beta_mode = beta_mode


# ------------------------------------------------------------------------------------------------ samples and trainer blocks
def sample_points_in_gaussians(self, num_samples, sampling_scale_factor=1.5, generator=None):
    """SS/:757-799 with mask = None and probabilities_proportional_to_volume = False (CD/:168, CS/:163); the rotation applied
    as quaternion_to_matrix(q) @ v (pytorch3d's quaternion_apply for a unit q).  The draw is detached: the samples are fixed."""
    with torch.no_grad():
        P = self.points.shape[0]
        random_indices = torch.randint(0, P, (num_samples,), generator=generator, device="cpu").to(self.points.device)
        noise = torch.randn((num_samples, 3), generator=generator, device="cpu").to(self.points.device, self.points.dtype)
    R = quaternion_to_matrix(self.quaternions[random_indices])
    v = sampling_scale_factor * self.scaling[random_indices] * noise
    random_points = self.points[random_indices] + (R @ v[..., None])[..., 0]
    return random_points, random_indices


def _projection_estimate(self, sdf_samples, sdf_gaussian_idx):
    """CD/:704-707 (use_projection_as_estimation): the signed distance along the sample's Gaussian's normal."""
    R = quaternion_to_matrix(self.quaternions)
    k = self.scaling.min(dim=-1)[1]
    normals = R[torch.arange(R.shape[0], device=R.device), :, k][sdf_gaussian_idx]
    return ((sdf_samples - self.points[sdf_gaussian_idx]) * normals).sum(dim=-1)


def density_block(self, sdf_samples, sdf_gaussian_idx, spatial_extent=1.0, sdf_estimation_factor=0.2):
    """coarse_density's block (CD/:692-742, sdf_estimation_mode 'density', density_factor 1, density_threshold 1) -> loss."""
    fields = self.get_field_values(sdf_samples, sdf_gaussian_idx, return_sdf=False, density_threshold=1., density_factor=1.,
                                   return_sdf_grad=False, sdf_grad_max_value=10., return_closest_gaussian_opacities=True,
                                   return_beta=True)
    sdf_estimation = _projection_estimate(self, sdf_samples, sdf_gaussian_idx)
    beta = fields['beta']
    densities = fields['density']
    target_densities = torch.exp(-0.5 * sdf_estimation.pow(2) / beta.pow(2))
    sdf_estimation_loss = (densities - target_densities).abs()
    # the better-normal loss reads the opacities detached (CD/:768): they weigh, but carry no gradient
    w = fields['closest_gaussian_opacities'].detach()
    return sdf_estimation_factor * sdf_estimation_loss.mean() + 1e-3 * (w.sum(-1) * densities).mean()


def sdf_block(self, sdf_samples, sdf_gaussian_idx, spatial_extent=1.0, sdf_estimation_factor=0.2):
    """coarse_sdf's block (CS/:671-713, sdf_estimation_mode 'sdf', density_factor 1/16, density_threshold 1) -> loss."""
    fields = self.get_field_values(sdf_samples, sdf_gaussian_idx, return_sdf=True, density_threshold=1., density_factor=1. / 16.,
                                   return_sdf_grad=False, sdf_grad_max_value=10., return_closest_gaussian_opacities=True,
                                   return_beta=False)
    sdf_estimation = _projection_estimate(self, sdf_samples, sdf_gaussian_idx)
    sdf_sample_std = spatial_extent / 10.
    sdf_values = fields['sdf']
    sdf_estimation_loss = (sdf_values - sdf_estimation.abs()).abs() / sdf_sample_std
    return sdf_estimation_factor * sdf_estimation_loss.clamp(max=10. * spatial_extent).mean()
