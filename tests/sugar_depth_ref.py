"""coarse_sdf's depth-map SDF estimate restated op for op in torch — test infrastructure.

"SS/" = sugar/sugar_scene/sugar_model.py, "CS/" = sugar/sugar_trainers/coarse_sdf.py, "SC/" = sugar/sugar_scene/cameras.py.
``get_points_depth_in_depth_map`` is SS/:1189-1204 (torch's own grid_sample), ``close_to_surface_mask`` CS/:655-666 and
``depth_sdf_estimation_loss`` CS/:689-712 with the trainers' defaults (sdf_estimation_mode 'sdf', not squared,
normalize_by_sdf_std False), before the trainer's sdf_estimation_factor.  Run in float64 they are the oracle; in float32 on the
GPU they are torch's own graph.

pytorch3d is not installed here, so ``Camera`` stands in for the FoVPerspectiveCameras that ``convert_camera_from_gs_to_pytorch3d``
(SC/:264-338) builds: R and T with the [-1, 1, -1] flips, the SfM K of ``_get_sfm_calibration_matrix`` (here with a principal-point
offset), ``get_world_to_view_transform`` = Rotate(R) then Translate(T), ``get_projection_transform`` = Transform3d(matrix=K^T), and
``transform_points`` = [p, 1] @ M divided by the last column with eps=None.  That arithmetic is restated from pytorch3d's
documented conventions; nothing here checks it against pytorch3d itself.
"""
from __future__ import annotations

import math

import torch

from tests import sugar_sample_ref as SSR


class Transform:
    """pytorch3d's Transform3d for one camera: get_matrix() [1,4,4] and transform_points (row vectors, eps=None)."""

    def __init__(self, matrix):
        self._m = matrix

    def get_matrix(self):
        return self._m

    def transform_points(self, points):
        pb = points.clone()
        if pb.dim() == 2:
            pb = pb[None]
        ones = torch.ones(pb.shape[0], pb.shape[1], 1, dtype=pb.dtype, device=pb.device)
        pb = torch.cat([pb, ones], dim=2)
        out = pb.bmm(self._m)  # _broadcast_bmm
        denom = out[..., 3:]
        out = out[..., :3] / denom
        if out.shape[0] == 1 and points.dim() == 2:
            out = out.reshape(points.shape)
        return out


class Camera:
    """One SuGaR camera (SC/:264-338) as FoVPerspectiveCameras(R, T, K, znear=0.0001) holds it."""

    def __init__(self, R, T, K, znear):
        self.R, self.T, self.K, self.znear = R, T, K, znear

    def get_world_to_view_transform(self):
        # [[R, 0], [T, 1]], built without element assignments (a Python scalar written into a CUDA tensor is a host copy)
        z, o = self.R.new_zeros(1, 3, 1), self.R.new_ones(1, 1, 1)
        return Transform(torch.cat([torch.cat([self.R, z], 2), torch.cat([self.T[:, None, :], o], 2)], 1))

    def get_projection_transform(self):
        return Transform(self.K.transpose(1, 2).contiguous())

    def get_camera_center(self):
        """pytorch3d takes row 3 of the inverted world-to-view matrix; for [[R, 0], [T, 1]] that row is -T R^T, written here
        without torch.inverse (which reads its error flag back to the host) and without a GEMM (not deterministic-flag safe)"""
        return -(self.T[:, None, :] * self.R).sum(-1)

    def to(self, dtype):
        return Camera(self.R.to(dtype), self.T.to(dtype), self.K.to(dtype), self.znear.to(dtype))


def gs_camera(eye, target, W, H, fov_x, principal=(0.0, 0.0), device="cuda", up=(0.0, 1.0, 0.0)):
    """A 3DGS camera (world-to-camera R^T, T; x right, y down, z forward) looking from eye at target, converted as SC/:264-338.
    principal = the principal point's offset from the image centre, in pixels (SuGaR's own cameras have none)."""
    eye, target, up = (torch.tensor(v, dtype=torch.float64) for v in (eye, target, up))
    f = torch.nn.functional.normalize(target - eye, dim=0)
    r = torch.nn.functional.normalize(torch.linalg.cross(f, up), dim=0)
    d = torch.linalg.cross(f, r)
    w2c_rot = torch.stack([r, d, f])  # rows: camera axes in world coordinates
    R_gs, T_gs = w2c_rot.T, -(w2c_rot @ eye)  # GS stores R = the camera-to-world rotation, T = the world-to-camera translation
    fov_y = 2 * math.atan(math.tan(fov_x / 2) * H / W)
    fx, fy = W / (2 * math.tan(fov_x / 2)), H / (2 * math.tan(fov_y / 2))
    cx, cy = W / 2. + principal[0], H / 2. + principal[1]
    w2c = torch.zeros(4, 4)
    w2c[:3, :3] = R_gs.T.float()
    w2c[:3, 3] = T_gs.float()
    w2c[3, 3] = 1
    c2w = w2c.inverse()
    c2w[:3, 1:3] *= -1
    c2w = c2w[:3, :]
    image_size = torch.tensor([[float(W), float(H)]])
    scale = image_size.min(dim=1, keepdim=True)[0] / 2.0
    c0 = image_size / 2.0
    p0 = -(torch.tensor([[cx, cy]]) - c0) / scale
    focal = torch.tensor([[fx, fy]]) / scale
    K = torch.zeros(1, 4, 4)  # _get_sfm_calibration_matrix, perspective
    K[0, 0, 0], K[0, 1, 1] = focal[0, 0], focal[0, 1]
    K[0, 0, 2], K[0, 1, 2] = p0[0, 0], p0[0, 1]
    K[0, 3, 2] = 1.0
    K[0, 2, 3] = 1.0
    cam2world = torch.cat([c2w, torch.tensor([[0.0, 0.0, 0.0, 1.0]])], dim=0)[None]
    world2cam = cam2world.inverse()
    R, T = world2cam.split([3, 1], dim=-1)
    R = R[:, :3].transpose(1, 2) * torch.tensor([-1.0, 1.0, -1])
    T = T.squeeze(2)[:, :3] * torch.tensor([-1.0, 1.0, -1])
    cam = Camera(R.to(device), T.to(device), K.to(device), torch.tensor([0.0001], device=device))
    cam.zfar = torch.tensor([100.0], device=device)
    cam.camera_to_world = c2w.to(device)  # [3,4], OpenGL axes: what SuGaR's CamerasWrapper holds for the renderer
    return cam


class Cameras:
    """SuGaR's CamerasWrapper for the renderer (autovfx_b200.renderer.sugar_camera): camera_to_worlds [N,3,4] and p3d_cameras[i],
    the latter the stand-ins above (their SfM K [1,4,4] has the principal point at K[0,0,2], K[0,1,2], where the renderer reads
    it)."""

    def __init__(self, cams):
        self.p3d_cameras = list(cams)
        self.camera_to_worlds = torch.stack([c.camera_to_world for c in cams])


class Model:
    """SuGaR's getters and image size: points, scaling, quaternions (leaves of the test's choosing), image_height, image_width."""

    def __init__(self, points, scaling, quaternions, H, W):
        self.points, self.scaling, self.quaternions = points, scaling, quaternions
        self.image_height, self.image_width = H, W


def get_points_depth_in_depth_map(self, fov_camera, depth, points_in_camera_space):  # SS/:1189-1204
    depth_view = depth.unsqueeze(0).unsqueeze(-1).permute(0, 3, 1, 2)
    pts_projections = fov_camera.get_projection_transform().transform_points(points_in_camera_space)
    factor = -1 * min(self.image_height, self.image_width)
    pts_projections[..., 0] = factor / self.image_width * pts_projections[..., 0]
    pts_projections[..., 1] = factor / self.image_height * pts_projections[..., 1]
    pts_projections = pts_projections[..., :2].view(1, -1, 1, 2)
    # align_corners=False is grid_sample's default; SuGaR leaves it unset, which only adds a warning
    return torch.nn.functional.grid_sample(input=depth_view, grid=pts_projections, mode='bilinear', padding_mode='border',
                                           align_corners=False)[0, 0, :, 0]


def surface_terms(self, fov_camera, depth, close_gaussian_threshold=2.):
    """CS/:655-666 -> (gaussians_close_to_surface, |map_z - z|, threshold * std): the two sides give the comparison's margin."""
    with torch.no_grad():
        gaussian_to_camera = torch.nn.functional.normalize(fov_camera.get_camera_center() - self.points, dim=-1)
        gaussian_centers_in_camera_space = fov_camera.get_world_to_view_transform().transform_points(self.points)
        gaussian_centers_z = gaussian_centers_in_camera_space[..., 2] + 0.
        gaussian_centers_map_z = get_points_depth_in_depth_map(self, fov_camera, depth, gaussian_centers_in_camera_space)
        gaussian_standard_deviations = (
            self.scaling * SSR.quaternion_apply(SSR.quaternion_invert(self.quaternions), gaussian_to_camera)).norm(dim=-1)
        lhs = (gaussian_centers_map_z - gaussian_centers_z).abs()
        rhs = close_gaussian_threshold * gaussian_standard_deviations
        return lhs < rhs, lhs, rhs


def close_to_surface_mask(self, fov_camera, depth, close_gaussian_threshold=2.):
    return surface_terms(self, fov_camera, depth, close_gaussian_threshold)[0]


def depth_sdf_estimation_loss(self, fov_camera, depth, sdf_samples, sdf_values, sdf_sample_std, clamp_max):  # CS/:689-712
    sdf_samples_in_camera_space = fov_camera.get_world_to_view_transform().transform_points(sdf_samples)
    sdf_samples_z = sdf_samples_in_camera_space[..., 2] + 0.
    proj_mask = sdf_samples_z > fov_camera.znear
    sdf_samples_map_z = get_points_depth_in_depth_map(self, fov_camera, depth, sdf_samples_in_camera_space[proj_mask])
    sdf_estimation = sdf_samples_map_z - sdf_samples_z[proj_mask]
    sdf_values = sdf_values[proj_mask]
    sdf_estimation_loss = (sdf_values - sdf_estimation.abs()).abs() / sdf_sample_std
    return sdf_estimation_loss.clamp(max=clamp_max).mean()
