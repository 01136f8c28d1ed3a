"""SuGaR's render wrapper restated for the tests — test infrastructure.

"SS/" = sugar/sugar_scene/sugar_model.py (SuGaR.render_image_gaussian_rasterizer, SS/:1956-2228).  sugar_model.py imports
pytorch3d and open3d, so neither the model nor the method can be imported; this module states, op for op:

  * pytorch3d's ``quaternion_to_matrix``, SuGaR's ``get_smallest_axis`` / ``get_points_rgb`` and its ``eval_sh``
    (sugar/sugar_utils/spherical_harmonics.py), SuGaR's ``getWorld2View`` / ``getProjectionMatrix`` (sugar_utils/graphics_utils.py);
  * the shading normal of SS/:2164-2168 in torch (``sugar_normal_torch``) and in numpy float32, one rounding per torch op
    (``sugar_normal_np``), with its closed-form vector-Jacobian product (``sugar_normal_vjp``);
  * the method itself as a literal two-call function over a ``GaussianRasterizer`` class (``sugar_render_two_pass``);
  * a SuGaR stand-in model (raw leaves and SuGaR's getters) and a camera stand-in with the fields the method reads.
"""
from __future__ import annotations

import math
import types

import numpy as np
import torch

from tests import wrapper_ref as WR

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
      -0.5900435899266435)


# ------------------------------------------------------------------------------------------------ torch restatements
def quaternion_to_matrix(q):
    """pytorch3d.transforms.quaternion_to_matrix: q real part first, not normalised; two_s = 2 / |q|^2."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def get_smallest_axis(quaternions, scaling, return_idx=False):  # SS/:801-815
    rotation_matrices = quaternion_to_matrix(quaternions)
    idx = scaling.min(dim=-1)[1][..., None, None].expand(-1, 3, -1)
    axis = rotation_matrices.gather(2, idx).squeeze(dim=2)
    return (axis, idx[..., 0, 0]) if return_idx else axis


def sugar_normal_torch(positions, scaling, quaternions, campos):
    """normal * 0.5 + 0.5 of SS/:2164-2168."""
    render_directions = torch.nn.functional.normalize(positions - campos, dim=-1)
    normal_axis = get_smallest_axis(quaternions, scaling)
    normal_axis, _ = WR.flip_align_view(normal_axis, render_directions)
    normal = normal_axis / normal_axis.norm(dim=1, keepdim=True)
    return normal * 0.5 + 0.5


def sugar_normal_forced(quaternions, k, sign):
    """The same normal as a function of the quaternions alone, with the axis index k [P] and the flip sign [P] fixed (the
    decisions are piecewise constant; this is what autograd differentiates)."""
    axis = quaternion_to_matrix(quaternions)[torch.arange(quaternions.shape[0]), :, k] * sign[:, None]
    return axis / axis.norm(dim=1, keepdim=True) * 0.5 + 0.5


def eval_sh(deg, sh, dirs):
    """SuGaR's eval_sh (sugar_utils/spherical_harmonics.py) for degrees 0-3: sh [..., C, >= (deg+1)^2], dirs [..., 3] unit."""
    assert 0 <= deg <= 3
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
    return result


def getWorld2View(R, t):  # sugar_utils/graphics_utils.py, numpy branch
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    return np.float32(Rt)


def getProjectionMatrix(znear, zfar, fovX, fovY):  # sugar_utils/graphics_utils.py
    tanHalfFovY, tanHalfFovX = math.tan(fovY / 2), math.tan(fovX / 2)
    top = tanHalfFovY * znear
    bottom = -top
    right = tanHalfFovX * znear
    left = -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


# ------------------------------------------------------------------------------------------------ numpy float32 oracle
def sugar_normal_np(positions, scaling, quaternions, campos):
    """float32, one rounding per torch op in torch's order.  Returns (normal * 0.5 + 0.5 [P,3], axis index k [P], sign [P])."""
    f = np.float32
    q = np.asarray(quaternions, dtype=f)
    r, i, j, k = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    ss = ((r * r + i * i) + j * j) + k * k
    t = (f(1) / ss) * f(2)
    cols = np.stack([np.stack((f(1) - t * (j * j + k * k), t * (i * j + k * r), t * (i * k - j * r)), -1),
                     np.stack((t * (i * j - k * r), f(1) - t * (i * i + k * k), t * (j * k + i * r)), -1),
                     np.stack((t * (i * k + j * r), t * (j * k - i * r), f(1) - t * (i * i + j * j)), -1)], 1)  # [P, col, 3]
    s = np.asarray(scaling, dtype=f)
    kk = np.argmin(s, axis=1)  # numpy: first minimal index, as torch.min(dim) documents
    axis = cols[np.arange(q.shape[0]), kk]
    d = np.asarray(positions, dtype=f) - np.asarray(campos, dtype=f).reshape(1, 3)
    dn = np.maximum(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]), f(1e-12))
    v = d / dn[:, None]
    dot = (axis[:, 0] * -v[:, 0] + axis[:, 1] * -v[:, 1]) + axis[:, 2] * -v[:, 2]
    sign = np.where(dot >= 0, f(1), f(-1))
    a = axis * sign[:, None]
    an = np.sqrt((a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2])
    n = a / an[:, None]
    return n * f(0.5) + f(0.5), kk, sign


def sugar_normal_vjp(quaternions, k, sign, g):
    """Closed-form dL/dq (float64) of sugar_normal_forced for dL/d(normal * 0.5 + 0.5) = g: with t = 2/|q|^2 the column is
    a = base + sigma t u(q), so dL/dq = t J_u^T (sigma c) - t^2 (sigma c . u) q, c = sign (e - m (m.e)) / |a|, e = g / 2."""
    q = np.asarray(quaternions, dtype=np.float64)
    r, i, j, kq = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    t = 2.0 / (q * q).sum(1)
    # u and du/dq (rows of the Jacobian: d/dr, d/di, d/dj, d/dk) of each column, and sigma
    z = np.zeros_like(r)
    U = {0: ((j * j + kq * kq, i * j + kq * r, i * kq - j * r),
             ((z, z, 2 * j, 2 * kq), (kq, j, i, r), (-j, kq, -r, i)), (-1, 1, 1), (1, 0, 0)),
         1: ((i * j - kq * r, i * i + kq * kq, j * kq + i * r),
             ((-kq, j, i, -r), (z, 2 * i, z, 2 * kq), (i, r, kq, j)), (1, -1, 1), (0, 1, 0)),
         2: ((i * kq + j * r, j * kq - i * r, i * i + j * j),
             ((j, kq, r, i), (-i, -r, kq, j), (z, 2 * i, 2 * j, z)), (1, 1, -1), (0, 0, 1))}
    out = np.zeros_like(q)
    for col, (u, du, sigma, base) in U.items():
        sel = np.asarray(k) == col
        if not sel.any():
            continue
        a = np.stack([base[l] + sigma[l] * t * u[l] for l in range(3)], 1)[sel]
        sg = np.asarray(sign, dtype=np.float64)[sel][:, None]
        an = np.linalg.norm(a, axis=1, keepdims=True)
        m = sg * a / an
        e = 0.5 * np.asarray(g, dtype=np.float64)[sel]
        c = sg * (e - m * (m * e).sum(1, keepdims=True)) / an
        G = sum(sigma[l] * c[:, l:l + 1] * np.stack(du[l], 1)[sel] for l in range(3))
        su = sum(sigma[l] * c[:, l] * u[l][sel] for l in range(3))
        out[sel] = t[sel, None] * G - (t[sel] ** 2 * su)[:, None] * q[sel]
    return out


# ------------------------------------------------------------------------------------------------ stand-ins
class P3DCamera:
    """The fields of a pytorch3d camera the method reads: znear, zfar, K [1,3,3] (K[0,0,2], K[0,1,2] patch the projection),
    get_camera_center() [1,3]."""

    def __init__(self, center, znear, zfar, px, py, device):
        self.znear = torch.tensor([znear], device=device)
        self.zfar = torch.tensor([zfar], device=device)
        self.K = torch.zeros(1, 3, 3, device=device)
        self.K[0, 0, 2], self.K[0, 1, 2], self.K[0, 2, 2] = px, py, 1.0
        self._center = torch.as_tensor(center, dtype=torch.float32).reshape(1, 3).to(device)

    def get_camera_center(self):
        return self._center.clone()


class Cameras:
    """SuGaR's CamerasWrapper stand-in: ``camera_to_worlds`` [N,3,4] (OpenGL axes: Y up, Z back) and ``p3d_cameras[i]``."""

    def __init__(self, eyes, target=(0.0, 0.0, 0.0), znear=0.01, zfar=100.0, principal=(0.0, 0.0), device="cuda"):
        c2ws, cams = [], []
        for e in eyes:
            e = np.asarray(e, dtype=np.float64)
            f = np.asarray(target, dtype=np.float64) - e
            f /= np.linalg.norm(f)
            right = np.cross(f, (0.0, 0.0, 1.0))
            right /= np.linalg.norm(right)
            up = np.cross(right, f)
            c2ws.append(np.concatenate([np.stack([right, up, -f, e], 1)], 0))
            cams.append(P3DCamera(e, znear, zfar, principal[0], principal[1], device))
        self.camera_to_worlds = torch.tensor(np.stack(c2ws), dtype=torch.float32, device=device)
        self.p3d_cameras = cams


class SugarModel:
    """A SuGaR model's raw leaves and getters (SS/:365-430 for an unbound model): points = _points, strengths =
    sigmoid(all_densities), scaling = exp(_scales), quaternions = _quaternions (raw), sh_coordinates = cat(dc, rest)."""

    def __init__(self, g, cameras, W, H, fov_x, quat_norms=None, grad=True):
        device = g["means3D"].device
        op = g["opacities"].reshape(-1, 1).double().clamp(1e-4, 1 - 1e-4)
        q = g["rotations"] if quat_norms is None else g["rotations"] * quat_norms[:, None].to(device)
        leaves = {"_points": g["means3D"], "all_densities": torch.log(op / (1 - op)).float(), "_scales": torch.log(g["scales"]),
                  "_quaternions": q, "_sh_coordinates_dc": g["shs"][:, :1], "_sh_coordinates_rest": g["shs"][:, 1:]}
        self.leaves = {}
        for k, v in leaves.items():
            self.leaves[k] = v.detach().float().contiguous().clone().requires_grad_(grad)
            setattr(self, k, self.leaves[k])
        self.scale_activation = torch.exp
        self.image_width, self.image_height = W, H
        self.fov_x = fov_x
        self.fov_y = 2 * math.atan(math.tan(fov_x / 2) * H / W)
        self.tanfovx, self.tanfovy = math.tan(self.fov_x * 0.5), math.tan(self.fov_y * 0.5)
        self.nerfmodel = types.SimpleNamespace(training_cameras=cameras, device=device)

    device = property(lambda s: s.nerfmodel.device)
    n_points = property(lambda s: len(s._points))
    points = property(lambda s: s._points)
    strengths = property(lambda s: torch.sigmoid(s.all_densities.view(-1, 1)))
    sh_coordinates = property(lambda s: torch.cat([s._sh_coordinates_dc, s._sh_coordinates_rest], dim=1))
    scaling = property(lambda s: s.scale_activation(s._scales))
    quaternions = property(lambda s: s._quaternions)

    def get_points_rgb(self, positions=None, camera_centers=None, directions=None, sh_levels=None, sh_coordinates=None):  # SS/:711-755
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

    def grads(self):
        return {k: v.grad for k, v in self.leaves.items() if v.grad is not None}


# ------------------------------------------------------------------------------------------------ the reference method
def sugar_render_two_pass(self, nerf_cameras=None, camera_indices=0, verbose=False, bg_color=None, sh_deg=None, sh_rotations=None,
                          compute_color_in_rasterizer=False, compute_covariance_in_rasterizer=True, return_2d_radii=False,
                          quaternions=None, use_same_scale_in_all_directions=False, return_opacities=False, return_colors=False,
                          positions=None, point_colors=None, rasterizer_module=None):
    """SS/:1956-2228 as the reference writes it: two calls of ``rasterizer_module.GaussianRasterizer`` (default: this repository's
    drop-in package ``diff_gaussian_rasterization``) with the same geometry, the normals and normal maps as torch ops."""
    if rasterizer_module is None:
        import diff_gaussian_rasterization as rasterizer_module
    if nerf_cameras is None:
        nerf_cameras = self.nerfmodel.training_cameras
    p3d_camera = nerf_cameras.p3d_cameras[camera_indices]
    if bg_color is None:
        bg_color = torch.Tensor([0.0, 0.0, 0.0]).to(self.device)
    if positions is None:
        positions = self.points
    c2w = nerf_cameras.camera_to_worlds[camera_indices]
    c2w = torch.cat([c2w, torch.Tensor([[0, 0, 0, 1]]).to(self.device)], dim=0).cpu().numpy()
    c2w[:3, 1:3] *= -1
    w2c = np.linalg.inv(c2w)
    R = np.transpose(w2c[:3, :3])
    T = w2c[:3, 3]
    world_view_transform = torch.Tensor(getWorld2View(R=R, t=T)).transpose(0, 1).to(self.device)
    proj_transform = getProjectionMatrix(p3d_camera.znear.item(), p3d_camera.zfar.item(), self.fov_x, self.fov_y).transpose(0, 1).to(self.device)
    proj_transform[..., 2, 0] = - p3d_camera.K[0, 0, 2]
    proj_transform[..., 2, 1] = - p3d_camera.K[0, 1, 2]
    full_proj_transform = (world_view_transform.unsqueeze(0).bmm(proj_transform.unsqueeze(0))).squeeze(0)
    camera_center = p3d_camera.get_camera_center()
    raster_settings = rasterizer_module.GaussianRasterizationSettings(
        image_height=int(self.image_height), image_width=int(self.image_width), tanfovx=self.tanfovx, tanfovy=self.tanfovy, bg=bg_color,
        scale_modifier=1., viewmatrix=world_view_transform, projmatrix=full_proj_transform, sh_degree=sh_deg, campos=camera_center,
        prefiltered=False, debug=False)
    rasterizer = rasterizer_module.GaussianRasterizer(raster_settings=raster_settings)
    if point_colors is None:
        if not compute_color_in_rasterizer:
            if sh_rotations is None:
                splat_colors = self.get_points_rgb(positions=positions, camera_centers=camera_center, sh_levels=sh_deg + 1)
            else:
                splat_colors = self.get_points_rgb(
                    positions=positions, camera_centers=None,
                    directions=(torch.nn.functional.normalize(positions - camera_center, dim=-1).unsqueeze(1) @ sh_rotations)[..., 0, :],
                    sh_levels=sh_deg + 1)
            shs = None
        else:
            shs = self.sh_coordinates
            splat_colors = None
    else:
        splat_colors = point_colors
        shs = None
    splat_opacities = self.strengths.view(-1, 1)
    if quaternions is None:
        quaternions = self.quaternions
    if not use_same_scale_in_all_directions:
        scales = self.scaling
    else:
        scales = self.scaling.mean(dim=-1, keepdim=True).expand(-1, 3)
        scales = scales.squeeze(0)
    if not compute_covariance_in_rasterizer:
        cov3Dmatrix = torch.zeros((scales.shape[0], 3, 3), dtype=torch.float, device=self.device)
        rotation = quaternion_to_matrix(quaternions)
        cov3Dmatrix[:, 0, 0] = scales[:, 0] ** 2
        cov3Dmatrix[:, 1, 1] = scales[:, 1] ** 2
        cov3Dmatrix[:, 2, 2] = scales[:, 2] ** 2
        cov3Dmatrix = rotation @ cov3Dmatrix @ rotation.transpose(-1, -2)
        cov3D = torch.zeros((cov3Dmatrix.shape[0], 6), dtype=torch.float, device=self.device)
        cov3D[:, 0] = cov3Dmatrix[:, 0, 0]
        cov3D[:, 1] = cov3Dmatrix[:, 0, 1]
        cov3D[:, 2] = cov3Dmatrix[:, 0, 2]
        cov3D[:, 3] = cov3Dmatrix[:, 1, 1]
        cov3D[:, 4] = cov3Dmatrix[:, 1, 2]
        cov3D[:, 5] = cov3Dmatrix[:, 2, 2]
        quaternions = None
        scales = None
    else:
        cov3D = None
    screenspace_points = torch.zeros(self.n_points, 3, dtype=self._points.dtype, requires_grad=True, device=self.device)
    if return_2d_radii:
        screenspace_points.retain_grad()
    means2D = screenspace_points
    rgb_image, depth_image, alpha_image, radii = rasterizer(
        means3D=positions, means2D=means2D, shs=shs, colors_precomp=splat_colors, opacities=splat_opacities, scales=scales,
        rotations=quaternions, cov3D_precomp=cov3D)
    rendered_image = torch.cat((rgb_image, alpha_image), dim=0)
    depth_image = depth_image.squeeze(0)
    normal_normed = sugar_normal_torch(positions, self.scaling, self.quaternions, camera_center)
    image = rasterizer(means3D=positions, means2D=means2D, shs=None, colors_precomp=normal_normed, opacities=splat_opacities,
                       scales=scales, rotations=quaternions, cov3D_precomp=cov3D)[0]
    normal_image = WR.normal_image(image)
    h, w = int(self.image_height), int(self.image_width)
    fx, fy = WR.fov2focal(self.tanfovx, w), WR.fov2focal(self.tanfovy, h)
    cx, cy = w / 2, h / 2
    directions = WR.get_ray_directions(h, w, torch.FloatTensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]]), self.device)
    c2w = torch.FloatTensor(c2w).to(self.device)
    rays_d = directions @ c2w[:3, :3].T
    rays_o = c2w[:3, 3].expand_as(rays_d)
    points3D = rays_o + rays_d * depth_image.unsqueeze(-1)
    pseudo_normal = WR.depth_pcd2normal(points3D)
    if not (return_2d_radii or return_opacities or return_colors):
        return rendered_image.transpose(0, 1).transpose(1, 2)
    outputs = {"image": rendered_image.transpose(0, 1).transpose(1, 2), "depth": depth_image, "normal": normal_image,
               "pseudo_normal": pseudo_normal, "radii": radii, "viewspace_points": screenspace_points}
    if return_opacities:
        outputs["opacities"] = splat_opacities
    if return_colors:
        outputs["colors"] = splat_colors
    return outputs


def ring_cameras(n, radius=3.0, height=0.8, device="cuda", principal=(0.0, 0.0)):
    """n cameras on a circle around the origin, looking at it."""
    eyes = [(radius * math.cos(2 * math.pi * t / n), radius * math.sin(2 * math.pi * t / n), height) for t in range(n)]
    return Cameras(eyes, principal=principal, device=device)
