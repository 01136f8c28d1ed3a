"""``render()`` — the per-frame wrapper around the rasterizer, mirror of the reference's
``sugar/gaussian_splatting/gaussian_renderer/__init__.py:83-218`` ("GR/"; the SuGaR variant ``sugar_scene/sugar_model.py:
1956-2228`` has the same two-pass structure).

The reference renders every camera twice with identical geometry (SH colours, then ``colors_precomp`` = per-Gaussian
normals), and surrounds the two passes with ~25 elementwise torch launches over P Gaussians and over H·W pixels
(direction normalisation, ``get_normal``, remaps, ``F.normalize``, meshgrid, ray directions, a 3x3 matmul per pixel, the
central-difference stencil).  Here, under ``torch.no_grad()`` (the frame loop of ``scene_representation.py:355-438``), one
frame is

    gsr_axis_normals -> gsr_forward_multi (ONE projection/binning/sort/blend pass, 6 colour channels) -> gsr_normal_maps

When gradients are required (training: ``train.py`` and the SuGaR trainers put ``normal`` and ``pseudo_normal`` in the loss)
the two rasterizer calls are one autograd call, ``rasterizer.rasterize_gaussians_multi``: gsr_forward_multi for both colour
sets, and gsr_backward_multi for both images' gradients in one blend backward (plain gsr_backward when the normal image gets
no gradient).  The normals fed to it still come from the model's own differentiable ``get_normal``, and the normal
normalisation and the pseudo-normal stencil are torch ops, so every parameter receives the gradient of the reference's graph
(two passes summed), up to the order of the floating-point sums.

``render_raw()`` takes the model's raw parameters instead (``_xyz``, ``_features_dc``, ``_features_rest``, ``_opacity``,
``_scaling``, ``_rotation``): gsr_activate_gaussians and gsr_axis_normals replace the activations and ``get_normal``, and one
gsr_activate_gaussians_backward launch replaces their autograd graph; the rest of the frame is render()'s.

``render_sugar()`` is SuGaR's wrapper (``sugar_scene/sugar_model.py:1956-2228``) with the same structure: gsr_sugar_normals (and
gsr_sugar_normals_backward) for SuGaR's own shading normals, one rasterizer pass for both colour sets, and a single colour pass
when the caller asks for the image alone.  ``render_sugar_raw()`` is render_sugar() with SuGaR's colours (get_points_rgb, eval_sh
up to degree 4) and opacities (strengths) computed from the model's raw SH leaves and densities by gsr_sugar_colors, and their
backward by one gsr_sugar_colors_backward launch.

Same argument names, return keys and error behaviour as the reference function.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import lib as _L
from . import rasterizer as R
from .rasterizer import GaussianRasterizationSettings, _dev_f32
from .scene import fov2focal

__all__ = ["render", "render_raw", "render_sugar", "render_sugar_raw", "sugar_normals", "quaternion_to_matrix", "axis_normals", "normal_maps", "pack_frame", "fov2focal", "TURBO_LUT_BGR"]


# ------------------------------------------------------------------------------------------ the three post kernels
def axis_normals(means3D: torch.Tensor, scales: torch.Tensor, rotations: torch.Tensor, campos: torch.Tensor, remap01: bool = False,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``GaussianModel.get_normal(dir_pp_normalized)`` (scene/gaussian_model.py:120-128) for every Gaussian: the axis of
    the smallest scale, flipped towards ``campos``, unit length; ``remap01`` additionally applies ``*0.5+0.5`` (GR/:147).
    [P,3] float32 on the device of ``means3D``.  Forward only."""
    if not means3D.is_cuda:
        raise RuntimeError("autovfx_b200.renderer: CUDA tensors required (there is no CPU path)")
    device = means3D.device
    with torch.cuda.device(device):
        m, s, r, c = (_dev_f32(t.detach(), device) for t in (means3D, scales, rotations, campos))
        P = m.shape[0]
        if s.shape != (P, 3) or r.shape != (P, 4) or c.numel() != 3:
            raise ValueError("axis_normals: expected scales [P,3], rotations [P,4], campos [3]")
        if out is None:
            out = torch.empty((P, 3), dtype=torch.float32, device=device)
        rc = _L.gsr_axis_normals(P, m.data_ptr() if P else None, s.data_ptr() if P else None, r.data_ptr() if P else None, c.data_ptr(),
                                 int(bool(remap01)), out.data_ptr() if P else None, _lib.stream_ptr(device))
        _lib.check(rc, "gsr_axis_normals")
    return out


def normal_maps(normal_img: Optional[torch.Tensor], depth: Optional[torch.Tensor], c2w: Optional[torch.Tensor], fx: float, fy: float,
                cx: float, cy: float, out: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None
                ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """(normal [H,W,3], pseudo_normal [H,W,3]) from the rendered ``normal*0.5+0.5`` image [3,H,W] and the depth map [H,W]
    (GR/:168-191).  ``c2w`` is the 4x4 the reference calls c2w (``world_view_transform.inverse()``)."""
    src = normal_img if normal_img is not None else depth
    if src is None:
        return None, None
    device = src.device
    with torch.cuda.device(device):
        out_n = out_p = None
        H, W = src.shape[-2], src.shape[-1]
        if normal_img is not None:
            normal_img = _dev_f32(normal_img, device)
            out_n = out[0] if out is not None and out[0] is not None else torch.empty((H, W, 3), dtype=torch.float32, device=device)
        if depth is not None:
            depth = _dev_f32(depth, device)
            c2w = _dev_f32(c2w, device)
            if c2w.numel() < 12:
                raise ValueError("normal_maps: c2w must hold at least 3x4 floats")
            out_p = out[1] if out is not None and out[1] is not None else torch.empty((H, W, 3), dtype=torch.float32, device=device)
        rc = _L.gsr_normal_maps(W, H, R._ptr(normal_img), R._ptr(depth), R._ptr(c2w) if depth is not None else None, fx, fy, cx, cy,
                                R._ptr(out_n), R._ptr(out_p), _lib.stream_ptr(device))
        _lib.check(rc, "gsr_normal_maps")
    return out_n, out_p


def pack_frame(rgb: Optional[torch.Tensor] = None, alpha: Optional[torch.Tensor] = None, depth: Optional[torch.Tensor] = None,
               normal_hwc: Optional[torch.Tensor] = None, depth_scale: float = 3.0, out: Optional[Dict[str, torch.Tensor]] = None
               ) -> Dict[str, torch.Tensor]:
    """8-bit images of a finished frame, exactly the bytes the reference's frame loop hands to its encoders
    (scene_representation.py:424-438): ``rgba8`` [H,W,4] (torchvision ``save_image`` rounding of cat(rgb, alpha)),
    ``normal8`` [H,W,3] (RGB order; the reference swaps to BGR only for cv2.imwrite) and ``depth8`` [H,W], the index of
    ``depth2img``'s TURBO colormap (``TURBO_LUT_BGR[depth8]`` is the image cv2.applyColorMap returns)."""
    src = rgb if rgb is not None else (depth if depth is not None else normal_hwc)
    if src is None:
        return {}
    device = src.device
    res: Dict[str, torch.Tensor] = {}
    with torch.cuda.device(device):
        if rgb is not None:
            H, W = rgb.shape[-2], rgb.shape[-1]
        elif depth is not None:
            H, W = depth.shape[-2], depth.shape[-1]
        else:
            H, W = normal_hwc.shape[0], normal_hwc.shape[1]
        rgb = _dev_f32(rgb, device) if rgb is not None else None
        alpha = _dev_f32(alpha, device) if alpha is not None else None
        depth = _dev_f32(depth, device) if depth is not None else None
        normal_hwc = _dev_f32(normal_hwc, device) if normal_hwc is not None else None

        def buf(name, shape):
            if out is not None and name in out:
                return out[name]
            return torch.empty(shape, dtype=torch.uint8, device=device)
        if rgb is not None:
            res["rgba8"] = buf("rgba8", (H, W, 4))
        if normal_hwc is not None:
            res["normal8"] = buf("normal8", (H, W, 3))
        if depth is not None:
            res["depth8"] = buf("depth8", (H, W))
        rc = _L.gsr_pack_frame(W, H, R._ptr(rgb), R._ptr(alpha), R._ptr(depth), R._ptr(normal_hwc), float(depth_scale),
                               R._ptr(res.get("rgba8")), R._ptr(res.get("normal8")), R._ptr(res.get("depth8")), _lib.stream_ptr(device))
        _lib.check(rc, "gsr_pack_frame")
    return res


# 256x3 uint8 (B,G,R): the table cv2.applyColorMap(..., cv2.COLORMAP_TURBO) applies (depth2img, sugar/render.py:18-22),
# generated by tools/make_turbo_lut.py from OpenCV 4.13 so that the hand-off does not need cv2 on the render box.
_TURBO_HEX = (
    "3b12304315324a1833511b34581e355f21366624376d2738732a39792d3a802f3b86323c8b353d91383e973b3f9c3e3fa24040a74341ac4641b14942"
    "b54b42ba4e43bf5144c35444c75644cb5945cf5c45d35e45d66146da6446dd6646e06946e36b46e66e47e97147eb7347ee7647f07847f27b47f47d46"
    "f68046f88246fa8546fb8746fc8a45fd8c45fe8f44fe9143ff9442ff9641ff9940fe9b3efe9e3dfda03bfca33afba538faa837f8ab35f7ad33f5af31"
    "f4b22ff2b42ef0b72ceeb92aebbc28e9be27e7c025e4c323e2c522dfc720ddc91fdacb1ed8cd1cd5d01bd2d21ad0d41acdd519cad718c8d918c5db18"
    "c2dd18c0de18bde018bbe219b9e319b6e41ab4e61cb2e71dafe91facea20aaeb22a7ec25a4ee27a1ef2a9ef02c9bf12f98f23294f33591f4388ef53c"
    "8af63f87f74384f84680f84a7df94e7afa5276fa5573fb596ffc5d6cfc6169fd6566fd6962fe6d5ffe715cfe7559fe7956ff7d53ff8051ff844eff88"
    "4bff8b49ff8f47ff9244fe9642fe9940fe9c3ffd9f3dfda13cfca43afca739fba938fbac37faaf36f9b136f8b435f7b735f6b934f5bc34f4be34f3c1"
    "34f1c334f0c634efc834edcb34eccd34ead035e9d235e7d435e5d736e4d936e2db37e0dd37dfdf37dde138dbe338d9e539d7e739d5e939d3eb3ad1ec"
    "3acfee3acdef3acbf13ac9f23ac7f43ac5f53ac3f63ac1f739bef839bcf939bafa38b8fb37b6fb36b3fc36b1fc35aefd34acfd33a9fe32a7fe31a4fe"
    "30a1fe2f9efe2d9bfe2c99fe2b96fe2a93fe2990fe278dfd268afd2587fc2384fc2281fb217efb1f7bfa1e78f91d75f91c72f81a6ff7196cf61869f5"
    "1766f41563f31460f2135df1125bf01158ef1055ed0f53ec0e50eb0d4eea0c4be80c49e70b47e50a45e40a43e20941e1083fdf083ddd073bdc0739da"
    "0637d80635d60533d40531d2052fd0042dce042bcc042aca0328c80326c50325c30223c10221be0220bc021eb9021db7011bb4011ab20118af0117ac"
    "0116a90114a70113a40112a101109e010f9b010e98010d95010b92010a8e02098b02088802078502068102057e03047a"
)
TURBO_LUT_BGR = torch.frombuffer(bytearray(bytes.fromhex(_TURBO_HEX)), dtype=torch.uint8).reshape(256, 3).clone()


# ------------------------------------------------------------------------------------------ SH -> RGB in Python (pipe.convert_SHs_python)
def _eval_sh_torch(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """Real spherical harmonics up to degree 3, sh [...,3,(max_deg+1)^2], dirs [...,3] unit -> [...,3]
    (same basis and sign convention as utils/sh_utils.py:57-112 and DGR/cuda_rasterizer/forward.cu:20-71)."""
    x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
    basis = [torch.full_like(x, 0.28209479177387814)]
    if deg > 0:
        c1 = 0.4886025119029199
        basis += [-c1 * y, c1 * z, -c1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        basis += [1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.31539156525252005 * (2.0 * zz - xx - yy),
                  -1.0925484305920792 * xz, 0.5462742152960396 * (xx - yy)]
        if deg > 2:
            basis += [-0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * xy * z, -0.4570457994644658 * y * (4 * zz - xx - yy),
                      0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy), -0.4570457994644658 * x * (4 * zz - xx - yy),
                      1.445305721320277 * z * (xx - yy), -0.5900435899266435 * x * (xx - 3 * yy)]
    B = torch.cat(basis, dim=-1)  # [..., n]
    return (sh[..., : B.shape[-1]] * B.unsqueeze(-2)).sum(-1)


# ------------------------------------------------------------------------------------------ render()
def _depth_pcd2normal(xyz: torch.Tensor) -> torch.Tensor:
    """Differentiable torch form of GR/:23-38 (used only when gradients are required)."""
    hd, wd, _ = xyz.shape
    l2r = xyz[1:hd - 1, 2:wd, :] - xyz[1:hd - 1, 0:wd - 2, :]
    b2t = xyz[0:hd - 2, 1:wd - 1, :] - xyz[2:hd, 1:wd - 1, :]
    n = torch.nn.functional.normalize(torch.cross(l2r, b2t, dim=-1), p=2, dim=-1)
    return torch.nn.functional.pad(n.permute(2, 0, 1), (1, 1, 1, 1), mode="constant").permute(1, 2, 0)


def _setup(viewpoint_camera, xyz, sh_degree, pipe, bg_color, scaling_modifier):
    # zero tensor whose gradient is the screen-space positional gradient (densification statistics, GR/:90-95)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:  # noqa: BLE001
        pass

    tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
    tanfovy = math.tan(viewpoint_camera.FoVy * 0.5)
    H, W = int(viewpoint_camera.image_height), int(viewpoint_camera.image_width)
    raster_settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=tanfovx, tanfovy=tanfovy, bg=bg_color, scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform, projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=sh_degree, campos=viewpoint_camera.camera_center, prefiltered=False, debug=pipe.debug)
    return screenspace_points, raster_settings


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0, override_color=None):
    """Render the scene.  Background tensor (bg_color) must be on GPU!  (GR/:83-218)

    viewpoint_camera: FoVx, FoVy, image_height, image_width, world_view_transform, full_proj_transform, camera_center.
    pc: get_xyz, get_opacity, get_scaling, get_rotation, get_features, active_sh_degree, max_sh_degree,
        get_covariance(scaling_modifier), get_normal(dir_pp_normalized=...).
    pipe: debug, compute_cov3D_python, convert_SHs_python.
    Returns {"render" [4,H,W] (rgb|alpha), "depth" [H,W], "normal" [H,W,3], "pseudo_normal" [H,W,3], "viewspace_points",
    "visibility_filter", "radii"}."""
    xyz = pc.get_xyz
    device = xyz.device
    opacity, scaling, rotation, features = pc.get_opacity, pc.get_scaling, pc.get_rotation, pc.get_features
    grad_mode = R._needs_backward(xyz, opacity, scaling, rotation, features, override_color)
    screenspace_points, raster_settings = _setup(viewpoint_camera, xyz, pc.active_sh_degree, pipe, bg_color, scaling_modifier)

    scales = rotations = cov3D_precomp = None
    if pipe.compute_cov3D_python:
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales, rotations = scaling, rotation

    shs = colors_precomp = None
    dir_pp_normalized = None
    if override_color is None:
        if pipe.convert_SHs_python:
            dir_pp = xyz - viewpoint_camera.camera_center.repeat(features.shape[0], 1)
            dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
            shs_view = features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
            colors_precomp = torch.clamp_min(_eval_sh_torch(pc.active_sh_degree, shs_view, dir_pp_normalized) + 0.5, 0.0)
        else:
            shs = features
    else:
        colors_precomp = override_color

    if not grad_mode:
        with torch.no_grad(), torch.cuda.device(device):
            normal_normed = axis_normals(xyz, scaling, rotation, viewpoint_camera.camera_center, remap01=True)
    else:
        if dir_pp_normalized is None:
            dir_pp = xyz - viewpoint_camera.camera_center.repeat(features.shape[0], 1)
            dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
        normal_normed = pc.get_normal(dir_pp_normalized=dir_pp_normalized) * 0.5 + 0.5
    return _render_outputs(viewpoint_camera, raster_settings, screenspace_points, grad_mode, xyz, shs, colors_precomp, normal_normed,
                           opacity, scales, rotations, cov3D_precomp)


def _render_outputs(viewpoint_camera, raster_settings, screenspace_points, grad_mode, *inputs):
    """_frame() with render()'s camera (GR/:168-191) and return keys; shared by render() and render_raw()."""
    H, W = int(viewpoint_camera.image_height), int(viewpoint_camera.image_width)
    w2c = viewpoint_camera.world_view_transform
    c2w = w2c.inverse if grad_mode else (lambda: torch.linalg.inv_ex(w2c.float())[0])  # GR/:185; inv_ex: no error-check sync
    image, depth, normal, pseudo_normal, radii = _frame(raster_settings, screenspace_points, grad_mode, *inputs, c2w,
                                                        fov2focal(viewpoint_camera.FoVx, W), fov2focal(viewpoint_camera.FoVy, H))
    return {"render": image, "depth": depth, "normal": normal, "pseudo_normal": pseudo_normal, "viewspace_points": screenspace_points,
            "visibility_filter": radii > 0, "radii": radii}


def _frame(raster_settings, screenspace_points, grad_mode, means3D, shs, colors_precomp, normal_normed, opacity, scales, rotations,
           cov3D_precomp, c2w, fx, fy):
    """The rasterizer call and the normal maps of every wrapper, from the tensors the rasterizer takes, the per-Gaussian normals
    remapped to [0,1] and the pseudo normal's camera: ``c2w()`` returns the 4x4 it unprojects with (called after the rasterizer,
    where the reference computes it), ``fx`` / ``fy`` are the focal lengths.  Returns (rgb|alpha [4,H,W], depth [H,W],
    normal [H,W,3], pseudo_normal [H,W,3], radii)."""
    device = means3D.device
    H, W = int(raster_settings.image_height), int(raster_settings.image_width)
    cx, cy = W / 2, H / 2

    if not grad_mode:
        # ---- one pass: 6-channel forward -> normal maps
        with torch.no_grad(), torch.cuda.device(device):
            frame = torch.empty((5, H, W), dtype=torch.float32, device=device)  # rgb | alpha | depth: "render" = frame[0:4] without a cat
            radii = torch.empty((means3D.shape[0],), dtype=torch.int32, device=device)
            _c, _d, _a, normal_img, radii, _ticket = R.forward_multi(
                means3D, shs, colors_precomp, normal_normed, opacity, scales, rotations, cov3D_precomp, raster_settings,
                out=(frame[0:3], frame[4:5], frame[3:4], radii))
            normal_image, pseudo_normal = normal_maps(normal_img, frame[4], c2w(), fx, fy, cx, cy)
        return frame[0:4], frame[4], normal_image, pseudo_normal, radii

    # ---- gradients required: one differentiable call renders both colour sets (SH colours and normals) on one projection /
    # binning / sort / blend, and its backward takes both images' gradients in one pass; the rest is the reference's graph
    rendered_image, depth_image, alpha_image, normal_image, radii = R.rasterize_gaussians_multi(
        means3D, screenspace_points, shs, colors_precomp, normal_normed, opacity, scales, rotations, cov3D_precomp, raster_settings)
    rendered_image = torch.cat((rendered_image, alpha_image), dim=0)
    depth_image = depth_image.squeeze(0)
    normal_image, pseudo_normal = _normal_maps_torch(normal_image, depth_image, c2w(), fx, fy, cx, cy)
    return rendered_image, depth_image, normal_image, pseudo_normal, radii


def _normal_maps_torch(normal_image, depth_image, c2w, fx, fy, cx, cy):
    """Differentiable torch form of normal_maps() (GR/:168-191): the rendered normal*0.5+0.5 image [3,H,W] and the depth map
    [H,W] -> (normal [H,W,3], pseudo_normal [H,W,3]), with ``c2w`` the 4x4 the wrapper unprojects with."""
    device = depth_image.device
    H, W = depth_image.shape
    normal_image = (normal_image - 0.5) * 2.
    normal_image = torch.nn.functional.normalize(normal_image.permute(1, 2, 0), p=2, dim=-1)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=device), torch.arange(W, dtype=torch.float32, device=device), indexing="ij")
    K = torch.tensor([fx, fy, cx, cy], dtype=torch.float32)
    directions = torch.stack([(xs - K[2] + 0.5) / K[0], (ys - K[3] + 0.5) / K[1], torch.ones_like(xs)], -1)
    rays_d = directions @ c2w[:3, :3].T
    rays_o = c2w[:3, 3].expand_as(rays_d)
    points3D = rays_o + rays_d * depth_image.unsqueeze(-1)
    return normal_image, _depth_pcd2normal(points3D)


# ------------------------------------------------------------------------------------------ render_raw()
_RAW_FIELDS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


def _raw_params(pc, pipe) -> Tuple[torch.Tensor, ...]:
    """pc's raw parameters (_xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation), checked."""
    missing = [f for f in _RAW_FIELDS if not isinstance(getattr(pc, f, None), torch.Tensor)]
    if missing:
        raise ValueError("render_raw: the model has no raw parameter tensor %s" % ", ".join(missing))
    for attr, fn, name in (("scaling_activation", torch.exp, "torch.exp"), ("opacity_activation", torch.sigmoid, "torch.sigmoid"),
                           ("rotation_activation", torch.nn.functional.normalize, "torch.nn.functional.normalize")):
        if getattr(pc, attr, None) is not fn:
            raise ValueError("render_raw: pc.%s must be %s, the activation this path differentiates" % (attr, name))
    for flag in ("compute_cov3D_python", "convert_SHs_python"):
        if getattr(pipe, flag, False):
            raise ValueError("render_raw: pipe.%s selects the torch arithmetic render_raw replaces; use render()" % flag)
    xyz, f_dc, f_rest, opacity, scaling, rotation = (getattr(pc, f) for f in _RAW_FIELDS)
    P = xyz.shape[0]
    want = {"_xyz": (P, 3), "_features_dc": (P, 1, 3), "_opacity": (P, 1), "_scaling": (P, 3), "_rotation": (P, 4)}
    for f, t in zip(_RAW_FIELDS, (xyz, f_dc, f_rest, opacity, scaling, rotation)):
        if t.device != xyz.device or t.dtype != torch.float32:
            raise ValueError("render_raw: pc.%s must be float32 on %s" % (f, xyz.device))
        if f in want and tuple(t.shape) != want[f]:
            raise ValueError("render_raw: pc.%s has shape %s, expected %s" % (f, tuple(t.shape), want[f]))
    if f_rest.dim() != 3 or f_rest.shape[0] != P or f_rest.shape[2] != 3:
        raise ValueError("render_raw: pc._features_rest has shape %s, expected [%d, M-1, 3]" % (tuple(f_rest.shape), P))
    if not xyz.is_cuda:
        raise RuntimeError("autovfx_b200.renderer: CUDA tensors required (there is no CPU path)")
    return xyz, f_dc, f_rest, opacity, scaling, rotation


class _ActivateRaw(torch.autograd.Function):
    """Raw parameters -> (shs, opacities, scales, rotations, normals * 0.5 + 0.5): gsr_activate_gaussians, then gsr_axis_normals
    on its output.  The backward is one gsr_activate_gaussians_backward launch.  _xyz and campos get no gradient here: the
    axis and its flip are piecewise constant, so the rasterizer's dL/dmeans3D is _xyz's whole gradient."""

    @staticmethod
    def forward(ctx, xyz, f_dc, f_rest, opacity, scaling, rotation, campos):
        device = xyz.device
        P, M = xyz.shape[0], f_rest.shape[1] + 1
        xyz, f_dc, f_rest, opacity, scaling, rotation = (t.detach().contiguous() for t in (xyz, f_dc, f_rest, opacity, scaling, rotation))
        campos = _dev_f32(campos.detach(), device)
        f = dict(dtype=torch.float32, device=device)
        shs, opacities, scales, rotations = torch.empty((P, M, 3), **f), torch.empty((P, 1), **f), torch.empty((P, 3), **f), torch.empty((P, 4), **f)
        normals = torch.empty((P, 3), **f)
        means = torch.empty((P, 3), **f)  # the kernel's copy of the positions; the rasterizer reads _xyz itself
        p = R._ptr
        with torch.cuda.device(device):
            st = _lib.stream_ptr(device)
            _lib.check(_L.gsr_activate_gaussians(P, M, p(xyz), p(f_dc), p(f_rest), p(opacity), p(scaling), p(rotation), None, p(means),
                                                 p(shs), p(opacities), p(scales), p(rotations), st), "gsr_activate_gaussians")
            _lib.check(_L.gsr_axis_normals(P, p(xyz), p(scales), p(rotations), campos.data_ptr(), 1, p(normals), st), "gsr_axis_normals")
        ctx.save_for_backward(opacities, scales, rotations, rotation, xyz, campos)
        ctx.M = M
        ctx.set_materialize_grads(False)  # no SH gradient (override_color) / no normal-image gradient arrive as None
        return shs, opacities, scales, rotations, normals

    @staticmethod
    def backward(ctx, g_shs, g_opacities, g_scales, g_rotations, g_normals):
        opacities, scales, rotations, rotation, xyz, campos = ctx.saved_tensors
        device, P, M = xyz.device, xyz.shape[0], ctx.M
        f = dict(dtype=torch.float32, device=device)

        def grad_in(g, like):
            return torch.zeros_like(like) if g is None else _dev_f32(g, device)
        g_opacities, g_scales, g_rotations = grad_in(g_opacities, opacities), grad_in(g_scales, scales), grad_in(g_rotations, rotations)
        g_shs = None if g_shs is None else _dev_f32(g_shs, device)
        g_normals = None if g_normals is None else _dev_f32(g_normals, device)
        d_op, d_sc, d_rot = torch.empty((P, 1), **f), torch.empty((P, 3), **f), torch.empty((P, 4), **f)
        d_dc = d_rest = None
        if g_shs is not None:
            d_dc, d_rest = torch.empty((P, 1, 3), **f), torch.empty((P, M - 1, 3), **f)
        p = R._ptr
        with torch.cuda.device(device):
            rc = _L.gsr_activate_gaussians_backward(P, M, p(xyz), campos.data_ptr(), p(opacities), p(scales), p(rotations), p(rotation),
                                                    p(g_opacities), p(g_scales), p(g_rotations), p(g_shs), p(g_normals), p(d_op), p(d_sc),
                                                    p(d_rot), p(d_dc), p(d_rest), _lib.stream_ptr(device))
            _lib.check(rc, "gsr_activate_gaussians_backward")
        return None, d_dc, d_rest, d_op, d_sc, d_rot, None


def render_raw(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0, override_color=None):
    """render() from the model's RAW parameters, differentiable with respect to them: ``pc._xyz [P,3]``, ``_features_dc [P,1,3]``,
    ``_features_rest [P,M-1,3]`` (M = 1 allowed), ``_opacity [P,1]``, ``_scaling [P,3]`` (log) and ``_rotation [P,4]``.

    Same arguments, return keys and shapes as render().  The activations (exp, F.normalize, sigmoid, cat) and the shading
    normals of ``get_normal`` are one gsr_activate_gaussians and one gsr_axis_normals launch, and their backward is one
    gsr_activate_gaussians_backward launch, instead of the model's torch ops and their autograd graph.  The arithmetic is the
    library's (``edit.activate``, ``axis_normals``), not the model's own torch calls, so the model must use the reference's
    activations (``scaling_activation = torch.exp``, ``opacity_activation = torch.sigmoid``, ``rotation_activation =
    F.normalize``) and ``pipe`` must not select ``compute_cov3D_python`` or ``convert_SHs_python``; otherwise ValueError.
    With ``override_color`` the SH coefficients get no gradient."""
    xyz, f_dc, f_rest, opacity_raw, scaling_raw, rotation_raw = _raw_params(pc, pipe)
    grad_mode = R._needs_backward(xyz, f_dc, f_rest, opacity_raw, scaling_raw, rotation_raw, override_color)
    screenspace_points, raster_settings = _setup(viewpoint_camera, xyz, pc.active_sh_degree, pipe, bg_color, scaling_modifier)
    with torch.set_grad_enabled(grad_mode):
        shs, opacity, scales, rotations, normal_normed = _ActivateRaw.apply(xyz, f_dc, f_rest, opacity_raw, scaling_raw, rotation_raw,
                                                                            viewpoint_camera.camera_center)
    if override_color is not None:
        shs = None
    return _render_outputs(viewpoint_camera, raster_settings, screenspace_points, grad_mode, xyz, shs, override_color, normal_normed,
                           opacity, scales, rotations, None)


# ------------------------------------------------------------------------------------------ render_sugar()
# "SS/" = sugar/sugar_scene/sugar_model.py (SuGaR.render_image_gaussian_rasterizer, SS/:1956-2228)
def quaternion_to_matrix(quaternions: torch.Tensor) -> torch.Tensor:
    """pytorch3d.transforms.quaternion_to_matrix, op for op: rotation matrices [...,3,3] of quaternions (real part first) that
    are NOT normalised first; the scale enters as two_s = 2 / |q|^2.  gsr_sugar_normals evaluates the same formula."""
    r, i, j, k = torch.unbind(quaternions, -1)
    two_s = 2.0 / (quaternions * quaternions).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(quaternions.shape[:-1] + (3, 3))


def sugar_normals(positions: torch.Tensor, scales: torch.Tensor, quaternions: torch.Tensor, campos: torch.Tensor,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """SuGaR's per-Gaussian shading normal remapped to [0,1] (SS/:2164-2168): the column of quaternion_to_matrix(quaternions)
    that belongs to ``scales.min(dim=-1)[1]``, flipped to face ``campos``, divided by its norm, ``* 0.5 + 0.5``.  [P,3] float32.
    Forward only; one gsr_sugar_normals launch."""
    if not positions.is_cuda:
        raise RuntimeError("autovfx_b200.renderer: CUDA tensors required (there is no CPU path)")
    device = positions.device
    with torch.cuda.device(device):
        m, s, q, c = (_dev_f32(t.detach(), device) for t in (positions, scales, quaternions, campos))
        P = m.shape[0]
        if m.shape != (P, 3) or s.shape != (P, 3) or q.shape != (P, 4) or c.numel() != 3:
            raise ValueError("sugar_normals: expected positions [P,3], scales [P,3], quaternions [P,4], campos [3]")
        if out is None:
            out = torch.empty((P, 3), dtype=torch.float32, device=device)
        _lib.check(_L.gsr_sugar_normals(P, R._ptr(m), R._ptr(s), R._ptr(q), c.data_ptr(), R._ptr(out), _lib.stream_ptr(device)),
                   "gsr_sugar_normals")
    return out


class _SugarNormals(torch.autograd.Function):
    """(positions, scales, quaternions, campos) -> sugar_normals(...), differentiable with respect to the quaternions: the backward is
    one gsr_sugar_normals_backward launch.  Positions, scales and campos get no gradient: the axis (an argmin over the scales) and
    the flip (a sign test on the view direction) are piecewise constant, and the reference's graph carries none through them."""

    @staticmethod
    def forward(ctx, positions, scales, quaternions, campos):
        device = positions.device
        m, s, q, c = (_dev_f32(t.detach(), device) for t in (positions, scales, quaternions, campos))
        out = sugar_normals(m, s, q, c)
        ctx.save_for_backward(m, s, q, c)
        return out

    @staticmethod
    def backward(ctx, g_normals):
        m, s, q, c = ctx.saved_tensors
        device, P = m.device, m.shape[0]
        d_q = torch.empty((P, 4), dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            g = _dev_f32(g_normals, device)
            rc = _L.gsr_sugar_normals_backward(P, R._ptr(m), R._ptr(s), R._ptr(q), c.data_ptr(), R._ptr(g), R._ptr(d_q),
                                               _lib.stream_ptr(device))
            _lib.check(rc, "gsr_sugar_normals_backward")
        return None, None, d_q, None


def _sugar_projection(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    """SuGaR's getProjectionMatrix (sugar/sugar_utils/graphics_utils.py): the 4x4 perspective matrix (row-major, z in [0, 1]),
    evaluated in Python floats and stored as float32, as the reference does."""
    top = math.tan(fovy / 2) * znear
    right = math.tan(fovx / 2) * znear
    bottom, left = -top, -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def sugar_camera(nerf_cameras, camera_indices, fov_x: float, fov_y: float, device):
    """The camera of SS/:2008-2035 -> (world_view_transform, full_proj_transform, camera_center [1,3], c2w [4,4] float32 numpy).
    c2w is the camera-to-world with the OpenGL -> COLMAP axis flip; the world-to-view matrix is np.linalg.inv of it in float32
    (getWorld2View: R^T = w2c[:3,:3], t = w2c[:3,3]); the projection is SuGaR's getProjectionMatrix with the principal point of
    K written into its third row; the product is the reference's bmm on the device."""
    import numpy as np
    p3d_camera = nerf_cameras.p3d_cameras[camera_indices]
    c2w = nerf_cameras.camera_to_worlds[camera_indices]
    c2w = torch.cat([c2w, torch.Tensor([[0, 0, 0, 1]]).to(device)], dim=0).cpu().numpy()
    c2w[:3, 1:3] *= -1
    w2c = np.linalg.inv(c2w)
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = w2c[:3, :3]  # getWorld2View(R = w2c[:3,:3]^T, t): Rt[:3,:3] = R^T
    Rt[:3, 3] = w2c[:3, 3]
    Rt[3, 3] = 1.0
    world_view_transform = torch.Tensor(np.float32(Rt)).transpose(0, 1).to(device)
    proj_transform = _sugar_projection(p3d_camera.znear.item(), p3d_camera.zfar.item(), fov_x, fov_y).transpose(0, 1).to(device)
    proj_transform[..., 2, 0] = - p3d_camera.K[0, 0, 2]
    proj_transform[..., 2, 1] = - p3d_camera.K[0, 1, 2]
    full_proj_transform = (world_view_transform.unsqueeze(0).bmm(proj_transform.unsqueeze(0))).squeeze(0)
    return world_view_transform, full_proj_transform, p3d_camera.get_camera_center(), c2w


def render_sugar(self, nerf_cameras=None, camera_indices=0, verbose=False, bg_color=None, sh_deg=None, sh_rotations=None,
                 compute_color_in_rasterizer=False, compute_covariance_in_rasterizer=True, return_2d_radii=False, quaternions=None,
                 use_same_scale_in_all_directions=False, return_opacities=False, return_colors=False, positions=None, point_colors=None):
    """SuGaR.render_image_gaussian_rasterizer (SS/:1956-2228) with the reference method's signature, arguments and return
    values; a SuGaR model opts in with ``SuGaR.render_image_gaussian_rasterizer = render_sugar``.

    ``self`` is the SuGaR model; only what the reference reads is read: points, strengths, scaling, quaternions,
    sh_coordinates, get_points_rgb, n_points, _points.dtype, device, image_height / image_width, fov_x / fov_y, tanfovx / tanfovy,
    nerfmodel.training_cameras.  The camera needs camera_to_worlds and p3d_cameras[i] with znear, zfar, K, get_camera_center().

    The reference renders twice with the same geometry (the colours, then the shading normals as colors_precomp) and computes the
    normals with ~15 torch ops.  Here:
      * without a ``return_*`` flag the reference returns the image alone and discards the normals: one rasterizer pass;
      * otherwise, without gradients: gsr_sugar_normals -> gsr_forward_multi (one pass, both colour sets) -> gsr_normal_maps;
      * otherwise, with gradients: the same normals differentiated by gsr_sugar_normals_backward, and rasterize_gaussians_multi
        (one forward, one backward for both images); the normal maps are torch ops, as in render().
    The normals come from the model's own ``quaternions`` and ``scaling``, whatever ``quaternions=`` or
    ``use_same_scale_in_all_directions`` hands the rasterizer, and face the camera from ``positions``, as in the reference.  So
    does the reference's pseudo normal: the flipped c2w and ``fx = fov2focal(self.tanfovx, w)`` (a tangent where a field of view is
    expected)."""
    return _render_sugar(self, None, nerf_cameras, camera_indices, verbose, bg_color, sh_deg, sh_rotations, compute_color_in_rasterizer,
                         compute_covariance_in_rasterizer, return_2d_radii, quaternions, use_same_scale_in_all_directions, return_opacities,
                         return_colors, positions, point_colors)


def _render_sugar(self, raw, nerf_cameras, camera_indices, verbose, bg_color, sh_deg, sh_rotations, compute_color_in_rasterizer,
                  compute_covariance_in_rasterizer, return_2d_radii, quaternions, use_same_scale_in_all_directions, return_opacities,
                  return_colors, positions, point_colors):
    """render_sugar()'s body.  ``raw`` None: the colours and opacities come from the model's get_points_rgb / strengths; otherwise
    it is the checked (sh_dc, sh_rest, densities) of render_sugar_raw() and they come from _SugarColors."""
    if nerf_cameras is None:
        nerf_cameras = self.nerfmodel.training_cameras
    device = self.device
    if bg_color is None:
        bg_color = torch.Tensor([0.0, 0.0, 0.0]).to(device)
    if positions is None:
        positions = self.points

    world_view_transform, full_proj_transform, camera_center, c2w = sugar_camera(nerf_cameras, camera_indices, self.fov_x, self.fov_y,
                                                                               device)
    if verbose:
        print("p3d camera_center", camera_center)
        print("ns camera_center", nerf_cameras.camera_to_worlds[camera_indices][..., 3])
    H, W = int(self.image_height), int(self.image_width)
    raster_settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=self.tanfovx, tanfovy=self.tanfovy, bg=bg_color, scale_modifier=1.,
        viewmatrix=world_view_transform, projmatrix=full_proj_transform, sh_degree=sh_deg, campos=camera_center, prefiltered=False,
        debug=False)

    if raw is not None:
        shs, splat_colors, splat_opacities = _sugar_raw_colors(self, raw, positions, camera_center, sh_deg, sh_rotations,
                                                               compute_color_in_rasterizer, point_colors)
    else:
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
    if verbose:
        print("Scales:", scales.shape, scales.min(), scales.max())

    if not compute_covariance_in_rasterizer:  # SS/:2093-2112
        cov3Dmatrix = torch.zeros((scales.shape[0], 3, 3), dtype=torch.float, device=device)
        rotation = quaternion_to_matrix(quaternions)
        cov3Dmatrix[:, 0, 0] = scales[:, 0] ** 2
        cov3Dmatrix[:, 1, 1] = scales[:, 1] ** 2
        cov3Dmatrix[:, 2, 2] = scales[:, 2] ** 2
        cov3Dmatrix = rotation @ cov3Dmatrix @ rotation.transpose(-1, -2)
        cov3D = torch.zeros((cov3Dmatrix.shape[0], 6), dtype=torch.float, device=device)
        for c, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
            cov3D[:, c] = cov3Dmatrix[:, a, b]
        quaternions = None
        scales = None
    else:
        cov3D = None

    # a fresh zero leaf whose gradient is the screen-space positional gradient (SS/:2117-2126)
    screenspace_points = torch.zeros(self.n_points, 3, dtype=self._points.dtype, requires_grad=True, device=device)
    if return_2d_radii:
        try:
            screenspace_points.retain_grad()
        except Exception:  # noqa: BLE001
            print("WARNING: return_2d_radii is True, but failed to retain grad of screenspace_points!")
    if verbose:
        print("points", positions.shape)
        if not compute_color_in_rasterizer:
            print("splat_colors", splat_colors.shape)
        print("splat_opacities", splat_opacities.shape)
        if not compute_covariance_in_rasterizer:
            print("cov3D", cov3D.shape)
            print(cov3D[0])
        else:
            print("quaternions", quaternions.shape)
            print("scales", scales.shape)
        print("screenspace_points", screenspace_points.shape)

    if not (return_2d_radii or return_opacities or return_colors):
        # the reference returns the image alone: its normal pass, normals and normal maps are not observable
        rgb_image, _depth, alpha_image, _radii = R.GaussianRasterizer(raster_settings=raster_settings)(
            means3D=positions, means2D=screenspace_points, shs=shs, colors_precomp=splat_colors, opacities=splat_opacities,
            scales=scales, rotations=quaternions, cov3D_precomp=cov3D)
        return torch.cat((rgb_image, alpha_image), dim=0).transpose(0, 1).transpose(1, 2)

    # the screen-space leaf requires grad, so the reference records a graph whenever grad mode is on
    grad_mode = torch.is_grad_enabled()
    normal_normed = (_SugarNormals.apply if grad_mode else sugar_normals)(positions, self.scaling, self.quaternions, camera_center)
    rendered_image, depth_image, normal_image, pseudo_normal, radii = _frame(
        raster_settings, screenspace_points, grad_mode, positions, shs, splat_colors, normal_normed, splat_opacities, scales, quaternions,
        cov3D, lambda: torch.from_numpy(c2w).to(device, torch.float32),
        fov2focal(self.tanfovx, W), fov2focal(self.tanfovy, H))  # SS/:2196-2197, reproduced as written
    outputs = {"image": rendered_image.transpose(0, 1).transpose(1, 2), "depth": depth_image, "normal": normal_image,
               "pseudo_normal": pseudo_normal, "radii": radii, "viewspace_points": screenspace_points}
    if return_opacities:
        outputs["opacities"] = splat_opacities
    if return_colors:
        outputs["colors"] = splat_colors
    return outputs


# ------------------------------------------------------------------------------------------ render_sugar_raw()
_SUGAR_RAW_FIELDS = ("_sh_coordinates_dc", "_sh_coordinates_rest", "all_densities")


def _sugar_raw_leaves(self, sh_deg, with_colors: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The SuGaR model's raw SH leaves and densities (_sh_coordinates_dc [P,1,3], _sh_coordinates_rest [P,M-1,3], all_densities
    with P elements), checked, and with ``with_colors`` the degree eval_sh will be called with."""
    dev = torch.device(self.device)
    leaves = []
    for f in _SUGAR_RAW_FIELDS:
        t = getattr(self, f, None)
        if not isinstance(t, torch.Tensor):
            raise ValueError("render_sugar_raw: the model has no tensor %s" % f)
        if t.dtype != torch.float32:
            raise ValueError("render_sugar_raw: self.%s must be float32, not %s" % (f, t.dtype))
        if t.device.type != dev.type or (dev.index is not None and t.device.index != dev.index):
            raise ValueError("render_sugar_raw: self.%s is on %s, the model on %s" % (f, t.device, dev))
        leaves.append(t)
    sh_dc, sh_rest, dens = leaves
    P = sh_dc.shape[0]
    if tuple(sh_dc.shape) != (P, 1, 3):
        raise ValueError("render_sugar_raw: self._sh_coordinates_dc has shape %s, expected [P, 1, 3]" % (tuple(sh_dc.shape),))
    if sh_rest.dim() != 3 or sh_rest.shape[0] != P or sh_rest.shape[2] != 3:
        raise ValueError("render_sugar_raw: self._sh_coordinates_rest has shape %s, expected [%d, M-1, 3]" % (tuple(sh_rest.shape), P))
    if dens.numel() != P:
        raise ValueError("render_sugar_raw: self.all_densities has %d elements, expected %d" % (dens.numel(), P))
    if getattr(self, "return_one_densities", False):
        raise ValueError("render_sugar_raw: self.return_one_densities is set; its strengths are ones, not the sigmoid this path "
                         "differentiates; use render_sugar")
    if with_colors:  # the asserts of SuGaR's eval_sh
        M = sh_rest.shape[1] + 1
        if isinstance(sh_deg, bool) or not isinstance(sh_deg, int) or not 0 <= sh_deg <= 4:
            raise ValueError("render_sugar_raw: sh_deg must be an integer in 0..4 (SuGaR's eval_sh), got %r" % (sh_deg,))
        if (sh_deg + 1) ** 2 > M:
            raise ValueError("render_sugar_raw: sh_deg %d needs %d SH coefficients per channel, the model stores M = %d"
                             % (sh_deg, (sh_deg + 1) ** 2, M))
    if not sh_dc.is_cuda:
        raise RuntimeError("autovfx_b200.renderer: CUDA tensors required (there is no CPU path)")
    return sh_dc, sh_rest, dens


class _SugarColors(torch.autograd.Function):
    """(src, campos, sh_dc, sh_rest, densities, deg, directions_mode) -> (colors [P,3], opacities [P,1]) of SuGaR's get_points_rgb and
    strengths: one gsr_sugar_colors launch, and one gsr_sugar_colors_backward launch for the backward.  src is the positions
    (camera-centre mode, with campos) or the view directions (directions_mode).  src = None gives the opacities alone; then the SH
    leaves are not read and get no gradient."""

    @staticmethod
    def forward(ctx, src, campos, sh_dc, sh_rest, densities, deg, directions_mode):
        device = densities.device
        P, M = sh_dc.shape[0], sh_rest.shape[1] + 1
        f = dict(dtype=torch.float32, device=device)
        dens = densities.detach().contiguous()
        opac = torch.empty((P, 1), **f)
        ctx.with_colors, ctx.deg, ctx.M, ctx.directions_mode = src is not None, int(deg), M, bool(directions_mode)
        ctx.set_materialize_grads(False)
        p = R._ptr
        if src is None:
            with torch.cuda.device(device):
                _lib.check(_L.gsr_sugar_colors(P, M, 0, None, None, None, None, None, p(dens), None, p(opac), _lib.stream_ptr(device)),
                           "gsr_sugar_colors")
            ctx.save_for_backward(dens)
            return opac
        src_ = _dev_f32(src.detach(), device)
        if tuple(src_.shape) != (P, 3):
            raise ValueError("render_sugar_raw: %s has shape %s, expected [%d, 3]" % ("directions" if directions_mode else "positions",
                                                                                   tuple(src_.shape), P))
        c = None if directions_mode else _dev_f32(campos.detach(), device).reshape(-1)
        dc, rest = sh_dc.detach().contiguous(), sh_rest.detach().contiguous()
        colors = torch.empty((P, 3), **f)
        with torch.cuda.device(device):
            pos, dirs = (None, p(src_)) if directions_mode else (p(src_), None)
            _lib.check(_L.gsr_sugar_colors(P, M, ctx.deg, pos, None if c is None else c.data_ptr(), dirs, p(dc), p(rest), p(dens), p(colors),
                                           p(opac), _lib.stream_ptr(device)), "gsr_sugar_colors")
        ctx.save_for_backward(dens, src_, dc, rest, *(() if c is None else (c,)))
        return colors, opac

    @staticmethod
    def backward(ctx, *grads):
        device = ctx.saved_tensors[0].device
        p = R._ptr
        if not ctx.with_colors:
            (dens,), (g_op,) = ctx.saved_tensors, grads
            if g_op is None:
                return None, None, None, None, None, None, None
            g_op = _dev_f32(g_op, device)
            d_dens = torch.empty_like(dens)
            with torch.cuda.device(device):
                _lib.check(_L.gsr_sugar_colors_backward(dens.numel(), ctx.M, 0, None, None, None, None, None, p(dens), None, p(g_op), None,
                                                        None, None, p(d_dens), _lib.stream_ptr(device)), "gsr_sugar_colors_backward")
            return None, None, None, None, d_dens, None, None
        dens, src, dc, rest = ctx.saved_tensors[:4]
        c = None if ctx.directions_mode else ctx.saved_tensors[4]
        g_col, g_op = grads
        g_col = None if g_col is None else _dev_f32(g_col, device)
        g_op = None if g_op is None else _dev_f32(g_op, device)
        d_src = d_dc = d_rest = d_dens = None
        if g_col is not None:
            d_src, d_dc, d_rest = torch.empty_like(src), torch.empty_like(dc), torch.empty_like(rest)
        if g_op is not None:
            d_dens = torch.empty_like(dens)
        if g_col is not None or g_op is not None:
            pos, dirs = (None, p(src)) if ctx.directions_mode else (p(src), None)
            with torch.cuda.device(device):
                _lib.check(_L.gsr_sugar_colors_backward(dc.shape[0], ctx.M, ctx.deg, pos, None if c is None else c.data_ptr(), dirs, p(dc),
                                                        p(rest), p(dens), p(g_col), p(g_op), p(d_dc), p(d_rest), p(d_src), p(d_dens),
                                                        _lib.stream_ptr(device)), "gsr_sugar_colors_backward")
        return d_src, None, d_dc, d_rest, d_dens, None, None


def _sugar_raw_colors(self, raw, positions, camera_center, sh_deg, sh_rotations, compute_color_in_rasterizer, point_colors):
    """(shs, splat_colors, splat_opacities) of SS/:2063-2080 from the raw leaves through _SugarColors."""
    sh_dc, sh_rest, dens = raw
    if point_colors is not None or compute_color_in_rasterizer:  # the opacities alone
        opacities = _SugarColors.apply(None, None, sh_dc, sh_rest, dens, 0, False)
        return (self.sh_coordinates if point_colors is None else None), point_colors, opacities
    if sh_rotations is None:
        colors, opacities = _SugarColors.apply(positions, camera_center, sh_dc, sh_rest, dens, sh_deg, False)
    else:
        directions = (torch.nn.functional.normalize(positions - camera_center, dim=-1).unsqueeze(1) @ sh_rotations)[..., 0, :]
        colors, opacities = _SugarColors.apply(directions, None, sh_dc, sh_rest, dens, sh_deg, True)
    return None, colors, opacities


def render_sugar_raw(self, nerf_cameras=None, camera_indices=0, verbose=False, bg_color=None, sh_deg=None, sh_rotations=None,
                     compute_color_in_rasterizer=False, compute_covariance_in_rasterizer=True, return_2d_radii=False, quaternions=None,
                     use_same_scale_in_all_directions=False, return_opacities=False, return_colors=False, positions=None, point_colors=None):
    """render_sugar() with SuGaR's colours and opacities computed in CUDA from the model's raw leaves; a SuGaR model opts in with
    ``SuGaR.render_image_gaussian_rasterizer = render_sugar_raw``.  Same signature, return values, shapes and strides.

    ``get_points_rgb`` (SuGaR's eval_sh, degrees 0-4, ``+ 0.5``, ``clamp_min(0)``) and ``strengths`` (``sigmoid(all_densities)``)
    are one gsr_sugar_colors launch, and their backward one gsr_sugar_colors_backward launch, instead of the model's torch graph.
    The raw leaves read are ``_sh_coordinates_dc`` [P,1,3], ``_sh_coordinates_rest`` [P,M-1,3] (M = 1 allowed) and
    ``all_densities``; everything else (points, scaling, quaternions, sh_coordinates, the camera) comes through the getters
    render_sugar reads, so a mesh-bound model works as an unbound one.  Branches: ``point_colors`` and
    ``compute_color_in_rasterizer=True`` take the opacities alone (the SH leaves get no gradient from them); ``sh_rotations``
    passes the rotated directions, built in torch as the reference builds them; ``positions=`` receives the direction gradient.
    ValueError: a missing, non-float32 or misplaced leaf, a leaf of the wrong shape, ``return_one_densities`` set, or, when the
    colours are evaluated, ``sh_deg`` outside 0..4 or needing more than M coefficients (the reference's asserts)."""
    raw = _sugar_raw_leaves(self, sh_deg, point_colors is None and not compute_color_in_rasterizer)
    return _render_sugar(self, raw, nerf_cameras, camera_indices, verbose, bg_color, sh_deg, sh_rotations, compute_color_in_rasterizer,
                         compute_covariance_in_rasterizer, return_2d_radii, quaternions, use_same_scale_in_all_directions, return_opacities,
                         return_colors, positions, point_colors)
