"""extract_object's scoring loop (extract/extract_object.py:195-221, :314-340) restated on the library's render(), and the model and
cameras the extraction tests and tools/bench_extract.py feed it."""
from __future__ import annotations

import copy
import math
import types
from typing import Dict, List

import numpy as np
import torch

from autovfx_b200 import scene

PIPE = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
RAW = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")


class GaussianModel:
    """The reference GaussianModel's raw fields and getters (scene/gaussian_model.py:95-115), deep-copyable like the original."""

    def __init__(self, raw: Dict[str, torch.Tensor], active_sh_degree: int = 3, max_sh_degree: int = 3):
        for k in RAW:
            setattr(self, k, raw[k])
        self.active_sh_degree, self.max_sh_degree = active_sh_degree, max_sh_degree

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def get_normal(self, dir_pp_normalized=None):
        from tests import wrapper_ref as WR
        n, _ = WR.flip_align_view(WR.get_minimum_axis(self.get_scaling, self.get_rotation), dir_pp_normalized)
        return n / n.norm(dim=1, keepdim=True)


def model_from(g: Dict[str, torch.Tensor], device, sh_degree: int = 3) -> GaussianModel:
    """Raw parameters whose activations are (up to one rounding) the activated tensors of scene.synthetic_gaussians."""
    op = g["opacities"].double().clamp(1e-6, 1 - 1e-6)
    shs = g["shs"]
    raw = {"_xyz": g["means3D"], "_features_dc": shs[:, :1], "_features_rest": shs[:, 1:], "_scaling": torch.log(g["scales"]),
           "_rotation": g["rotations"], "_opacity": torch.log(op / (1 - op))}
    return GaussianModel({k: v.float().contiguous().to(device) for k, v in raw.items()}, sh_degree, sh_degree)


def render_camera(cam: scene.Camera, device):
    """The reference Camera's fields for a scene.Camera."""
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.image_height,
                                 image_width=cam.image_width, world_view_transform=cam.world_view_transform.to(device),
                                 full_proj_transform=cam.full_proj_transform.to(device), camera_center=cam.camera_center.to(device))


def orbit_views(cam: scene.Camera, n: int, device) -> List:
    """``cam`` and n - 1 cameras on its orbit about the z axis through the origin, same image size and field of view."""
    eye = cam.camera_center.double().cpu().numpy()
    fov = math.degrees(2 * math.atan(cam.tanfovx))
    views = [render_camera(cam, device)]
    for k in range(1, n):
        a = 2 * math.pi * k / n
        e = (eye[0] * math.cos(a) - eye[1] * math.sin(a), eye[0] * math.sin(a) + eye[1] * math.cos(a), eye[2] + 0.1 * k)
        views.append(render_camera(scene.lookat_camera(e, (0.0, 0.0, 0.0), cam.image_width, cam.image_height, fov), device))
    return views


def crop(gaussians: GaussianModel, mask3d: torch.Tensor, deep: bool = False) -> GaussianModel:
    """The cropped copy of :196-202: ``t[mask3d]`` of the six raw tensors (after a deepcopy of the model when ``deep``)."""
    out = copy.deepcopy(gaussians) if deep else GaussianModel({k: getattr(gaussians, k) for k in RAW}, gaussians.active_sh_degree,
                                                              gaussians.max_sh_degree)
    for k in RAW:
        setattr(out, k, getattr(gaussians, k)[mask3d])
    return out


def missed_pixels(gaussians: GaussianModel, camera_views, obj_masks, mask3d: torch.Tensor, background: torch.Tensor,
                  deep: bool = False) -> int:
    """total_missed_pixels of one ratio, as the reference loop computes it (:195-221), on the library's render()."""
    from autovfx_b200.renderer import render
    cropped_object_gaussians = crop(gaussians, mask3d, deep)
    total_missed_pixels = 0
    for idx, view in enumerate(camera_views):
        if "{0:05d}.png".format(idx) not in obj_masks.keys():
            continue
        object_mask_tracking = obj_masks["{0:05d}.png".format(idx)]
        with torch.no_grad():
            results = render(view, cropped_object_gaussians, PIPE, background)
        object_alpha_image = results["render"].permute(1, 2, 0)[:, :, 3].cpu().numpy()
        object_mask_rendered = object_alpha_image >= 0.8
        object_mask_tracking = np.array(object_mask_tracking) == 255
        xor_mask = np.logical_xor(object_mask_rendered, object_mask_tracking)
        xor_pixels = np.count_nonzero(xor_mask)
        total_missed_pixels += xor_pixels
    return total_missed_pixels


def box_subset(xyz: torch.Tensor, fraction: float) -> torch.Tensor:
    """The Gaussians inside an axis-aligned box about the scene's median point holding about ``fraction`` of them (the
    shape of an object's subset)."""
    c = xyz.median(dim=0).values
    d = (xyz - c).abs().max(dim=1).values
    r = torch.quantile(d[torch.randperm(d.numel(), generator=torch.Generator().manual_seed(0))[:100000].to(d.device)], fraction)
    return d <= r
