"""TEST INFRASTRUCTURE ONLY — numpy (float32, one rounding per operation like the reference's torch ops) restatement of the
per-Gaussian and per-pixel work of the reference's render() wrapper around its two rasterizer passes, and of the 8-bit
conversions of its frame loop.  Never imported by the product (autovfx_b200/); used by tests/ as the checker.

"GR/" = sugar/gaussian_splatting/gaussian_renderer/__init__.py, "GU/" = sugar/gaussian_splatting/utils/general_utils.py,
"GM/" = sugar/gaussian_splatting/scene/gaussian_model.py, "SR/" = scene_representation.py of haoyuhsu/autovfx.

Parity status: the reference ships no golden vectors for these functions and they cannot be imported here (GR/ imports
kornia, GU/:83 hard-codes device='cuda'); this restatement is pinned by tests/wrapper_ref.py — the same functions
restated op for op in torch and executed with torch's own CUDA kernels on the GPU box (tests/test_gpu_wrapper.py) —, by the
golden vectors that combination produced around the compiled reference rasterizer (tests/golden/wrapper_small_sh.npz,
tests/golden/make_golden.py) and by torch-CPU execution of the restatement in the CPU suite.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def build_rotation(r: np.ndarray) -> np.ndarray:
    """GU/:78-99 — normalised quaternion (r,x,y,z) -> rotation matrices [P,3,3]."""
    r = r.astype(f32)
    norm = np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.zeros((q.shape[0], 3, 3), dtype=f32)
    two = f32(2)
    R[:, 0, 0] = f32(1) - two * (y * y + z * z)
    R[:, 0, 1] = two * (x * y - w * z)
    R[:, 0, 2] = two * (x * z + w * y)
    R[:, 1, 0] = two * (x * y + w * z)
    R[:, 1, 1] = f32(1) - two * (x * x + z * z)
    R[:, 1, 2] = two * (y * z - w * x)
    R[:, 2, 0] = two * (x * z - w * y)
    R[:, 2, 1] = two * (y * z + w * x)
    R[:, 2, 2] = f32(1) - two * (x * x + y * y)
    return R


def get_minimum_axis(scales: np.ndarray, rotations: np.ndarray) -> np.ndarray:
    """GU/:136-141 — the rotation-matrix column of the smallest scale (argsort ascending, first entry; ties: lowest index)."""
    k = np.argmin(scales.astype(f32), axis=-1)  # first minimum = stable argsort()[0]
    R = build_rotation(rotations)
    return R[np.arange(R.shape[0]), :, k]


def norm3(v: np.ndarray) -> np.ndarray:
    """x.norm(dim=-1): sqrt of the left-to-right sum of squares."""
    v = v.astype(f32)
    return np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])


def get_normal(means3D: np.ndarray, scales: np.ndarray, rotations: np.ndarray, campos: np.ndarray, remap01: bool = False) -> np.ndarray:
    """GM/:120-124 with dir_pp_normalized of GR/:131-132 and flip_align_view GU/:151-157; remap01 = GR/:147."""
    dir_pp = means3D.astype(f32) - campos.astype(f32)[None, :]
    d = dir_pp / norm3(dir_pp)[:, None]
    n = get_minimum_axis(scales, rotations)
    nd = -d
    dot = n[:, 0] * nd[:, 0] + n[:, 1] * nd[:, 1] + n[:, 2] * nd[:, 2]
    sign = np.where(dot >= 0, f32(1), f32(-1)).astype(f32)
    n = n * sign[:, None]
    n = n / norm3(n)[:, None]
    if remap01:
        n = n * f32(0.5) + f32(0.5)
    return n.astype(f32)


def normalize_last(v: np.ndarray, eps: float = 1e-12) -> np.ndarray:
    """torch.nn.functional.normalize(p=2, dim=-1): v / max(||v||, eps)."""
    n = np.maximum(norm3(v), f32(eps))
    return (v.astype(f32) / n[..., None]).astype(f32)


def normal_image(normal_img_chw: np.ndarray) -> np.ndarray:
    """GR/:168-176 — (img - 0.5) * 2, HWC, unit length."""
    v = (normal_img_chw.astype(f32) - f32(0.5)) * f32(2.0)
    return normalize_last(np.transpose(v, (1, 2, 0)))


def ray_directions(H: int, W: int, fx: float, fy: float, cx: float, cy: float) -> np.ndarray:
    """GR/:41-80 (pass-by-centre branch): ((u - cx + 0.5)/fx, (v - cy + 0.5)/fy, 1) with u = column, v = row."""
    u = np.arange(W, dtype=f32)[None, :].repeat(H, 0)
    v = np.arange(H, dtype=f32)[:, None].repeat(W, 1)
    fx, fy, cx, cy = f32(fx), f32(fy), f32(cx), f32(cy)
    return np.stack([(u - cx + f32(0.5)) / fx, (v - cy + f32(0.5)) / fy, np.ones_like(u)], -1).astype(f32)


def pseudo_normal(depth_hw: np.ndarray, c2w: np.ndarray, fx: float, fy: float, cx: float, cy: float) -> np.ndarray:
    """GR/:178-191 + depth_pcd2normal GR/:23-38.  c2w = inverse of the stored world_view_transform (4x4)."""
    H, W = depth_hw.shape
    d = ray_directions(H, W, fx, fy, cx, cy)
    A = c2w.astype(f32)[:3, :3].T  # rays_d = directions @ c2w[:3,:3].T
    rays_d = np.stack([(d[..., 0] * A[0, k] + d[..., 1] * A[1, k]) + d[..., 2] * A[2, k] for k in range(3)], -1).astype(f32)
    rays_o = c2w.astype(f32)[:3, 3]
    xyz = (rays_o[None, None, :] + rays_d * depth_hw.astype(f32)[..., None]).astype(f32)
    l2r = xyz[1:H - 1, 2:W, :] - xyz[1:H - 1, 0:W - 2, :]
    b2t = xyz[0:H - 2, 1:W - 1, :] - xyz[2:H, 1:W - 1, :]
    n = np.stack([l2r[..., 1] * b2t[..., 2] - l2r[..., 2] * b2t[..., 1],
                  l2r[..., 2] * b2t[..., 0] - l2r[..., 0] * b2t[..., 2],
                  l2r[..., 0] * b2t[..., 1] - l2r[..., 1] * b2t[..., 0]], -1).astype(f32)
    out = np.zeros((H, W, 3), dtype=f32)
    if H > 2 and W > 2:
        out[1:H - 1, 1:W - 1] = normalize_last(n)
    return out


def rgba8(rgb_chw: np.ndarray, alpha_hw: np.ndarray) -> np.ndarray:
    """torchvision.utils.save_image of cat(rgb, alpha) (SR/:424-425, GR/:143): mul(255).add(0.5).clamp(0,255) -> uint8, HWC."""
    img = np.concatenate([rgb_chw.astype(f32), alpha_hw.astype(f32)[None]], 0)
    v = np.clip(img * f32(255) + f32(0.5), f32(0), f32(255))
    return np.transpose(v, (1, 2, 0)).astype(np.uint8)


def normal8(normal_hwc: np.ndarray) -> np.ndarray:
    """SR/:433-436 — ((n + 1) / 2 * 255).astype(uint8), RGB order."""
    v = (normal_hwc.astype(f32) + f32(1)) / f32(2)
    return (v * f32(255)).astype(np.uint8)


def depth8(depth_hw: np.ndarray, scale: float = 3.0) -> np.ndarray:
    """depth2img (sugar/render.py:18-22) up to the colormap: (clip(depth/scale, 0, 1) * 255).astype(uint8)."""
    d = np.clip(depth_hw.astype(f32) / f32(scale), f32(0), f32(1))
    return (d * f32(255)).astype(np.uint8)


# ----------------------------------------------------------------------------- per-frame edit path
def matrix_to_quaternion(R: np.ndarray) -> np.ndarray:
    """rotation_utils.py:24-84 for one 3x3 matrix: (w,x,y,z) of the best-conditioned candidate."""
    m = R.astype(f32).reshape(9)
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m
    sq = np.array([f32(1) + m00 + m11 + m22, f32(1) + m00 - m11 - m22, f32(1) - m00 + m11 - m22, f32(1) - m00 - m11 + m22], dtype=f32)
    q_abs = np.where(sq > 0, np.sqrt(np.maximum(sq, f32(0))), f32(0)).astype(f32)
    cand = np.array([[q_abs[0] ** 2, m21 - m12, m02 - m20, m10 - m01], [m21 - m12, q_abs[1] ** 2, m10 + m01, m02 + m20],
                     [m02 - m20, m10 + m01, q_abs[2] ** 2, m12 + m21], [m10 - m01, m20 + m02, m21 + m12, q_abs[3] ** 2]], dtype=f32)
    cand = cand / (f32(2) * np.maximum(q_abs, f32(0.1)))[:, None]
    return cand[int(np.argmax(q_abs))].astype(f32)


def quaternion_multiply(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """rotation_utils.py:113-150 (product, then real part made non-negative); a [4], b [N,4]."""
    aw, ax, ay, az = (f32(v) for v in a)
    bw, bx, by, bz = (b[:, i].astype(f32) for i in range(4))
    ow = aw * bw - ax * bx - ay * by - az * bz
    ox = aw * bx + ax * bw + ay * bz - az * by
    oy = aw * by - ax * bz + ay * bw + az * bx
    oz = aw * bz + ax * by - ay * bx + az * bw
    q = np.stack([ow, ox, oy, oz], -1).astype(f32)
    return np.where(q[:, 0:1] < 0, -q, q).astype(f32)


def transform_gaussians(raw: dict, center, rotation, scaling: float, initial_center) -> dict:
    """gaussians_utils.py:88-125 on a dict of raw float32 arrays (xyz, scaling (log), rotation; the rest passes through)."""
    c = np.asarray(initial_center, dtype=f32)[None, :]
    R = np.asarray(rotation, dtype=f32).reshape(3, 3)
    s = f32(scaling)
    xyz = raw["xyz"].astype(f32) - c
    xyz = xyz * s
    xyz = xyz + c
    scales = raw["scaling"].astype(f32) + f32(np.log(scaling))
    xyz = xyz - c
    A = R.T  # xyz @ R.T, accumulated left to right with fused multiply-adds like a K=3 GEMM
    acc = (xyz[:, 0:1] * A[0][None, :]).astype(f32)
    for j in (1, 2):
        acc = (xyz[:, j:j + 1].astype(np.float64) * A[j][None, :].astype(np.float64) + acc.astype(np.float64)).astype(f32)
    xyz = acc + c
    rot = quaternion_multiply(matrix_to_quaternion(R), raw["rotation"].astype(f32))
    xyz = xyz + (np.asarray(center, dtype=f32)[None, :] - c)
    out = dict(raw)
    out["xyz"], out["rotation"], out["scaling"] = xyz.astype(f32), rot, scales.astype(f32)
    return out


def activate(raw: dict) -> dict:
    """scene/gaussian_model.py:95-115: exp, normalize, sigmoid, cat(dc, rest)."""
    q = raw["rotation"].astype(f32)
    n = np.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    op = raw["opacity"].astype(f32)
    return {"means3D": raw["xyz"].astype(f32), "shs": np.concatenate([raw["f_dc"], raw["f_rest"]], 1).astype(f32),
            "opacities": (f32(1) / (f32(1) + np.exp(-op))).astype(f32), "scales": np.exp(raw["scaling"].astype(f32)),
            "rotations": (q / np.maximum(n, f32(1e-12))[:, None]).astype(f32)}
