"""CPU checks of the render()-wrapper oracle (oracle/render_oracle.py) against the torch restatement of the reference's
helper functions (tests/wrapper_ref.py) executed with torch's CPU kernels."""
import math

import numpy as np
import pytest
import torch

from oracle import render_oracle as RO
from tests import wrapper_ref as WR
from tests.helpers import case_inputs


def _scene(P=4000, seed=0):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(P, 3, generator=g) * 4 - 2
    scales = torch.exp(torch.randn(P, 3, generator=g) * 0.6 - 3)
    rot = torch.randn(P, 4, generator=g)
    rot[:7] *= 3.0  # not normalised on purpose: build_rotation normalises
    campos = torch.tensor([0.3, -3.5, 0.7])
    return xyz, scales, rot, campos


def test_get_normal_matches_torch():
    xyz, scales, rot, campos = _scene()
    ref = WR.get_normal(xyz, scales, rot, campos).numpy()
    got = RO.get_normal(xyz.numpy(), scales.numpy(), rot.numpy(), campos.numpy())
    assert np.abs(got - ref).max() <= 5e-7  # torch's CPU norm may sum the squares in another order
    assert np.abs(np.linalg.norm(got, axis=1) - 1).max() < 1e-6
    got01 = RO.get_normal(xyz.numpy(), scales.numpy(), rot.numpy(), campos.numpy(), remap01=True)
    assert np.abs(got01 - (ref * 0.5 + 0.5)).max() <= 5e-7


def test_get_normal_faces_camera_and_picks_shortest_axis():
    xyz, scales, rot, campos = _scene(500, seed=3)
    n = RO.get_normal(xyz.numpy(), scales.numpy(), rot.numpy(), campos.numpy())
    view = (xyz - campos).numpy()
    assert ((n * -view).sum(1) >= -1e-6).all()
    R = RO.build_rotation(rot.numpy())
    k = scales.numpy().argmin(1)
    axis = R[np.arange(500), :, k]
    cosang = np.abs((axis * n).sum(1))
    assert np.abs(cosang - 1).max() < 1e-5


@pytest.mark.parametrize("H,W", [(37, 53), (16, 16), (3, 3), (2, 5)])
def test_normal_and_pseudo_normal_match_torch(H, W):
    g = torch.Generator().manual_seed(H * 100 + W)
    nimg = torch.rand(3, H, W, generator=g)
    nimg[:, 0, 0] = 0.5  # zero vector -> eps clamp
    depth = torch.rand(H, W, generator=g) * 3 + 0.5
    depth[H // 2:, : W // 3] = 0.0  # background
    cam = case_inputs("small_sh")["cam"]
    FoVx, FoVy = 2 * math.atan(cam.tanfovx), 2 * math.atan(cam.tanfovy)
    ref_n = WR.normal_image(nimg).numpy()
    got_n = RO.normal_image(nimg.numpy())
    assert np.abs(got_n - ref_n).max() <= 5e-7
    ref_p = WR.pseudo_normal(depth, cam.world_view_transform, FoVx, FoVy).numpy()
    c2w = torch.inverse(cam.world_view_transform).numpy()
    got_p = RO.pseudo_normal(depth.numpy(), c2w, WR.fov2focal(FoVx, W), WR.fov2focal(FoVy, H), W / 2, H / 2)
    assert got_p.shape == (H, W, 3)
    # the per-pixel 3x3 product is a GEMM in torch (summation order unspecified) and the stencil cancels: compare directions
    assert np.abs(got_p - ref_p).max() < 5e-3
    if H > 2 and W > 2:
        assert np.abs(got_p[0]).max() == 0 and np.abs(got_p[:, 0]).max() == 0 and np.abs(got_p[-1]).max() == 0


def test_8bit_conversions_match_torch_and_numpy():
    g = torch.Generator().manual_seed(5)
    H, W = 24, 40
    rgb = torch.rand(3, H, W, generator=g) * 1.4 - 0.2  # exercises the clamp
    alpha = torch.rand(H, W, generator=g)
    ref = WR.save_image_bytes(torch.cat([rgb, alpha[None]], 0)).numpy()
    assert (RO.rgba8(rgb.numpy(), alpha.numpy()) == ref).all()
    n = torch.nn.functional.normalize(torch.randn(H, W, 3, generator=g), dim=-1).numpy()
    ref_n = (((n + 1) / 2) * 255).astype(np.uint8)  # scene_representation.py:433-436
    assert (RO.normal8(n) == ref_n).all()
    d = (torch.rand(H, W, generator=g) * 5 - 0.5).numpy()
    ref_d = (np.clip(d / 3.0, a_min=0., a_max=1.) * 255).astype(np.uint8)  # sugar/render.py:18-21
    assert (RO.depth8(d, 3.0) == ref_d).all()


def test_turbo_table_shape():
    import importlib.util
    import os
    # the table lives in the product package, which needs the CUDA library to import; read the constant from the source
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "autovfx_b200", "renderer.py")).read()
    i0 = src.index("_TURBO_HEX = (")
    hexs = "".join(l.strip().strip('"') for l in src[i0:src.index(")\n", i0)].splitlines()[1:])
    raw = bytes.fromhex(hexs)
    assert len(raw) == 768
    lut = np.frombuffer(raw, dtype=np.uint8).reshape(256, 3)
    assert tuple(lut[0]) == (59, 18, 48) and tuple(lut[255]) == (3, 4, 122)  # cv2.COLORMAP_TURBO end points (B,G,R)
    del importlib


def _raw(N, M, seed):
    g = torch.Generator().manual_seed(seed)
    return {"xyz": torch.randn(N, 3, generator=g), "f_dc": torch.randn(N, 1, 3, generator=g), "f_rest": torch.randn(N, M - 1, 3, generator=g) * 0.1,
            "opacity": torch.randn(N, 1, generator=g) * 2, "scaling": torch.randn(N, 3, generator=g) * 0.5 - 3, "rotation": torch.randn(N, 4, generator=g)}


def _rot(seed):
    from scipy.spatial.transform import Rotation
    return torch.tensor(Rotation.random(random_state=seed).as_matrix(), dtype=torch.float32)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_matrix_to_quaternion_oracle_vs_scipy(seed):
    R = _rot(seed)
    q = RO.matrix_to_quaternion(R.numpy())
    ref = WR.matrix_to_quaternion(R).numpy()
    if q[0] < 0:
        q = -q
    assert np.abs(q - ref).max() < 1e-6
    assert abs(np.linalg.norm(q) - 1) < 1e-6


def test_transform_and_activate_oracle_vs_torch():
    raw = _raw(3000, 16, 4)
    R = _rot(5)
    center, pivot, s = torch.tensor([0.4, -1.2, 0.3]), torch.tensor([0.1, 0.2, -0.5]), 1.7
    quat = torch.from_numpy(RO.matrix_to_quaternion(R.numpy()))
    ref = WR.activate(WR.transform_gaussians(raw, center, R, s, pivot, quat=quat))
    rn = {k: v.numpy() for k, v in raw.items()}
    got = RO.activate(RO.transform_gaussians(rn, center.numpy(), R.numpy(), s, pivot.numpy()))
    assert np.abs(got["means3D"] - ref["means3D"].numpy()).max() < 2e-6
    assert np.abs(got["scales"] / ref["scales"].numpy() - 1).max() < 1e-6
    assert np.abs(got["rotations"] - ref["rotations"].numpy()).max() < 3e-7
    assert np.abs(got["opacities"] - ref["opacities"].numpy()).max() < 2e-7
    assert (got["shs"] == ref["shs"].numpy()).all() and got["shs"].shape == (3000, 16, 3)
    # identity transform = plain activation
    ident = RO.transform_gaussians(rn, pivot.numpy(), np.eye(3, dtype=np.float32), 1.0, pivot.numpy())
    assert np.abs(ident["xyz"] - rn["xyz"]).max() < 1e-6 and np.abs(ident["scaling"] - rn["scaling"]).max() == 0


def test_wrapper_oracle_against_golden_from_the_gpu():
    """tests/golden/wrapper_small_sh.npz: the reference's two rasterizer passes (compiled reference) around the wrapper's
    helper functions executed with torch's CUDA kernels (tests/golden/make_golden.py).  Pins oracle/render_oracle.py."""
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wrapper_small_sh.npz")
    if not os.path.exists(path):
        pytest.skip("golden file missing")
    z = np.load(path)
    case = case_inputs(str(z["case"]))
    g, cam = case["g"], case["cam"]
    n01 = RO.get_normal(g["means3D"].numpy(), g["scales"].numpy(), g["rotations"].numpy(), cam.camera_center.numpy(), remap01=True)
    assert np.abs(n01 - z["normal_normed"]).max() <= 5e-7
    assert np.abs(RO.normal_image(z["normal_raw_image"]) - z["normal"]).max() <= 5e-7
    H, W = z["depth"].shape
    fx, fy = WR.fov2focal(float(z["FoVx"]), W), WR.fov2focal(float(z["FoVy"]), H)
    pn = RO.pseudo_normal(z["depth"], z["c2w"], fx, fy, W / 2, H / 2)
    assert np.abs(pn - z["pseudo_normal"]).max() < 5e-3
    assert (RO.rgba8(z["render"][0:3], z["render"][3]) == z["rgba8"]).all()
    assert (RO.normal8(z["normal"]) == z["normal8"]).all()
    assert (RO.depth8(z["depth"], 3.0) == z["depth8"]).all()
