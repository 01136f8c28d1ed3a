"""CPU checks of render_sugar(), the mirror of SuGaR's render_image_gaussian_rasterizer: SuGaR's shading normal stated in numpy float32
(tests/sugar_ref.py, the arithmetic gsr_sugar_normals implements) and its closed-form VJP (the formula of
gsr_sugar_normals_backward) against fp64 autograd of the torch restatement; the quaternion_to_matrix restatement against scipy; the
camera matrices against a literal statement of SuGaR's graphics utilities; and the new C exports.  The GPU side is checked in
tests/test_gpu_sugar_render.py."""
import os
import re

import numpy as np
import pytest
import torch

from tests import sugar_ref as SR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sugar_rows(P, seed):
    """Quaternions with norms over 0.3..3, rows with two and three equal smallest scales, positions on both sides of every axis
    (both flip signs), and one row whose axis is exactly orthogonal to the view direction (dot = 0: kept)."""
    g = np.random.default_rng(seed)
    q = g.normal(size=(P, 4))
    q *= (0.3 * 10.0 ** g.uniform(0, 1, size=P) / np.linalg.norm(q, axis=1))[:, None]
    sc = np.exp(g.normal(-3.0, 0.7, size=(P, 3)))
    sc[0:8, 1] = sc[0:8, 0]  # 2-way tie on the smallest scale
    sc[0:8, 2] = sc[0:8, 0] * 2
    sc[8:12, 2] = sc[8:12, 1]  # 2-way tie between axes 1 and 2
    sc[8:12, 0] = sc[8:12, 1] * 3
    sc[12:20] = sc[12:20, :1]  # 3-way ties
    pos = g.normal(size=(P, 3))
    campos = np.array([0.25, -0.5, 0.125])
    # row 20: q = 2 * (1, 0, 0, 0) -> column 0 is (1, 0, 0) exactly; a view direction in the y-z plane makes the dot exactly 0
    q[20], sc[20], pos[20] = (2.0, 0.0, 0.0, 0.0), (0.01, 0.02, 0.03), campos + np.array([0.0, 1.5, -0.75])
    return pos.astype(np.float32), sc.astype(np.float32), q.astype(np.float32), campos.astype(np.float32)


def _autograd(q32, k, sign, g):
    q = torch.from_numpy(q32).double().requires_grad_(True)
    out = SR.sugar_normal_forced(q, torch.from_numpy(k), torch.from_numpy(sign).double())
    out.backward(torch.from_numpy(g).double())
    return out.detach().numpy(), q.grad.numpy()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_normal_and_vjp_against_fp64_autograd(seed):
    pos, sc, q, campos = sugar_rows(512, seed)
    n32, k, sign = SR.sugar_normal_np(pos, sc, q, campos)
    # the decisions: torch.min's index (first minimal on ties) and both flip signs, with the dot = 0 row kept
    tk = torch.from_numpy(sc).min(dim=-1)[1].numpy()
    assert np.array_equal(k, tk) and (k[0:8] == 0).all() and (k[8:12] == 1).all() and (k[12:20] == 0).all()
    assert (sign > 0).any() and (sign < 0).any() and sign[20] == 1
    n64, _ = _autograd(q, k, sign, np.zeros((512, 3)))
    assert np.abs(n32 - n64).max() <= 5e-7
    # the torch graph of the reference (float32, its own decisions) agrees with the numpy statement
    t32 = SR.sugar_normal_torch(torch.from_numpy(pos), torch.from_numpy(sc), torch.from_numpy(q), torch.from_numpy(campos).reshape(1, 3))
    assert np.abs(t32.numpy() - n32).max() <= 2.5e-7
    g = np.random.default_rng(seed + 10).normal(size=(512, 3))
    _, want = _autograd(q, k, sign, g)
    got = SR.sugar_normal_vjp(q, k, sign, g)
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()
    assert np.abs(got[20]).max() > 0


def test_overrides_change_the_flip_not_the_axis():
    """render_sugar's normals read the model's quaternions and scaling, and face the camera from the `positions` argument: moving
    the positions through the camera flips the normal; other quaternions handed to the rasterizer do not enter."""
    pos, sc, q, campos = sugar_rows(256, 4)
    n, k, sign = SR.sugar_normal_np(pos, sc, q, campos)
    mirrored = (2 * campos[None] - pos).astype(np.float32)
    n2, k2, sign2 = SR.sugar_normal_np(mirrored, sc, q, campos)
    flipped = sign2 != sign
    assert np.array_equal(k, k2) and flipped.sum() >= 250
    assert np.allclose((n2 - 0.5)[flipped], -(n - 0.5)[flipped], atol=1e-7)


def test_quaternion_to_matrix_against_scipy():
    from scipy.spatial.transform import Rotation
    from autovfx_b200.renderer import quaternion_to_matrix
    g = np.random.default_rng(3)
    q = g.normal(size=(200, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    want = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix()  # scipy: (x, y, z, w)
    for fn in (quaternion_to_matrix, SR.quaternion_to_matrix):
        got = fn(torch.from_numpy(q)).numpy()
        assert np.abs(got - want).max() <= 1e-12
        s = torch.from_numpy(10.0 ** g.uniform(-0.5, 0.5, size=(200, 1)))
        assert np.abs(fn(torch.from_numpy(q) * s).numpy() - want).max() <= 1e-12  # scale-invariant
    qf = torch.from_numpy(q).float() * 1.7
    assert torch.equal(quaternion_to_matrix(qf), SR.quaternion_to_matrix(qf))


def test_camera_matrices_reproduce_sugars_graphics_utils():
    from autovfx_b200.renderer import _sugar_projection, sugar_camera
    cams = SR.ring_cameras(5, device="cpu", principal=(0.03, -0.02))
    fov_x = 1.1
    fov_y = 2 * np.arctan(np.tan(fov_x / 2) * 90 / 160)
    for i in range(5):
        wv, full, center, c2w = sugar_camera(cams, i, fov_x, fov_y, torch.device("cpu"))
        # the literal statement of SS/:2010-2032
        c = torch.cat([cams.camera_to_worlds[i], torch.Tensor([[0, 0, 0, 1]])], dim=0).numpy()
        c[:3, 1:3] *= -1
        w2c = np.linalg.inv(c)
        wv_ref = torch.Tensor(SR.getWorld2View(R=np.transpose(w2c[:3, :3]), t=w2c[:3, 3])).transpose(0, 1)
        proj = SR.getProjectionMatrix(0.01, 100.0, fov_x, fov_y).transpose(0, 1)
        proj[..., 2, 0], proj[..., 2, 1] = -cams.p3d_cameras[i].K[0, 0, 2], -cams.p3d_cameras[i].K[0, 1, 2]
        full_ref = wv_ref.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
        assert torch.equal(wv, wv_ref) and torch.equal(full, full_ref) and np.array_equal(c2w, c)
        assert c2w.dtype == np.float32 and center.shape == (1, 3)
        # the camera centre maps to the view-space origin; the projection's focal terms are 1 / tan(fov / 2)
        assert np.abs((np.append(center.numpy()[0], 1.0) @ wv.numpy())[:3]).max() <= 1e-5
        assert float((torch.tensor([0.0, 0.0, 0.0, 1.0]) @ wv)[2]) > 0  # the target (the origin) lies in front: COLMAP axes
    P = _sugar_projection(0.01, 100.0, fov_x, fov_y)
    assert torch.equal(P, SR.getProjectionMatrix(0.01, 100.0, fov_x, fov_y))
    assert abs(float(P[0, 0]) - 1 / np.tan(fov_x / 2)) <= 1e-6 and float(P[3, 2]) == 1.0


def test_batched_camera_indices_fail_as_in_the_reference():
    """sugar/render.py's batched call cannot run in the reference either (torch.cat of [[0,0,0,1]] with a batch of c2w)."""
    from autovfx_b200.renderer import sugar_camera
    cams = SR.ring_cameras(3, device="cpu")
    with pytest.raises((RuntimeError, TypeError)):
        sugar_camera(cams, torch.tensor([0, 1]), 1.0, 1.0, torch.device("cpu"))


def test_sugar_normal_exports():
    from autovfx_b200 import _lib, renderer
    assert {"gsr_sugar_normals", "gsr_sugar_normals_backward"} <= set(_lib.EXPORTS) and _lib.ABI_VERSION == 4
    hdr = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    assert re.search(r"int gsr_sugar_normals\(", hdr) and re.search(r"int gsr_sugar_normals_backward\(", hdr)
    L = _lib.lib
    assert L.gsr_sugar_normals(0, None, None, None, None, None, None) == 0  # P = 0 is a no-op
    assert L.gsr_sugar_normals_backward(0, None, None, None, None, None, None, None) == 0
    # partly-NULL argument lists are rejected before any launch
    assert L.gsr_sugar_normals(4, 16, None, 16, 16, 16, None) != 0
    assert "gsr_sugar_normals" in L.gsr_last_error().decode()
    assert L.gsr_sugar_normals_backward(4, 16, 16, 16, 16, None, 16, None) != 0
    assert L.gsr_sugar_normals(-1, None, None, None, None, None, None) != 0
    with pytest.raises(RuntimeError, match="no CPU path"):
        renderer.sugar_normals(torch.zeros(4, 3), torch.ones(4, 3), torch.ones(4, 4), torch.zeros(3))
