"""CPU tests of coarse_sdf's depth-map estimate: the exports of autovfx_b200.sugar_field's close_to_surface_mask and
depth_sdf_estimation_loss, their argument errors (raised before any device is touched), the C-ABI validation, and pins against
torch on CPU of the conventions the kernels restate (tests/sugar_depth_ref.py): the float32 rounding of SuGaR's rescaling factor,
grid_sample's border clip and its gradient at and beyond the clip limits, and the tap a coordinate on a texel edge takes."""
import os
import re

import numpy as np
import pytest
import torch

from tests import sugar_depth_ref as SD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = {"gsr_sugar_surface_mask", "gsr_sugar_depth_sdf_loss_bytes", "gsr_sugar_depth_sdf_loss", "gsr_sugar_depth_sdf_loss_backward",
         "gsr_sugar_depth_sdf_loss_backward_det_bytes", "gsr_sugar_depth_sdf_loss_backward_det"}


def test_exports():
    from autovfx_b200 import _lib, sugar_field
    assert NAMES <= set(_lib.EXPORTS) and _lib.ABI_VERSION == 4
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsr_b200.h")).read(), flags=re.S)
    for n in NAMES:
        assert re.search(r"\b%s\(" % n, hdr), n
    L = _lib.lib
    assert len(L.gsr_sugar_surface_mask.argtypes) == 16 and len(L.gsr_sugar_depth_sdf_loss.argtypes) == 18
    assert len(L.gsr_sugar_depth_sdf_loss_backward.argtypes) == 19 and len(L.gsr_sugar_depth_sdf_loss_backward_det.argtypes) == 21
    assert L.gsr_sugar_depth_sdf_loss_bytes(2048) == 16 and L.gsr_sugar_depth_sdf_loss_bytes(2049) == 32
    assert L.gsr_sugar_depth_sdf_loss_backward_det_bytes(1000, 1080, 1920) > 4 * 4 * 4000
    assert {"close_to_surface_mask", "depth_sdf_estimation_loss"} <= set(sugar_field.__all__)


def _model(P=8, H=6, W=10, dtype=torch.float32):
    g = torch.Generator().manual_seed(0)
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    return SD.Model(torch.randn(P, 3, generator=g).to(dtype), torch.rand(P, 3, generator=g).to(dtype), q.to(dtype), H, W)


def test_argument_errors():
    from autovfx_b200.sugar_field import close_to_surface_mask, depth_sdf_estimation_loss
    m = _model()
    cam = SD.gs_camera((0, 0, -4.), (0, 0, 0.), 10, 6, 1.0, device="cpu")
    depth = torch.rand(6, 10)
    x, sdf = torch.randn(5, 3), torch.rand(5)
    with pytest.raises(ValueError, match="depth must be a float32"):
        close_to_surface_mask(m, cam, depth.double())
    with pytest.raises(ValueError, match="depth must be a float32"):
        close_to_surface_mask(m, cam, depth[None])
    with pytest.raises(ValueError, match="close_gaussian_threshold"):
        close_to_surface_mask(m, cam, depth, close_gaussian_threshold=torch.tensor(2.))
    with pytest.raises(ValueError, match="self.quaternions"):
        close_to_surface_mask(SD.Model(m.points, m.scaling, m.quaternions[:, :3], 6, 10), cam, depth)
    with pytest.raises(ValueError, match="self.image_width"):
        close_to_surface_mask(SD.Model(m.points, m.scaling, m.quaternions, 6, 0), cam, depth)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        close_to_surface_mask(m, cam, depth)
    with pytest.raises(ValueError, match="sdf_samples"):
        depth_sdf_estimation_loss(m, cam, depth, x[:, :2], sdf, 0.1, 10.)
    with pytest.raises(ValueError, match="sdf_values"):
        depth_sdf_estimation_loss(m, cam, depth, x, sdf[:4], 0.1, 10.)
    with pytest.raises(ValueError, match="sdf_sample_std"):
        depth_sdf_estimation_loss(m, cam, depth, x, sdf, torch.tensor(0.1), 10.)
    with pytest.raises(ValueError, match="clamp_max"):
        depth_sdf_estimation_loss(m, cam, depth, x, sdf, 0.1, None)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        depth_sdf_estimation_loss(m, cam, depth, x, sdf, 0.1, 10.)


def test_c_abi_rejects_bad_arguments_before_any_launch():
    from autovfx_b200 import _lib
    L = _lib.lib

    def mask(P=10, H=4, W=4, depth=256, cam=256, pts=256, out=256):
        return L.gsr_sugar_surface_mask(P, H, W, 4, 1, depth, -1.0, -1.0, cam, pts, 256, 256, 2.0, out, None, None)

    for kw in (dict(P=-1), dict(H=0), dict(W=0), dict(H=65536, W=65536), dict(depth=None), dict(cam=None), dict(pts=None), dict(out=None)):
        assert mask(**kw) == -1, kw
    assert mask(P=0, pts=None, out=None) == 0  # P = 0 is a no-op

    def loss(N=10, ws=256, nbytes=1 << 20, out=256):
        return L.gsr_sugar_depth_sdf_loss(N, 4, 4, 4, 1, 256, -1.0, -1.0, 256, 256, 256, 10.0, 100.0, out, 256, ws, nbytes, None)

    assert loss(N=-1) == -1 and loss(out=None) == -1
    assert loss(ws=None) == -2 and b"workspace" in L.gsr_last_error()
    assert loss(ws=264) == -2 and loss(nbytes=15) == -2

    def bwd(N=10, dd=256, count=256):
        return L.gsr_sugar_depth_sdf_loss_backward(N, 4, 4, 4, 1, 256, -1.0, -1.0, 256, 256, 256, 10.0, 100.0, count, 256, 256, 256, dd,
                                                   None)

    assert bwd(dd=None) == -1 and bwd(count=None) == -1 and bwd(N=-1) == -1

    def det(scratch=256, nbytes=1 << 30):
        return L.gsr_sugar_depth_sdf_loss_backward_det(10, 4, 4, 4, 1, 256, -1.0, -1.0, 256, 256, 256, 10.0, 100.0, 256, 256, 256, 256,
                                                       256, scratch, nbytes, None)

    assert det(scratch=None) == -1 and det(scratch=264) == -1
    assert det(nbytes=L.gsr_sugar_depth_sdf_loss_backward_det_bytes(10, 4, 4) - 1) == -2 and b"scratch" in L.gsr_last_error()


def test_rescaling_factor_is_a_float32_multiply():
    # SS/:1195-1196 multiplies a float32 tensor by a Python double: torch rounds the double to float32 first
    H, W = 1079, 1917
    factor = -1 * min(H, W)
    t = torch.randn(100000, generator=torch.Generator().manual_seed(1))
    got = factor / W * t
    want = torch.from_numpy(np.float32(factor / W) * t.numpy())
    assert torch.equal(got, want)
    assert float(np.float32(factor / W)) != factor / W  # the rounding is there to pin


def _grid(ix, iy, W, H):
    """grid coordinates whose unnormalized source index ((g + 1) W - 1) / 2 is exactly ix (exact in float32 for these sizes)"""
    return torch.tensor([[[[(2 * ix + 1) / W - 1, (2 * iy + 1) / H - 1]]]], dtype=torch.float32)


def test_border_clip_and_texel_edges_against_torch():
    H, W = 4, 8
    depth = torch.arange(H * W, dtype=torch.float32).reshape(1, 1, H, W) ** 1.5

    def run(ix, iy):
        g = _grid(ix, iy, W, H).requires_grad_(True)
        out = torch.nn.functional.grid_sample(depth, g, mode="bilinear", padding_mode="border", align_corners=False)
        out.sum().backward()
        return out.item(), g.grad[0, 0, 0].tolist()

    d = depth[0, 0]
    # exactly on a texel edge: floor takes the texel itself, the gradient is the one-sided difference to the next texel
    v, (gx, gy) = run(3.0, 1.5)
    assert v == pytest.approx(0.5 * (d[1, 3] + d[2, 3]).item())
    assert gx == pytest.approx(0.5 * ((d[1, 4] - d[1, 3]) + (d[2, 4] - d[2, 3])).item() * W / 2, rel=1e-6)
    # exactly on the clip limits, and beyond them: the value is the border texel's and that coordinate's gradient is 0
    for ix in (0.0, W - 1.0, -3.0, W + 5.0):
        v, (gx, gy) = run(ix, 1.5)
        x = 0 if ix <= 0 else W - 1
        assert v == pytest.approx(0.5 * (d[1, x] + d[2, x]).item())
        assert gx == 0.0 and gy != 0.0
    for iy in (0.0, H - 1.0):
        v, (gx, gy) = run(2.5, iy)
        assert gy == 0.0 and gx != 0.0
    # just inside a limit the gradient is not 0
    assert run(np.nextafter(np.float32(W - 1), np.float32(0)).item(), 1.5)[1][0] != 0.0
