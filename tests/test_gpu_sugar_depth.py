"""coarse_sdf's depth-map estimate on the GPU: autovfx_b200.sugar_field's close_to_surface_mask and depth_sdf_estimation_loss
against the op-for-op torch restatement (tests/sugar_depth_ref.py), torch on the GPU being the live oracle.

- The lookup equals torch's grid_sample bit for bit on identical camera-space points (an identity world-to-view and a centred
  principal point, so that torch's projection GEMM has only one rounding per coordinate); with a principal-point offset the
  projection's multiply-add may round differently from torch's GEMM, and the bound reached is pinned.
- The mask equals the restatement's except where the comparison's two sides are within 1e-5 of the depth scale of each other
  (the count is printed; 0 on an H100 at 200k and 3M Gaussians).
- The loss and its three gradients meet, element by element, the fp64 restatement within a bound that torch's float32 graph meets.
- Edge cases, the deterministic backward (repeat-bitwise, next to a concurrent stream, the per-texel order pinned on the host) and
  the restatement's grid_sample backward raising under the flag.
- coarse_sdf's chain from the depth render (render_sugar with point_colors) through the mask, the sampler, the field, the depth
  loss and the better-normal loss, its leaf gradients against the torch restatement; and that chain as a seeded 20-step loop,
  under the flag, repeating bit for bit across processes."""
from __future__ import annotations

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import sugar_depth_ref as SD  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def _sf():
    from autovfx_b200 import sugar_field
    return sugar_field


@pytest.fixture
def deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was)


def _identity_camera(fx=1.3, fy=1.1, px=0.0, py=0.0):
    K = torch.zeros(1, 4, 4, device=DEV)
    K[0, 0, 0], K[0, 1, 1], K[0, 0, 2], K[0, 1, 2], K[0, 3, 2], K[0, 2, 3] = fx, fy, px, py, 1.0, 1.0
    return SD.Camera(torch.eye(3, device=DEV)[None], torch.zeros(1, 3, device=DEV), K, torch.tensor([0.0001], device=DEV))


def _depth(H, W, seed=0, strided=False):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    d = 4.0 + 0.3 * torch.sin(3 * xx) * torch.cos(2 * yy) + 0.01 * torch.rand(H, W, generator=g)
    if strided:  # render(...)[..., 0]: the first channel of an [H, W, 3] image
        img = torch.stack([d, d + 1, d + 2], -1).to(DEV)
        return img[..., 0]
    return d.to(DEV)


def _scene(P, N, H, W, seed=0, principal=(0.0, 0.0)):
    g = torch.Generator().manual_seed(seed)
    cam = SD.gs_camera((0.3, -0.2, -4.0), (0.0, 0.0, 0.0), W, H, 1.0, principal=principal, device=DEV)
    pts = torch.cat([torch.rand(P, 2, generator=g) * 4 - 2, torch.randn(P, 1, generator=g) * 0.3], 1)
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    sc = torch.rand(P, 3, generator=g) * 0.2 + 0.01
    model = SD.Model(pts.to(DEV), sc.to(DEV), q.to(DEV), H, W)
    x = torch.cat([torch.rand(N, 2, generator=g) * 5 - 2.5, torch.randn(N, 1, generator=g) * 0.5], 1).to(DEV)
    sdf = (torch.rand(N, generator=g) * 0.6 - 0.1).to(DEV)
    return model, cam, x, sdf


# ---- 1. the lookup ----------------------------------------------------------------------------------------------------------------
def _lookup_points(H, W, n=200_000, seed=1):
    g = torch.Generator().manual_seed(seed)
    z = torch.rand(n, generator=g) * 6 - 1  # some behind the camera
    xy = (torch.rand(n, 2, generator=g) * 3 - 1.5) * z.abs()[:, None]  # some outside the image
    p = torch.cat([xy, z[:, None]], 1)
    p[:4] = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, -1.0, 0.0], [0.5, 0.5, -2.0]])  # z = 0 (0 / 0, x / 0), behind
    return p.to(DEV)


def _map_z(model, cam, depth):
    return _sf()._surface_mask(model, cam, depth, 2.0, True)[1]


@pytest.mark.parametrize("H,W,strided", [(48, 64, False), (64, 48, False), (37, 37, True)])
def test_lookup_is_grid_sample_bit_for_bit(H, W, strided):
    depth = _depth(H, W, strided=strided)
    cam = _identity_camera()
    p = _lookup_points(H, W)
    model = SD.Model(p, torch.ones_like(p), torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(len(p), 4).contiguous(), H, W)
    got = _map_z(model, cam, depth)
    want = SD.get_points_depth_in_depth_map(model, cam, depth, p)
    assert torch.equal(got, want), int((got != want).sum())


def test_lookup_on_texel_edges_and_clip_limits():
    # a square map: SuGaR's factors are exactly -1, so grid = -(x / z) and the source index is exact in float32
    H = W = 16
    depth = _depth(H, W)
    cam = _identity_camera(fx=1.0, fy=1.0)
    ix = torch.tensor([0.0, 0.5, 1.0, 7.0, 14.0, 14.5, 15.0, 15.25, 15.5, 16.0, -0.5, -3.0])
    gx = (2 * ix + 1) / W - 1
    xs, ys = torch.meshgrid(gx, gx, indexing="ij")
    p = torch.stack([-xs.reshape(-1), -ys.reshape(-1), torch.ones(xs.numel())], 1).to(DEV)
    model = SD.Model(p, torch.ones_like(p), torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(len(p), 4).contiguous(), H, W)
    assert torch.equal(_map_z(model, cam, depth), SD.get_points_depth_in_depth_map(model, cam, depth, p))


def test_lookup_with_a_principal_point_offset():
    """The projection's x fx + z px is one multiply-add here; torch's GEMM may round the product first.  Pinned: the map depths
    differ from torch's by at most 1e-5 of the depth range, and most are identical."""
    H, W = 48, 64
    depth = _depth(H, W)
    cam = _identity_camera(px=0.137, py=-0.071)
    p = _lookup_points(H, W)
    p = p[p[:, 2] > 0.1]
    model = SD.Model(p, torch.ones_like(p), torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(len(p), 4).contiguous(), H, W)
    got = _map_z(model, cam, depth)
    want = SD.get_points_depth_in_depth_map(model, cam, depth, p)
    rng = float(depth.max() - depth.min())
    diff = (got - want).abs()
    print("principal offset: %d of %d map depths differ, max %.3g (depth range %.3g)" % (int((diff > 0).sum()), len(p), float(diff.max()), rng))
    assert float(diff.max()) <= 1e-5 * rng
    assert float((diff > 0).float().mean()) < 0.05


# ---- 2. the mask ------------------------------------------------------------------------------------------------------------------
def _mask_check(model, cam, depth):
    got = _sf().close_to_surface_mask(model, cam, depth)
    want, lhs, rhs = SD.surface_terms(model, cam, depth)
    bad = got != want
    # the band: camera-space coordinates rounded differently from torch's GEMM move z and map_z by float32 ulps of the depth
    band = (lhs - rhs).abs() <= 1e-5 * float(depth.abs().max())
    print("mask: %d of %d differ from the restatement, all within the band: %s; %d in the band" %
          (int(bad.sum()), len(got), bool(band[bad].all()), int(band.sum())))
    assert got.dtype == torch.bool and got.shape == want.shape
    assert bool(band[bad].all())
    assert 0 < int(got.sum()) < len(got)
    return got


@pytest.mark.parametrize("H,W,strided,principal", [(90, 160, False, (3.0, -2.0)), (160, 90, True, (0.0, 0.0))])
def test_mask_matches_the_restatement(H, W, strided, principal):
    model, cam, _, _ = _scene(200_000, 1, H, W, principal=principal)
    _mask_check(model, cam, _depth(H, W, strided=strided))


# ---- 3. the loss and its gradients ------------------------------------------------------------------------------------------------
def _run_ours(model, cam, depth, x, sdf, std=0.1, cmax=1.0):
    xr, sr = x.clone().requires_grad_(True), sdf.clone().requires_grad_(True)
    if depth.is_contiguous():
        leaf = depth.detach().clone().requires_grad_(True)
        dr = leaf
    else:  # keep the channel view of an [H, W, 3] render: the library reads it in place
        leaf = torch.stack([depth, depth + 1, depth + 2], -1).detach().requires_grad_(True)
        dr = leaf[..., 0]
    loss = _sf().depth_sdf_estimation_loss(model, cam, dr, xr, sr, std, cmax)
    loss.backward()
    return loss.detach(), xr.grad, leaf.grad if leaf is dr else leaf.grad[..., 0], sr.grad


def _run_ref(model, cam, depth, x, sdf, dtype, std=0.1, cmax=1.0):
    c = cam.to(dtype)
    c.znear = cam.znear.to(dtype)
    xr, dr, sr = (t.detach().to(dtype).clone().requires_grad_(True) for t in (x, depth, sdf))
    loss = SD.depth_sdf_estimation_loss(model, c, dr, xr, sr, std, cmax)
    loss.backward()
    return loss.detach(), xr.grad, dr.grad, sr.grad


def _assert_bound(ours, t32, f64, what, k=4.0, floor=1e-5):
    """|ours - f64| <= k |torch32 - f64| + floor * max|f64|, element by element (torch's float32 graph meets it by construction).
    A sample whose source coordinate lies within float32 rounding of a texel edge takes the neighbouring texel's one-sided
    gradient in float32, ours and torch's alike but not always on the same samples (the camera-space coordinates may differ from
    torch's GEMM by an ulp): such a sample may exceed the bound, up to torch's own largest error, and at most 1 in 200 of the
    elements may (0.14 % of dL/dsamples at 1M samples on a 1080p map)."""
    ours, t32, f64 = ours.double(), t32.double(), f64.double()
    bound = k * (t32 - f64).abs() + floor * f64.abs().max().clamp_min(1e-30)
    err = (ours - f64).abs()
    bad = ~(err <= bound)
    t32_max = float((t32 - f64).abs().max())
    print("%s: max err %.3g, torch32 max err %.3g, over the bound: %d of %d" % (what, float(err.max()), t32_max, int(bad.sum()),
                                                                           err.numel()))
    assert int(bad.sum()) <= max(2, err.numel() // 200), (what, int(bad.sum()))
    assert float(err.max()) <= k * t32_max + floor * float(f64.abs().max()), what


def _compare(model, cam, depth, x, sdf, **kw):
    ours = _run_ours(model, cam, depth, x, sdf, **kw)
    t32 = _run_ref(model, cam, depth, x, sdf, torch.float32, **kw)
    f64 = _run_ref(model, cam, depth, x, sdf, F64, **kw)
    for name, o, a, b in zip(("loss", "dL/dsamples", "dL/ddepth", "dL/dsdf"), ours, t32, f64):
        _assert_bound(o, a, b, name)
    return ours


@pytest.mark.parametrize("H,W,strided,principal", [(90, 160, False, (3.0, -2.0)), (160, 90, False, (0.0, 0.0)),
                                                   (120, 120, True, (-1.5, 4.0))])
def test_loss_and_gradients_against_float64(H, W, strided, principal):
    model, cam, x, sdf = _scene(100, 200_000, H, W, principal=principal)
    ours = _compare(model, cam, _depth(H, W, strided=strided), x, sdf)
    assert 0 < float(ours[0])


def test_clamped_terms_get_no_gradient():
    model, cam, x, sdf = _scene(100, 50_000, 90, 160)
    loss, dx, dd, ds = _run_ours(model, cam, _depth(90, 160), x, sdf, std=0.01, cmax=5.0)
    _compare(model, cam, _depth(90, 160), x, sdf, std=0.01, cmax=5.0)
    assert int((ds == 0).sum()) > 1000  # many terms are clamped


def test_edge_samples():
    """Samples exactly at znear (not in front: z > znear is strict), at z = 0, behind the camera, projecting outside the image on
    every side, on texel edges and exactly on the clip limits, with sdf = |est| (sign(0))."""
    H = W = 16
    depth = _depth(H, W)
    cam = _identity_camera(fx=1.0, fy=1.0)
    znear = float(np.float32(0.0001))
    ix = torch.tensor([0.0, 1.0, 7.0, 15.0, 15.5, -2.0, 20.0])
    gx = (2 * ix + 1) / W - 1
    xs, ys = torch.meshgrid(gx, gx, indexing="ij")
    edge = torch.stack([-xs.reshape(-1), -ys.reshape(-1), torch.ones(xs.numel())], 1)
    special = torch.tensor([[0.0, 0.0, znear], [0.1, 0.1, znear], [0.0, 0.0, 0.0], [0.2, 0.1, -1.0], [0.0, 0.0, 2 * znear]])
    x = torch.cat([edge, special]).to(DEV)
    model = SD.Model(x, torch.ones_like(x), torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(len(x), 4).contiguous(), H, W)
    sdf = torch.rand(len(x), generator=torch.Generator().manual_seed(3)).to(DEV)
    map_z = _map_z(model, cam, depth)
    sdf[:5] = (map_z[:5] - x[:5, 2]).abs()  # sign(0) of the outer |.|
    loss, dx, dd, ds = _run_ours(model, cam, depth, x, sdf, cmax=100.0)
    loss_r, dx_r, dd_r, ds_r = _run_ref(model, cam, depth, x, sdf, torch.float32, cmax=100.0)
    torch.testing.assert_close(loss, loss_r, rtol=1e-6, atol=0)
    torch.testing.assert_close(ds, ds_r, rtol=1e-5, atol=1e-12)
    torch.testing.assert_close(dx, dx_r, rtol=1e-3, atol=1e-9)
    torch.testing.assert_close(dd, dd_r, rtol=1e-5, atol=1e-9)
    n_edge = len(edge)
    assert torch.equal(ds[n_edge:n_edge + 4], torch.zeros(4, device=DEV))  # at znear, z = 0, behind: not in front
    assert float(ds[n_edge + 4]) != 0.0
    assert torch.equal(ds[:5], torch.zeros(5, device=DEV))


def test_every_sample_masked_and_no_sample():
    sf = _sf()
    model, cam, x, sdf = _scene(10, 1000, 32, 48)
    x[:, 2] = -10.0  # behind the camera: in world space the camera looks along +z from z = -4
    for xs, ss in ((x, sdf), (x[:0], sdf[:0])):
        xr, dr, sr = xs.clone().requires_grad_(True), _depth(32, 48).requires_grad_(True), ss.clone().requires_grad_(True)
        loss = sf.depth_sdf_estimation_loss(model, cam, dr, xr, sr, 0.1, 1.0)
        assert torch.isnan(loss)
        if len(xs):
            assert torch.isnan(SD.depth_sdf_estimation_loss(model, cam, dr.detach(), xs, ss, 0.1, 1.0))
        loss.backward()
        assert torch.equal(dr.grad, torch.zeros_like(dr)) and torch.equal(xr.grad, torch.zeros_like(xr))
        assert torch.equal(sr.grad, torch.zeros_like(sr))


def test_no_host_synchronisation():
    sf = _sf()
    model, cam, x, sdf = _scene(1000, 10_000, 90, 160)
    depth = _depth(90, 160).requires_grad_(True)
    xr, sr = x.clone().requires_grad_(True), sdf.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mask = sf.close_to_surface_mask(model, cam, depth.detach())
        loss = sf.depth_sdf_estimation_loss(model, cam, depth, xr, sr, 0.1, 1.0)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert mask.any() and xr.grad is not None and depth.grad is not None


def test_full_size_scene():
    """3M Gaussians, 1M samples, a 1080p depth map read as the channel of an [H, W, 3] render."""
    H, W = 1080, 1920
    model, cam, x, sdf = _scene(3_000_000, 1_000_000, H, W, principal=(0.0, 0.0))
    depth = _depth(H, W, strided=True)
    _mask_check(model, cam, depth)
    _compare(model, cam, depth, x, sdf)


# ---- 4. the deterministic backward ------------------------------------------------------------------------------------------------
def _grads(model, cam, depth, x, sdf):
    return _run_ours(model, cam, depth, x, sdf)[1:]


def test_deterministic_backward_repeats_bitwise(deterministic):
    model, cam, x, sdf = _scene(100, 300_000, 90, 160)
    depth = _depth(90, 160, strided=True)
    a = _grads(model, cam, depth, x, sdf)
    for _ in range(2):
        b = _grads(model, cam, depth, x, sdf)
        for u, v in zip(a, b):
            assert torch.equal(u.view(torch.int32), v.view(torch.int32))
    # next to a concurrent stream of other work
    side = torch.cuda.Stream()
    big = torch.randn(4096, 4096, device=DEV)
    with torch.cuda.stream(side):
        for _ in range(8):
            big = big @ big.T * 1e-4
    c = _grads(model, cam, depth, x, sdf)
    torch.cuda.synchronize()
    for u, v in zip(a, c):
        assert torch.equal(u.view(torch.int32), v.view(torch.int32))
    # the default (atomic) path gives the same per-sample gradients and the same depth gradient up to the summation order
    torch.use_deterministic_algorithms(False)
    d = _grads(model, cam, depth, x, sdf)
    assert torch.equal(a[0], d[0]) and torch.equal(a[2], d[2])
    torch.testing.assert_close(a[1], d[1], rtol=1e-5, atol=1e-9)


def test_deterministic_order_per_texel(deterministic, monkeypatch):
    """Every texel is the float32 sum from +0.0 of its samples' partials in ascending sample id (then tap): pinned by one backward
    per sample, the upstream gradient pre-divided by the count, summed on the host."""
    H, W = 6, 8
    model, cam, x, sdf = _scene(10, 64, H, W)
    depth = _depth(H, W)
    loss, _, dd, _ = _run_ours(model, cam, depth, x, sdf)
    sf = _sf()
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # the restatement's transform_points is a bmm
    cnt = int((cam.get_world_to_view_transform().transform_points(x)[:, 2] > cam.znear).sum())
    assert cnt > 10
    g = float(np.float32(1) / np.float32(cnt))
    acc = np.zeros(H * W, dtype=np.float32)
    for n in range(len(x)):
        dr = depth.detach().clone().requires_grad_(True)
        one = sf.depth_sdf_estimation_loss(model, cam, dr, x[n:n + 1], sdf[n:n + 1], 0.1, 1.0)
        if torch.isnan(one):
            continue
        (one * g).backward()  # count 1: the partial is g * dL/dmap_z * w, as in the full backward
        part = dr.grad.reshape(-1).cpu().numpy()
        nz = part != 0
        acc[nz] = (acc[nz] + part[nz]).astype(np.float32)
    assert np.array_equal(acc.view(np.int32), dd.reshape(-1).cpu().numpy().view(np.int32))


def test_torch_restatement_cannot_run_under_the_flag(deterministic, monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # so that the bmm of transform_points runs and grid_sample is reached
    model, cam, x, sdf = _scene(10, 1000, 32, 48)
    dr = _depth(32, 48).requires_grad_(True)
    loss = SD.depth_sdf_estimation_loss(model, cam, dr, x, sdf, 0.1, 1.0)
    with pytest.raises(RuntimeError, match="grid_sampler_2d_backward"):
        loss.backward()


# ---- 5. the coarse_sdf chain through the renderer, and a seeded step loop across processes ------------------------------------------
CH_W, CH_H, CH_FOV, CH_N = 160, 120, 1.0, 20_000


def _chain_model(dev):
    """A SuGaR stand-in (tests/sugar_field_ref.FieldModel: raw leaves, normalising quaternions getter, knn_idx, beta_mode) with
    one camera whose pytorch3d stand-in and renderer wrapper are the same camera (tests/sugar_depth_ref.Cameras)."""
    import math
    import types
    from autovfx_b200 import scene
    from autovfx_b200.knn import knn_points
    from tests import sugar_field_ref as SF
    g = scene.synthetic_gaussians(3000, seed=3, extent=(1.0, 1.0, 0.5), log_scale_mean=math.log(0.03), log_scale_std=0.5, sh_degree=3,
                                  M=16)
    g = {k: v.to(dev) for k, v in g.items()}
    knn = knn_points(g["means3D"][None], g["means3D"][None], K=16).idx[0]
    model = SF.FieldModel(g, knn)
    cams = SD.Cameras([SD.gs_camera((0.5, -3.0, 0.8), (0.0, 0.0, 0.0), CH_W, CH_H, CH_FOV, device=dev, up=(0.0, 0.0, 1.0))])
    model.image_width, model.image_height = CH_W, CH_H
    model.fov_x = CH_FOV
    model.fov_y = 2 * math.atan(math.tan(CH_FOV / 2) * CH_H / CH_W)
    model.tanfovx, model.tanfovy = math.tan(model.fov_x * 0.5), math.tan(model.fov_y * 0.5)
    model.nerfmodel = types.SimpleNamespace(training_cameras=cams, device=torch.device(dev))
    return model


def _chain(model, arm, seed=7, factor=0.2):
    """coarse_sdf.py:619-760 with its default flags for camera 0: the depth render (render_sugar with point_colors = the view
    depth, bg = its max, [..., 0]), the close-to-surface mask, the samples in it, the field, the depth estimation loss and the
    better-normal loss -> (loss, mask).  arm 'ours' runs the library; 'torch' runs the trainer's lines restated (the mask and the
    loss of tests/sugar_depth_ref.py, the field of tests/sugar_field_ref.py, the better-normal loss of tests/sugar_normal_ref.py
    with the library's sign convention, and the sampler restated with the library's draws so that both arms see the same
    samples).  The render is the library's in both arms."""
    from autovfx_b200 import sugar_field as sf
    from autovfx_b200.renderer import render_sugar
    from tests import sugar_field_ref as SF
    from tests import sugar_normal_ref as SN
    from tests import sugar_sample_ref as SSR
    fov_camera = model.nerfmodel.training_cameras.p3d_cameras[0]
    point_depth = fov_camera.get_world_to_view_transform().transform_points(model.points)[..., 2:].expand(-1, 3)
    max_depth = point_depth.max()
    depth = render_sugar(model, camera_indices=0, bg_color=max_depth + torch.zeros(3, dtype=torch.float, device=point_depth.device),
                         sh_deg=0, compute_color_in_rasterizer=False, compute_covariance_in_rasterizer=True, return_2d_radii=False,
                         use_same_scale_in_all_directions=False, point_colors=point_depth)[..., 0]
    extent = 1.0
    if arm == "ours":
        mask = sf.close_to_surface_mask(model, fov_camera, depth, 2.0)
        torch.manual_seed(seed)
        x, gidx = sf.sample_points_in_gaussians(model, CH_N, 1.5, mask=mask)
        fields = sf.get_field_values(model, x, gidx, return_sdf=True, density_threshold=1., density_factor=1. / 16.,
                                     return_closest_gaussian_opacities=True)
        est = sf.depth_sdf_estimation_loss(model, fov_camera, depth, x, fields["sdf"], extent / 10., 10. * extent)
        normal = sf.better_normal_loss(model, x, gidx, fields["closest_gaussian_opacities"])
    else:
        mask = SD.close_to_surface_mask(model, fov_camera, depth, 2.0)
        u, z = SSR.draws(CH_N, depth.device, seed)
        gidx, _ = SSR.select_rows(SSR.prefix(SSR.weights(model.scaling.detach(), mask=mask), mask), u)
        x = SSR.place(model.points, model.scaling, model.quaternions, gidx, z, 1.5)
        fields = SF.get_field_values(model, x, gidx, return_sdf=True, density_threshold=1., density_factor=1. / 16.,
                                     return_closest_gaussian_opacities=True)
        est = SD.depth_sdf_estimation_loss(model, fov_camera, depth, x, fields["sdf"], extent / 10., 10. * extent)
        normal = SN.better_normal_loss(model, x, gidx, fields["closest_gaussian_opacities"], sign=SN.pinned_signs(model, gidx))
    return factor * est + factor * normal.mean(), mask


def _chain_grads(dev, arm):
    model = _chain_model(dev)
    loss, mask = _chain(model, arm)
    loss.backward()
    return loss.detach(), mask, {k: v.detach().clone() for k, v in model.grads().items()}


def test_coarse_sdf_chain_through_the_renderer():
    """The gradients on the raw leaves (through the depth render's point_colors and geometry, the strided [..., 0] view, the
    mask, the samples, the field, the depth loss and the better-normal loss) against the torch restatement, flag off.  The
    renderer's backward adds with atomics, so torch's own graph differs from itself between runs; the bound is a relative
    Frobenius error per leaf of max(4x that spread, 1e-4), which torch's second run meets by construction."""
    loss_o, mask_o, g_o = _chain_grads(DEV, "ours")
    loss_a, mask_a, g_a = _chain_grads(DEV, "torch")
    loss_b, _, g_b = _chain_grads(DEV, "torch")
    assert torch.equal(mask_o, mask_a) and 100 < int(mask_o.sum()) < len(mask_o), int(mask_o.sum())
    torch.testing.assert_close(loss_o, loss_a, rtol=1e-5, atol=0)
    for k in ("_points", "all_densities", "_scales", "_quaternions"):
        assert k in g_o and k in g_a, k
        ref = g_a[k].double()
        spread = float((g_b[k].double() - ref).norm() / ref.norm())
        err = float((g_o[k].double() - ref).norm() / ref.norm())
        print("chain %s: relative Frobenius error %.3g, torch against itself %.3g" % (k, err, spread))
        assert float(ref.norm()) > 0 and err <= max(4 * spread, 1e-4), (k, err, spread)
    assert set(g_o) == set(g_a), (sorted(g_o), sorted(g_a))


def _sdf_loop(dev, steps=20):
    """coarse_sdf's SDF block on the library, 20 seeded steps: the depth render, the mask, the sampler, the field, the depth
    estimation loss and the better-normal loss, backward and plain SGD on the raw leaves."""
    model = _chain_model(dev)
    leaves = [model.leaves[k] for k in ("_points", "all_densities", "_scales", "_quaternions")]
    for _ in range(steps):
        loss, _ = _chain(model, "ours", seed=int(torch.randint(0, 2 ** 31 - 1, (1,))))
        loss.backward()
        with torch.no_grad():
            for p in leaves:
                p -= 1e-3 * p.grad
        for p in model.leaves.values():
            p.grad = None
    return {"p%d" % i: p.detach().cpu().numpy() for i, p in enumerate(leaves)}


def test_sdf_loop_is_bit_identical_across_processes(tmp_path):
    outs = []
    for i in range(2):
        path = tmp_path / ("sdf%d.npz" % i)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--sdf-worker", str(path)]
        res = subprocess.run(cmd, env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"), cwd=ROOT, capture_output=True, text=True,
                             timeout=900)
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        outs.append(dict(np.load(path)))
    a, b = outs
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k].view(np.int32), b[k].view(np.int32)), k
    assert not np.array_equal(a["p0"], _chain_model(DEV)._points.detach().cpu().numpy())  # the points moved


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--sdf-worker":
    torch.use_deterministic_algorithms(True)
    torch.manual_seed(0)
    np.savez(sys.argv[2], **_sdf_loop(DEV))
