"""render_sugar(): SuGaR's render_image_gaussian_rasterizer with one rasterizer pass per call, and SuGaR's shading normals and their
backward in CUDA (gsr_sugar_normals, gsr_sugar_normals_backward).  Run with -m gpu on an H100.  Checked here, in both image modes,
against the reference method restated as two GaussianRasterizer calls on the drop-in (tests/sugar_ref.sugar_render_two_pass):

  1. per-Gaussian normals: the kernel's axis is torch.min's index (also on 2- and 3-way ties) and its values are the torch graph's;
  2. the forward of every option branch, with and without gradients: image, depth and radii bit for bit, the normal maps within
     the wrapper bounds of DESIGN §2;
  3. the image-only call makes one rasterizer pass and no normals, with the reference's shape and strides;
  4. gradients of every raw leaf and of viewspace_points against the two-call graph, and the quaternion gradient of the normal
     against fp64 autograd;
  5. the empty scene, a scene behind the camera, and the image-only return under autograd.
"""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402
from tests import sugar_ref as SR  # noqa: E402

pytestmark = pytest.mark.gpu

W, H, FOV_X = 160, 120, 1.0
# against the two-call graph, per gradient tensor: the same non-zero rows, a median relative row error <= MED (test_gpu_fused_grads.py's
# median bound) and ||ours - two||_F <= FRO ||two||_F.  test_gpu_fused_grads.py's per-row bound (5e-5 ||two|| + 1e-5 max ||two||) does not
# hold here for the reference's own graph: on these scenes (160x120, 3000 Gaussians) the two-call graph run twice exceeds it by up to
# 72x on rows of _scales / _points, because the blend backward sums with atomics in a run-dependent order and many rows cancel (with
# cov3D_precomp it stays at 0.02x).  Measured on an H100 80GB HBM3 over four runs: render_sugar against it reached 44x that row bound,
# and a relative Frobenius error of 1.3e-3 on _scales under a depth-only loss, where both arms run the identical single backward; the
# spread of the two-call graph against itself varied from 1e-6 to the same order between runs.  FRO is 8x the worst Frobenius error
# seen; medians stayed at 6e-7 or less.  The kernel's own quaternion gradient is held to a per-row bound against fp64 below.
FRO, MED = 1e-2, 4e-6
LEAVES = ("_points", "all_densities", "_scales", "_quaternions", "_sh_coordinates_dc", "_sh_coordinates_rest")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import rasterizer  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


@pytest.fixture(params=[False, True], ids=["default", "exact"])
def exact(request, dev):
    from autovfx_b200 import rasterizer as R
    R.set_exact_images(request.param)
    yield request.param
    R.set_exact_images(False)


def _scene(dev, M=16, seed=3, P=3000, grad=True, cameras=None):
    """A SuGaR stand-in: quaternion norms over 0.3..3, 2-way ties on rows 0-15 and 3-way ties on rows 16-23 of the log-scales, and
    cameras on a ring with an off-centre principal point."""
    from autovfx_b200 import scene
    g = scene.synthetic_gaussians(P, seed=seed, extent=(1.0, 1.0, 0.5), log_scale_mean=math.log(0.03), log_scale_std=0.5, sh_degree=3, M=M)
    s = torch.log(g["scales"])
    s[0:16, 1] = s[0:16, 0]
    s[0:16, 2] = s[0:16, 0] + 0.5
    s[16:24] = s[16:24, :1]
    g["scales"] = torch.exp(s)
    norms = 0.3 * 10.0 ** torch.rand(P, generator=torch.Generator().manual_seed(seed))
    g = {k: v.to(dev) for k, v in g.items()}
    cams = cameras or SR.ring_cameras(4, device=dev, principal=(0.04, -0.03))
    model = SR.SugarModel(g, cams, W, H, FOV_X, quat_norms=norms, grad=grad)
    model._scales.data[0:24] = s[0:24].to(dev)  # the ties exactly in log space, so exp gives equal scales
    return model


def _options(model, name, dev):
    """Keyword arguments of one option branch of SS/:1956-2228 (the bg_color default is decided by the caller)."""
    P = model.n_points
    gen = torch.Generator().manual_seed(11)
    if name in ("plain", "bg_none"):
        return {}
    if name == "rasterizer_sh":
        return dict(compute_color_in_rasterizer=True)
    if name == "cov_python":
        return dict(compute_covariance_in_rasterizer=False)
    if name == "same_scale":
        return dict(use_same_scale_in_all_directions=True)
    if name == "quaternions":
        return dict(quaternions=model._quaternions.roll(1, dims=1) * 0.7)
    if name == "positions":
        return dict(positions=model._points * 1.05 + 0.02)
    if name == "sh_rotations":
        c, s = math.cos(0.4), math.sin(0.4)
        return dict(sh_rotations=torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]], device=dev))
    if name == "point_colors":
        return dict(point_colors=torch.rand(P, 3, generator=gen).to(dev))
    if name == "depth_call":  # the SDF branch of coarse_density.py: point_colors = point_depth, bg = max_depth
        return dict(point_colors=None, depth_call=True)
    raise KeyError(name)


def _call(fn, model, name, dev, sh_deg, **flags):
    kw = _options(model, name, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    if kw.pop("depth_call", False):
        from autovfx_b200.renderer import sugar_camera
        wvt = sugar_camera(model.nerfmodel.training_cameras, 1, model.fov_x, model.fov_y, dev)[0]  # view-space z of each point
        point_depth = (model.points @ wvt[:3, 2:3] + wvt[3, 2]).expand(-1, 3)
        kw["point_colors"] = point_depth
        bg = point_depth.max().detach().expand(3).contiguous()
    if name == "bg_none":
        bg = None
    return fn(model, camera_indices=1, bg_color=bg, sh_deg=sh_deg, **kw, **flags)


OPTS = ["plain", "rasterizer_sh", "cov_python", "same_scale", "quaternions", "positions", "sh_rotations", "point_colors", "depth_call"]
CFGS = [(16, 3), (25, 2), (16, 0), (25, 1)]
FLAGS = dict(return_2d_radii=True, return_opacities=True, return_colors=True)


# ---- 1. per-Gaussian normals --------------------------------------------------------------------------------------------------------
def test_normals_against_the_torch_graph_and_torch_min(dev):
    from autovfx_b200.renderer import sugar_normals
    model = _scene(dev, grad=False)
    campos = model.nerfmodel.training_cameras.p3d_cameras[0].get_camera_center()
    got = sugar_normals(model.points, model.scaling, model.quaternions, campos)
    want = SR.sugar_normal_torch(model.points, model.scaling, model.quaternions, campos)
    assert Hh.maxabs(got, want) <= 5e-7, Hh.maxabs(got, want)
    # torch.min(dim=-1) on this GPU returns the first minimal index on 2-way and 3-way ties; the kernel's column is that one
    s = model.scaling
    assert torch.equal(s[0:16, 0], s[0:16, 1]) and torch.equal(s[16:24, 0], s[16:24, 2])
    tk = s.min(dim=-1)[1]
    assert (tk[0:24] == 0).all()
    cols = SR.quaternion_to_matrix(model.quaternions)
    n = (got - 0.5) * 2
    for k in range(3):  # the kernel's normal is +-(column tk) normalised, not another column
        c = cols[:, :, k] / cols[:, :, k].norm(dim=1, keepdim=True)
        match = ((n * c).sum(-1).abs() - 1).abs() <= 1e-5
        assert bool(match[tk == k].all()), k
    # and on rows tied on axes 1 and 2 only
    s2 = s.clone()
    s2[0:16] = torch.stack((s[0:16, 0] * 2, s[0:16, 0], s[0:16, 0]), -1)
    assert (s2.min(dim=-1)[1][0:16] == 1).all()
    g2 = sugar_normals(model.points, s2, model.quaternions, campos)
    assert Hh.maxabs(g2, SR.sugar_normal_torch(model.points, s2, model.quaternions, campos)) <= 5e-7


# ---- 2. forward of every option branch --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", OPTS + ["bg_none"])
@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_forward_matches_the_two_call_method(dev, exact, name, grad):
    from autovfx_b200.renderer import render_sugar
    M, deg = CFGS[(OPTS + ["bg_none"]).index(name) % len(CFGS)]
    model = _scene(dev, M=M, grad=grad)
    with torch.set_grad_enabled(grad):
        got = _call(render_sugar, model, name, dev, deg, **FLAGS)
        want = _call(SR.sugar_render_two_pass, model, name, dev, deg, **FLAGS)
    assert sorted(got) == sorted(want)
    for k in ("image", "depth", "radii"):
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), (name, k)
    assert got["image"].stride() == want["image"].stride()
    assert got["image"].requires_grad == want["image"].requires_grad == grad
    assert int(got["radii"].gt(0).sum()) > 100
    assert Hh.maxabs(got["normal"], want["normal"]) <= 1e-4, (name, Hh.maxabs(got["normal"], want["normal"]))
    assert Hh.maxabs(got["pseudo_normal"], want["pseudo_normal"]) < 5e-3
    assert torch.equal(got["opacities"], want["opacities"])
    assert (got["colors"] is None) == (want["colors"] is None)
    if got["colors"] is not None:
        assert torch.equal(got["colors"], want["colors"])


# ---- 3. the image-only call ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_image_only_call_is_one_pass(dev, exact, grad, monkeypatch):
    from autovfx_b200 import rasterizer as R, renderer
    model = _scene(dev, M=25, grad=grad)
    calls = {"forward": 0, "normals": 0}
    real_fw, real_sn, real_apply = R.forward_raw, renderer.sugar_normals, renderer._SugarNormals.apply

    def fw(*a, **k):
        calls["forward"] += 1
        return real_fw(*a, **k)

    def sn(*a, **k):
        calls["normals"] += 1
        return real_sn(*a, **k)

    def ap(*a, **k):
        calls["normals"] += 1
        return real_apply(*a, **k)
    monkeypatch.setattr(R, "forward_raw", fw)
    monkeypatch.setattr(renderer, "sugar_normals", sn)
    monkeypatch.setattr(renderer._SugarNormals, "apply", ap)
    with torch.set_grad_enabled(grad):
        got = _call(renderer.render_sugar, model, "plain", dev, 2)
        assert calls == {"forward": 1, "normals": 0}
        want = _call(SR.sugar_render_two_pass, model, "plain", dev, 2)
    assert got.shape == want.shape == (H, W, 4) and got.stride() == want.stride()
    assert torch.equal(got, want)


# ---- 4. gradients ------------------------------------------------------------------------------------------------------------------
def _weights(dev, seed=5):
    gen = torch.Generator().manual_seed(seed)
    w = {"image": torch.randn(H, W, 4, generator=gen), "depth": torch.randn(H, W, generator=gen),
         "normal": torch.randn(H, W, 3, generator=gen)}
    return {k: v.to(dev) for k, v in w.items()}


def _loss(out, w, term):
    parts = {k: (out[k] * w[k]).sum() for k in ("image", "depth", "normal")}
    return sum(parts.values()) if term == "all" else parts[term]


def _assert_rows(got, want, what):
    g, w = got.double().cpu().reshape(want.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    assert torch.equal(g.ne(0).any(1), w.ne(0).any(1)), (what, "non-zero rows differ")
    if float(w.abs().max()) == 0.0:
        return
    fro = float((g - w).norm() / w.norm())
    med = float(np.median(Hh.row_errors(g, w)))
    assert fro <= FRO and med <= MED, (what, "relative Frobenius error %.3g, median relative row error %.3g" % (fro, med))


@pytest.mark.parametrize("name,M,deg", [("plain", 16, 3), ("plain", 25, 2), ("cov_python", 16, 1), ("rasterizer_sh", 25, 3),
                                        ("positions", 16, 2), ("depth_call", 16, 0)])
def test_gradients_match_the_two_call_graph(dev, exact, name, M, deg):
    from autovfx_b200.renderer import render_sugar
    w = _weights(dev)
    for term in ("image", "depth", "normal", "all"):
        res = {}
        for which, fn in (("ours", render_sugar), ("two", SR.sugar_render_two_pass)):
            model = _scene(dev, M=M)
            out = _call(fn, model, name, dev, deg, **FLAGS)
            _loss(out, w, term).backward()
            res[which] = dict(model.grads(), viewspace_points=out["viewspace_points"].grad)
        # with a loss on `normal` alone the two-call graph never reaches the colour pass, so the SH leaves have no gradient; the one
        # fused call gives them zeros (as render() does)
        for k in set(res["ours"]) ^ set(res["two"]):
            assert term == "normal" and k in res["ours"] and torch.count_nonzero(res["ours"][k]) == 0, (name, term, k)
        for k in res["two"]:
            _assert_rows(res["ours"][k], res["two"][k], (name, term, k))
        if term in ("normal", "all"):
            assert torch.count_nonzero(res["ours"]["_quaternions"]) > 0


def test_quaternion_gradient_of_the_normal_against_fp64(dev):
    from autovfx_b200.renderer import _SugarNormals
    model = _scene(dev)
    campos = model.nerfmodel.training_cameras.p3d_cameras[2].get_camera_center()
    q = model._quaternions.detach().clone().requires_grad_(True)
    out = _SugarNormals.apply(model.points.detach(), model.scaling.detach(), q, campos)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(9)).to(dev)
    out.backward(g)
    # the kernel's decisions: torch.min's index, and the sign of the output against that column
    k = model.scaling.min(dim=-1)[1]
    col = SR.quaternion_to_matrix(q.detach())[torch.arange(q.shape[0], device=dev), :, k]
    sign = torch.where(((out.detach() - 0.5) * col).sum(-1) >= 0, 1.0, -1.0)
    assert (sign > 0).any() and (sign < 0).any()
    q64 = q.detach().double().requires_grad_(True)
    SR.sugar_normal_forced(q64, k, sign.double()).backward(g.double())
    want = q64.grad
    d, n = (q.grad.double() - want).norm(dim=1), want.norm(dim=1)
    assert float((d / (1e-5 * n + 1e-7 * n.max())).max()) <= 1.0
    assert float(np.median(Hh.row_errors(q.grad, want))) <= 2e-6
    # and the numpy closed form the kernel implements
    vjp = SR.sugar_normal_vjp(q.detach().cpu().numpy(), k.cpu().numpy(), sign.cpu().numpy(), g.cpu().numpy())
    assert np.abs(vjp - want.cpu().numpy()).max() <= 1e-9 * float(n.max())


# ---- 5. edge cases ------------------------------------------------------------------------------------------------------------------
def test_empty_scene(dev):
    from autovfx_b200.renderer import render_sugar
    model = _scene(dev, P=0)
    out = render_sugar(model, camera_indices=0, sh_deg=3, **FLAGS)
    assert out["radii"].numel() == 0 and out["image"].shape == (H, W, 4)
    (out["image"].sum() + out["depth"].sum() + out["normal"].sum()).backward()
    with torch.no_grad():
        out = render_sugar(model, camera_indices=0, sh_deg=3, return_opacities=True)
    assert out["radii"].numel() == 0


@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_everything_behind_the_camera(dev, grad):
    from autovfx_b200.renderer import render_sugar
    cams = SR.Cameras([(3.0, 0.0, 0.5)], target=(6.0, 0.0, 0.5), device=dev)
    model = _scene(dev, grad=grad, cameras=cams)
    with torch.set_grad_enabled(grad):
        got = render_sugar(model, camera_indices=0, sh_deg=3, **FLAGS)
        want = SR.sugar_render_two_pass(model, camera_indices=0, sh_deg=3, **FLAGS)
    assert int(got["radii"].count_nonzero()) == 0
    for k in ("image", "depth", "radii"):
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(got["normal"], want["normal"]) and torch.equal(got["pseudo_normal"], want["pseudo_normal"])
    if grad:
        (got["image"].sum() + got["normal"].sum()).backward()


def test_image_only_return_under_autograd(dev, exact):
    from autovfx_b200.renderer import render_sugar
    w = torch.randn(H, W, 4, generator=torch.Generator().manual_seed(2)).to(dev)
    res = {}
    for which, fn in (("ours", render_sugar), ("two", SR.sugar_render_two_pass)):
        model = _scene(dev, M=16)
        img = fn(model, camera_indices=3, sh_deg=3)
        assert img.requires_grad and img.shape == (H, W, 4)
        (img * w).sum().backward()
        res[which] = model.grads()
    assert sorted(res["ours"]) == sorted(res["two"])
    for k in res["two"]:  # the same single pass and the same backward, up to the order of its atomic sums
        _assert_rows(res["ours"][k], res["two"][k], k)
