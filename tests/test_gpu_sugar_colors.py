"""render_sugar_raw(): render_sugar() with SuGaR's colours (get_points_rgb, eval_sh up to degree 4) and opacities (strengths) computed
from the raw leaves by gsr_sugar_colors, and their backward by gsr_sugar_colors_backward.  Run with -m gpu on an H100.  Checked here,
in both image modes, on the scenes and option branches of tests/test_gpu_sugar_render.py plus degree 4 at M = 25:

  1. per-Gaussian outputs: colours bit for bit the numpy float32 restatement (tests/sugar_colors_ref.py) and, in directions mode,
     torch's get_points_rgb; in camera-centre mode within 1e-6 of torch's; opacities within 1.2e-7 of torch.sigmoid;
  2. the forward of every option branch, with and without gradients: bit for bit render_sugar on a model whose get_points_rgb and
     strengths return the kernels' own outputs, and within DESIGN §2's bounds of render_sugar on the plain model;
  3. the kernel backward against fp64 autograd per Gaussian row, and every leaf's gradient end to end against render_sugar and the
     two-call method;
  4. the empty scene, a scene behind the camera, a Gaussian at the camera centre, M = 1, sh_deg beyond the storage, and a mesh-bound
     model whose points, scaling and quaternions are functions of other leaves.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import math  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402
from tests import sugar_colors_ref as SC  # noqa: E402
from tests import sugar_ref as SR  # noqa: E402
from tests import test_gpu_sugar_render as TS  # noqa: E402

pytestmark = pytest.mark.gpu

ROW_REL, ROW_ABS, MED = 1e-5, 1e-7, 2e-6  # test_gpu_raw_render.py's bounds against fp64 autograd
FLAGS, OPTS, CFGS = TS.FLAGS, TS.OPTS, TS.CFGS
BRANCHES = [(n, *CFGS[i % len(CFGS)]) for i, n in enumerate(OPTS + ["bg_none"])] + [("plain", 25, 4), ("sh_rotations", 25, 4),
                                                                                     ("point_colors", 25, 4), ("plain", 1, 0)]


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


def _scene(dev, M=16, grad=True, **kw):
    """test_gpu_sugar_render's SuGaR stand-in, with SuGaR's eval_sh up to degree 4."""
    model = TS._scene(dev, M=M, grad=grad, **kw)
    model.__class__ = SC.SugarModel4
    return model


class KernelModel(SC.SugarModel4):
    """A SuGaR stand-in whose get_points_rgb and strengths return the kernels' outputs: render_sugar on it is render_sugar_raw's
    frame by construction."""

    def get_points_rgb(self, positions=None, camera_centers=None, directions=None, sh_levels=None, sh_coordinates=None):
        from autovfx_b200.renderer import _SugarColors
        raw = (self._sh_coordinates_dc, self._sh_coordinates_rest, self.all_densities, sh_levels - 1)
        if camera_centers is not None:
            return _SugarColors.apply(positions, camera_centers, *raw, False)[0]
        return _SugarColors.apply(directions, None, *raw, True)[0]

    @property
    def strengths(self):
        from autovfx_b200.renderer import _SugarColors
        return _SugarColors.apply(None, None, self._sh_coordinates_dc, self._sh_coordinates_rest, self.all_densities, 0, False)


def _as(model, cls):
    model.__class__ = cls
    return model


# ---- 1. per-Gaussian outputs --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,deg", [(16, 3), (25, 2), (16, 0), (25, 1), (25, 4), (9, 2), (1, 0)])
def test_per_gaussian_outputs(dev, M, deg):
    from autovfx_b200.renderer import _SugarColors
    model = _scene(dev, M=M, grad=False)
    campos = model.nerfmodel.training_cameras.p3d_cameras[1].get_camera_center()
    dc, rest, dens = model._sh_coordinates_dc, model._sh_coordinates_rest, model.all_densities
    sh = model.sh_coordinates.cpu().numpy()
    pos = model.points
    c, s = math.cos(0.4), math.sin(0.4)
    rot = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]], device=dev)
    dirs = ((torch.nn.functional.normalize(pos - campos, dim=-1).unsqueeze(1) @ rot)[..., 0, :] * 1.1).contiguous()
    # directions mode: torch's get_points_rgb(directions=...) bit for bit
    got, op = _SugarColors.apply(dirs, None, dc, rest, dens, deg, True)
    want = model.get_points_rgb(positions=pos, camera_centers=None, directions=dirs, sh_levels=deg + 1)
    assert torch.equal(got, want)
    assert np.array_equal(got.cpu().numpy(), SC.colors_np(deg, sh, dirs.cpu().numpy())[0])
    # camera-centre mode: the kernel is the float32 restatement bit for bit; torch's F.normalize rounds its norm differently
    got_c, op_c = _SugarColors.apply(pos, campos, dc, rest, dens, deg, False)
    want_c = model.get_points_rgb(positions=pos, camera_centers=campos, sh_levels=deg + 1)
    ref_c = SC.colors_np(deg, sh, SC.view_dirs_np(pos.cpu().numpy(), campos.cpu().numpy()))[0]
    assert np.array_equal(got_c.cpu().numpy(), ref_c)
    assert Hh.maxabs(got_c, want_c) <= 1e-6, Hh.maxabs(got_c, want_c)
    share = float((got_c == want_c).all(1).float().mean())
    print("M=%d deg=%d: camera-centre colours bit-equal to torch on %.4f of the rows" % (M, deg, share))
    # opacities: sigmoid = 1 / (1 + exp(-x)), within edit.activate's bound of torch.sigmoid
    assert torch.equal(op, op_c) and op.shape == (model.n_points, 1) and op.stride() == (1, 1)
    assert Hh.maxabs(op, torch.sigmoid(dens.view(-1, 1))) <= 1.2e-7
    assert got.shape == (model.n_points, 3) and got.stride() == (3, 1)


# ---- 2. forward of every option branch ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,M,deg", BRANCHES)
@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_forward_matches_render_sugar(dev, exact, name, M, deg, grad):
    from autovfx_b200.renderer import render_sugar, render_sugar_raw
    model = _scene(dev, M=M, grad=grad)
    with torch.set_grad_enabled(grad):
        got = TS._call(render_sugar_raw, model, name, dev, deg, **FLAGS)
        want = TS._call(render_sugar, _as(model, KernelModel), name, dev, deg, **FLAGS)
        got_img = TS._call(render_sugar_raw, _as(model, SC.SugarModel4), name, dev, deg)
        want_img = TS._call(render_sugar, _as(model, KernelModel), name, dev, deg)
        plain = TS._call(render_sugar, _as(model, SC.SugarModel4), name, dev, deg, **FLAGS)
    assert sorted(got) == sorted(want) == sorted(plain)
    for k in ("image", "depth", "radii", "normal", "pseudo_normal", "opacities"):
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), (name, k)
        assert got[k].stride() == plain[k].stride(), (name, k)
    assert (got["colors"] is None) == (plain["colors"] is None)
    if got["colors"] is not None:
        assert torch.equal(got["colors"], want["colors"]) and got["colors"].stride() == plain["colors"].stride()
    assert got_img.shape == plain["image"].shape and got_img.stride() == want_img.stride() and torch.equal(got_img, want_img)
    assert got["image"].requires_grad == plain["image"].requires_grad == grad
    # against the model's own torch colours and sigmoid: DESIGN §2's default-mode bounds
    assert torch.equal(got["radii"], plain["radii"]) and int(got["radii"].gt(0).sum()) > 100
    assert Hh.maxabs(got["image"], plain["image"]) <= 1e-5, (name, Hh.maxabs(got["image"], plain["image"]))
    assert Hh.maxabs(got["depth"], plain["depth"]) <= 5e-5
    assert Hh.maxabs(got["normal"], plain["normal"]) <= 1e-4
    assert Hh.maxabs(got["pseudo_normal"], plain["pseudo_normal"]) < 5e-3


# ---- 3. gradients -------------------------------------------------------------------------------------------------------------------
def _rows(got, want, what):
    g, w = got.double().cpu().reshape(want.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    d, n = (g - w).norm(dim=1), w.norm(dim=1)
    if float(n.max()) == 0.0:
        assert float(d.max()) == 0.0, what
        return
    assert bool((d <= ROW_REL * n + ROW_ABS * n.max()).all()), (what, float((d / (ROW_REL * n + ROW_ABS * n.max())).max()))
    assert float(np.median(Hh.row_errors(g, w))) <= MED, what


@pytest.mark.parametrize("M,deg", [(16, 3), (25, 2), (16, 0), (25, 1), (25, 4), (9, 2), (1, 0)])
@pytest.mark.parametrize("mode", ["camera", "directions"])
def test_kernel_backward_against_fp64(dev, M, deg, mode):
    from autovfx_b200.renderer import _SugarColors
    model = _scene(dev, M=M, grad=False)
    campos = model.nerfmodel.training_cameras.p3d_cameras[2].get_camera_center()
    dc = model._sh_coordinates_dc.detach().clone()
    rest = model._sh_coordinates_rest.detach().clone()
    dc[30:60] = -3.0  # negative pre-clamp colours
    dc[60:64], rest[60:64] = float(np.float32(-1.7724538)), 0.0  # exactly 0 before the clamp: the gradient passes
    dens = model.all_densities.detach().clone()
    for t in (dc, rest, dens):
        t.requires_grad_(True)
    pos = model._points.detach().clone()
    if mode == "directions":
        src = (torch.nn.functional.normalize(pos - campos, dim=-1) * 1.2).roll(1, dims=1).contiguous().requires_grad_(True)
        colors, op = _SugarColors.apply(src, None, dc, rest, dens, deg, True)
        dirs_np = src.detach().cpu().numpy()
    else:
        src = pos.requires_grad_(True)
        colors, op = _SugarColors.apply(src, campos, dc, rest, dens, deg, False)
        dirs_np = SC.view_dirs_np(pos.detach().cpu().numpy(), campos.cpu().numpy())
    gen = torch.Generator().manual_seed(M * 5 + deg)
    gc, go = torch.randn(colors.shape, generator=gen).to(dev), torch.randn(op.shape, generator=gen).to(dev)
    ((colors * gc).sum() + (op * go).sum()).backward()
    sh = torch.cat([dc, rest], 1).detach().cpu().numpy()
    col_np, pre = SC.colors_np(deg, sh, dirs_np)
    assert np.array_equal(colors.detach().cpu().numpy(), col_np)
    passed = (pre >= 0).astype(np.float64)
    assert deg > 0 or not passed[30:60].any()
    sh64 = torch.from_numpy(sh).double().requires_grad_(True)
    src64 = src.detach().cpu().double().requires_grad_(True)
    kw = {"directions": src64} if mode == "directions" else {"positions": src64, "campos": campos.cpu().double().reshape(1, 3)}
    SC.colors_forced(deg, sh64, torch.from_numpy(passed), **kw).backward(gc.cpu().double())
    n = (deg + 1) ** 2
    assert torch.count_nonzero(rest.grad[:, n - 1:]) == 0  # coefficients beyond the active degree
    _rows(dc.grad, sh64.grad[:, :1], "sh_dc")
    if M > 1:
        _rows(rest.grad, sh64.grad[:, 1:], "sh_rest")
    _rows(src.grad, torch.zeros_like(src64) if src64.grad is None else src64.grad, mode)
    o = torch.sigmoid(dens.detach().cpu().double())
    _rows(dens.grad, go.cpu().double() * o * (1 - o), "densities")


E2E = [("plain", 16, 3), ("plain", 25, 2), ("plain", 25, 4), ("sh_rotations", 25, 4), ("cov_python", 16, 1), ("rasterizer_sh", 25, 3),
       ("positions", 16, 2), ("depth_call", 16, 0), ("point_colors", 16, 3), ("plain", 1, 0)]


@pytest.mark.parametrize("name,M,deg", E2E)
def test_gradients_match_render_sugar_and_the_two_call_graph(dev, exact, name, M, deg):
    from autovfx_b200.renderer import render_sugar, render_sugar_raw
    w = TS._weights(dev)
    for term in ("image", "depth", "normal", "all"):
        res = {}
        for which, fn in (("ours", render_sugar_raw), ("sugar", render_sugar), ("two", SR.sugar_render_two_pass)):
            model = _scene(dev, M=M)
            out = TS._call(fn, model, name, dev, deg, **FLAGS)
            TS._loss(out, w, term).backward()
            res[which] = dict(model.grads(), viewspace_points=out["viewspace_points"].grad)
        # the same leaves receive a gradient as under render_sugar; against the two-call graph as test_gpu_sugar_render allows
        assert sorted(res["ours"]) == sorted(res["sugar"]), (name, term)
        for k in set(res["ours"]) ^ set(res["two"]):
            assert term == "normal" and k in res["ours"] and torch.count_nonzero(res["ours"][k]) == 0, (name, term, k)
        for other in ("sugar", "two"):
            for k in res[other]:
                if res[other][k].numel() == 0:  # _sh_coordinates_rest at M = 1
                    assert res["ours"][k].shape == res[other][k].shape
                    continue
                TS._assert_rows(res["ours"][k], res[other][k], (name, term, other, k))
        if term in ("image", "all") and name not in ("point_colors", "depth_call", "rasterizer_sh"):
            assert torch.count_nonzero(res["ours"]["_sh_coordinates_dc"]) > 0


def test_image_only_return_under_autograd(dev, exact):
    from autovfx_b200.renderer import render_sugar, render_sugar_raw
    w = torch.randn(TS.H, TS.W, 4, generator=torch.Generator().manual_seed(2)).to(dev)
    res = {}
    for which, fn in (("ours", render_sugar_raw), ("sugar", render_sugar)):
        model = _scene(dev, M=25)
        img = fn(model, camera_indices=3, sh_deg=4)
        assert img.requires_grad and img.shape == (TS.H, TS.W, 4)
        (img * w).sum().backward()
        res[which] = model.grads()
    assert sorted(res["ours"]) == sorted(res["sugar"])
    for k in res["sugar"]:
        TS._assert_rows(res["ours"][k], res["sugar"][k], k)


# ---- 4. edge cases ------------------------------------------------------------------------------------------------------------------
def test_empty_scene(dev):
    from autovfx_b200.renderer import render_sugar_raw
    model = _scene(dev, P=0)
    out = render_sugar_raw(model, camera_indices=0, sh_deg=3, **FLAGS)
    assert out["radii"].numel() == 0 and out["image"].shape == (TS.H, TS.W, 4) and out["colors"].shape == (0, 3)
    (out["image"].sum() + out["depth"].sum() + out["normal"].sum()).backward()
    with torch.no_grad():
        out = render_sugar_raw(model, camera_indices=0, sh_deg=3, return_opacities=True)
    assert out["radii"].numel() == 0 and out["opacities"].shape == (0, 1)


@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_everything_behind_the_camera(dev, grad):
    from autovfx_b200.renderer import render_sugar, render_sugar_raw
    cams = SR.Cameras([(3.0, 0.0, 0.5)], target=(6.0, 0.0, 0.5), device=dev)
    model = _scene(dev, grad=grad, cameras=cams)
    with torch.set_grad_enabled(grad):
        got = render_sugar_raw(model, camera_indices=0, sh_deg=3, **FLAGS)
        want = render_sugar(model, camera_indices=0, sh_deg=3, **FLAGS)
    assert int(got["radii"].count_nonzero()) == 0
    for k in ("image", "depth", "radii", "normal", "pseudo_normal"):
        assert torch.equal(got[k], want[k]), k
    if grad:
        (got["image"].sum() + got["normal"].sum()).backward()
        assert model._sh_coordinates_dc.grad is not None


def test_gaussian_at_the_camera_centre(dev):
    """F.normalize of a zero vector: the direction is 0 (finite colours), and the gradient is dL/ddir / 1e-12, as torch gives."""
    from autovfx_b200.renderer import _SugarColors
    model = _scene(dev, M=16, grad=False)
    campos = model.nerfmodel.training_cameras.p3d_cameras[0].get_camera_center()
    pos = model._points.detach().clone()
    pos[5] = campos[0]
    raw = [t.detach().clone().requires_grad_(True) for t in (model._sh_coordinates_dc, model._sh_coordinates_rest, model.all_densities)]
    p1 = pos.clone().requires_grad_(True)
    colors, _ = _SugarColors.apply(p1, campos, *raw, 3, False)
    g = torch.randn(colors.shape, generator=torch.Generator().manual_seed(4)).to(dev)
    (colors * g).sum().backward()
    ref = SC.SugarModel4.__new__(SC.SugarModel4)
    ref._points, ref._sh_coordinates_dc, ref._sh_coordinates_rest = None, *[t.detach() for t in raw[:2]]
    p2 = pos.clone().requires_grad_(True)
    want = SC.SugarModel4.get_points_rgb(ref, positions=p2, camera_centers=campos, sh_levels=4)
    (want * g).sum().backward()
    assert bool(torch.isfinite(colors).all()) and torch.equal(colors[5], want[5].detach())
    assert float(p2.grad[5].abs().max()) > 1e9
    assert float((p1.grad[5] - p2.grad[5]).norm() / p2.grad[5].norm()) <= 1e-5


def test_sh_deg_beyond_the_storage_raises(dev):
    from autovfx_b200.renderer import render_sugar_raw
    for M, deg in ((16, 4), (9, 3), (1, 1), (25, 5)):
        model = _scene(dev, M=M)
        with pytest.raises(ValueError, match="sh_deg"):
            render_sugar_raw(model, camera_indices=0, sh_deg=deg, **FLAGS)


def _mesh_scene(dev):
    from autovfx_b200 import scene
    g = scene.synthetic_gaussians(3000, seed=3, extent=(1.0, 1.0, 0.5), log_scale_mean=math.log(0.03), log_scale_std=0.5, M=25)
    g = {k: v.to(dev) for k, v in g.items()}
    return SC.MeshBoundModel(g, SR.ring_cameras(4, device=dev, principal=(0.04, -0.03)), TS.W, TS.H, TS.FOV_X)


def test_mesh_bound_model_gets_gradients_through_its_getters(dev, exact):
    from autovfx_b200.renderer import render_sugar, render_sugar_raw
    w = TS._weights(dev)
    res = {}
    for which, fn in (("ours", render_sugar_raw), ("sugar", render_sugar)):
        model = _mesh_scene(dev)
        out = fn(model, camera_indices=2, sh_deg=4, **FLAGS)
        TS._loss(out, w, "all").backward()
        res[which] = model.grads()
    assert sorted(res["ours"]) == sorted(res["sugar"])
    for k in ("_vertices", "_scale_shift", "_quat_gain", "_scales", "_quaternions", "_sh_coordinates_dc", "all_densities"):
        assert torch.count_nonzero(res["ours"][k]) > 0, k
    for k in res["sugar"]:
        TS._assert_rows(res["ours"][k], res["sugar"][k], k)
