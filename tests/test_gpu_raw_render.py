"""render_raw(): render() from a GaussianModel's raw parameters, with the activations, the shading normals and their backward in
CUDA (gsr_activate_gaussians, gsr_axis_normals, gsr_activate_gaussians_backward).  Run with -m gpu on an H100.  Checked here,
in both image modes:

  1. the forward equals render() bit for bit on a model whose getters return the same kernels' activated tensors;
  2. the raw gradients against torch fp64 autograd of exp / F.normalize / sigmoid / cat / get_normal * 0.5 + 0.5, fed the
     activated-space gradients of the same backward, with the axis and flip forced to the kernel's;
  3. end to end against the reference graph: render() on raw leaves with torch activations and the reference get_normal;
  4. the empty scene, M = 1, override_color, a loss without the normal image, SH coefficients beyond the active degree and
     isotropic Gaussians.
"""
import math
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402
from tests import wrapper_ref as WR  # noqa: E402
from tests.test_gpu_fused_grads import _cam  # noqa: E402
from tests.test_raw_render_cpu import fp64_autograd  # noqa: E402

pytestmark = pytest.mark.gpu

NAMED = ["small_sh", "small_deg1_m25", "big_splats", "dense_tile", "coplanar", "config1"]
FAMILIES = ["M1_D0", "M4_D1", "M9_D2", "M16_D3", "M25_D3", "M25_D2_off"]  # M25_D2_off: _features_rest rows 4 bytes off alignment
TERMS = ("color", "depth", "alpha", "normal", "all")
RAW = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
# GPU against fp64 autograd, per Gaussian row: ||gpu - fp64|| <= ROW_REL ||fp64|| + ROW_ABS max ||fp64||, median relative error <= MED
ROW_REL, ROW_ABS, MED = 1e-5, 1e-7, 2e-6
# render_raw against the reference graph end to end, same form.  The activated inputs of the two rasterizer calls differ by up to one
# rounding (sigmoid, normalize), which the blend backward amplifies on big_splats (median 1.35e-5 on _features_rest, whose own
# backward is a copy) and config1 (worst _xyz row 1.74x test_gpu_fused_grads.py's bound): 2x its per-row and 5x its median bound.
E2E_ROW_REL, E2E_ROW_ABS, E2E_MED = 1e-4, 2e-5, 2e-5
PIPE = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)


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


def _case(name, dev, tiny=0, ties=False):
    """(raw float32 parameters, camera, bg, active degree, shs offset) of a named case or gradient family.  Quaternion norms are
    spread over 0.1..10; `tiny` rows are scaled below F.normalize's 1e-12 clamp.  `ties`: 8 isotropic rows, and 32 rows whose two
    smallest log-scales differ by one ulp at |log-scale| < 0.5, where exp may round them to equal scales."""
    if name in Hh.GRAD_FAMILIES:
        a, offset = Hh.grad_args(name, dev), Hh.GRAD_FAMILIES[name][2]
        g = dict(means3D=a["means3D"], scales=a["scales"], rotations=a["rotations"], opacities=a["opacities"], shs=a["shs"])
        cam = types.SimpleNamespace(FoVx=2 * math.atan(a["tanfovx"]), FoVy=2 * math.atan(a["tanfovy"]), image_height=a["H"],
                                    image_width=a["W"], world_view_transform=a["view"], full_proj_transform=a["proj"],
                                    camera_center=a["campos"])
        bg, D, mod = a["bg"], a["sh_degree"], a["scale_modifier"]
    else:
        c = Hh.case_inputs(name)
        g, cam, bg, D, mod, offset = c["g"], _cam(c["cam"], dev), torch.tensor(c["bg"], device=dev), c["sh_degree"], c["scale_modifier"], False
    gen = torch.Generator().manual_seed(len(name) + 7 * tiny)
    P = g["means3D"].shape[0]
    scaling = torch.log(g["scales"].detach().cpu().double())
    if ties:
        c0 = -0.05 - 0.4 * torch.rand(32, generator=gen, dtype=torch.float64)
        lo = torch.from_numpy(np.nextafter(c0.float().numpy(), np.float32(-np.inf))).double()
        scaling[tiny:tiny + 32] = torch.stack((c0.float().double(), lo, c0 + 0.5), -1)
        scaling[tiny + 32:tiny + 40] = scaling[tiny + 32:tiny + 40, :1]
    q = g["rotations"].detach().cpu() * (10.0 ** (torch.rand(P, generator=gen) * 2 - 1))[:, None]
    q[:tiny] *= 1e-14
    op = g["opacities"].detach().cpu().double().clamp(1e-4, 1 - 1e-4)
    shs = g["shs"].detach().cpu().contiguous()
    raw = {"_xyz": g["means3D"].detach().cpu(), "_features_dc": shs[:, :1], "_features_rest": shs[:, 1:], "_opacity": torch.log(op / (1 - op)),
           "_scaling": scaling, "_rotation": q}
    raw = {k: v.float().contiguous().to(dev) for k, v in raw.items()}
    return raw, cam, bg.to(dev), D, mod, offset


class _RawPC:
    """The reference GaussianModel's raw fields as leaves (``_features_rest`` optionally a view 4 bytes into a flat leaf)."""

    def __init__(self, raw, D, offset=False, grad=True):
        self.leaves = {}
        for k, v in raw.items():
            if k == "_features_rest" and offset:
                buf = torch.zeros(v.numel() + 1, device=v.device)
                buf[1:] = v.reshape(-1)
                self.leaves[k] = buf.requires_grad_(grad)
                setattr(self, k, buf[1:].view(v.shape))
            else:
                self.leaves[k] = v.detach().clone().requires_grad_(grad)
                setattr(self, k, self.leaves[k])
        self.scaling_activation, self.opacity_activation = torch.exp, torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize
        self.active_sh_degree, self.max_sh_degree = D, 4

    def grads(self):
        out = {}
        for k, v in self.leaves.items():
            if v.grad is not None:
                out[k] = v.grad[1:].view(getattr(self, k).shape) if v.dim() == 1 else v.grad
        return out


class _TorchPC(_RawPC):
    """The reference graph: torch activations of the raw leaves and the reference get_normal (scene/gaussian_model.py:95-128)."""
    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def get_normal(self, dir_pp_normalized=None):
        n, _ = WR.flip_align_view(WR.get_minimum_axis(self.get_scaling, self.get_rotation), dir_pp_normalized)
        return n / n.norm(dim=1, keepdim=True)


class _DuckPC:
    """Getters return edit.activate's tensors of the raw parameters and get_normal returns axis_normals: the kernels render_raw
    runs, called one by one."""

    def __init__(self, raw, D, campos, grad):
        from autovfx_b200 import edit
        act = edit.activate({k[1:].replace("features_", "f_"): v.detach() for k, v in raw.items()})
        self.act = {k: v.requires_grad_(grad) for k, v in act.items()}
        self.campos, self.active_sh_degree, self.max_sh_degree = campos, D, 4

    get_xyz = property(lambda s: s.act["means3D"])
    get_scaling = property(lambda s: s.act["scales"])
    get_rotation = property(lambda s: s.act["rotations"])
    get_opacity = property(lambda s: s.act["opacities"])
    get_features = property(lambda s: s.act["shs"])

    def get_normal(self, dir_pp_normalized=None):
        from autovfx_b200.renderer import axis_normals
        return axis_normals(self.act["means3D"], self.act["scales"], self.act["rotations"], self.campos, remap01=False)


def _weights(cam, dev, seed=5):
    gen = torch.Generator().manual_seed(seed)
    H, W = int(cam.image_height), int(cam.image_width)
    w = {"color": torch.randn(3, H, W, generator=gen), "alpha": torch.randn(H, W, generator=gen), "depth": torch.randn(H, W, generator=gen),
         "normal": torch.randn(H, W, 3, generator=gen)}
    return {k: v.to(dev) for k, v in w.items()}


def _loss(out, w, term):
    parts = {"color": (out["render"][:3] * w["color"]).sum(), "alpha": (out["render"][3] * w["alpha"]).sum(),
             "depth": (out["depth"] * w["depth"]).sum(), "normal": (out["normal"] * w["normal"]).sum()}
    return sum(parts.values()) if term == "all" else parts[term]


def _capture(monkeypatch):
    """Record the activated-space gradients render_raw's activation Function receives in its backward."""
    from autovfx_b200 import renderer
    seen = []
    real = renderer._ActivateRaw.backward

    def bw(ctx, *g):
        seen.append(tuple(None if t is None else t.detach().clone() for t in g))
        return real(ctx, *g)
    monkeypatch.setattr(renderer._ActivateRaw, "backward", staticmethod(bw))
    return seen


def _decisions(raw, campos):
    """The kernel's axis (smallest activated scale, lowest index on ties) and flip sign, read from its own outputs."""
    from autovfx_b200 import edit
    from autovfx_b200.renderer import axis_normals
    act = edit.activate({k[1:].replace("features_", "f_"): v.detach() for k, v in raw.items()})
    s = act["scales"]
    k = torch.where(s[:, 1] < s[:, 0], 1, 0)
    k = torch.where(s[:, 2] < torch.minimum(s[:, 0], s[:, 1]), 2, k)
    n = axis_normals(act["means3D"], s, act["rotations"], campos)
    col = WR.build_rotation(act["rotations"])[torch.arange(s.shape[0], device=s.device), :, k]
    sgn = torch.where((n * col).sum(-1) >= 0, 1.0, -1.0)
    return act, k.cpu().numpy(), sgn.double().cpu().numpy()


def _assert_rows(got, want, what, rel=ROW_REL, abs_=ROW_ABS, med_max=MED):
    g, w = got.double().cpu().reshape(want.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    d, n = (g - w).norm(dim=1), w.norm(dim=1)
    if float(n.max()) == 0.0:
        assert float(d.max()) == 0.0, what
        return
    excess = float((d / (rel * n + abs_ * n.max())).max())
    med = float(np.median(Hh.row_errors(g, w)))
    assert excess <= 1.0 and med <= med_max, (what, "worst row at %.3g of its bound, median relative error %.3g" % (excess, med))


def _assert_e2e(got, want, what):
    """Same gradient tensors, the same non-zero rows, and every tensor within the end-to-end bounds."""
    assert sorted(got) == sorted(want), what
    for k in got:
        g, w = got[k].detach(), want[k].detach()
        assert torch.equal(g.reshape(g.shape[0], -1).ne(0).any(1), w.reshape(w.shape[0], -1).ne(0).any(1)), (what, k, "non-zero rows differ")
        _assert_rows(g, w, (what, k), E2E_ROW_REL, E2E_ROW_ABS, E2E_MED)


# ---- 1. forward identity with the kernels called one by one ------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMED + FAMILIES)
@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
def test_forward_equals_render_on_the_activated_model(dev, exact, name, grad):
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, offset = _case(name, dev, tiny=3)
    with torch.set_grad_enabled(grad):
        got = renderer.render_raw(cam, _RawPC(raw, D, offset, grad), PIPE, bg, scaling_modifier=mod)
        want = renderer.render(cam, _DuckPC(raw, D, cam.camera_center, grad), PIPE, bg, scaling_modifier=mod)
    assert got["render"].requires_grad == grad
    for k in ("render", "depth", "normal", "pseudo_normal", "radii", "visibility_filter"):
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), (name, k)
    assert int(got["radii"].gt(0).sum()) > 0


# ---- 2. raw gradients against fp64 autograd -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small_sh", "small_deg1_m25", "coplanar", "M1_D0", "M16_D3", "M25_D2_off"])
def test_raw_gradients_against_fp64(dev, exact, name, monkeypatch):
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, offset = _case(name, dev, tiny=4, ties=True)
    assert float(bg.abs().max()) > 0
    act, k, sgn = _decisions(raw, cam.camera_center)
    sc = raw["_scaling"][4:36]
    equal = (act["scales"][4:36, 0] == act["scales"][4:36, 1]) & (sc[:, 1] < sc[:, 0])
    assert int(equal.sum()) >= 4  # rows where the raw scales and the activated scales pick different axes
    assert (k[4:36][equal.cpu().numpy()] == 0).all() and (k[36:44] == 0).all()
    assert (sgn > 0).any() and (sgn < 0).any()
    w = _weights(cam, dev)
    seen = _capture(monkeypatch)
    for term in TERMS:
        seen.clear()
        pc = _RawPC(raw, D, offset)
        _loss(renderer.render_raw(cam, pc, PIPE, bg, scaling_modifier=mod), w, term).backward()
        got = pc.grads()
        (g_sh, g_o, g_s, g_r, g_e), = seen
        assert (g_e is not None) == (term in ("normal", "all"))
        rawd = {k_[1:].replace("features_", "f_"): v.detach().double().cpu().numpy() for k_, v in raw.items()}
        grads = {"g_s": g_s.double().cpu().numpy(), "g_r": g_r.double().cpu().numpy(), "g_o": g_o.double().cpu().numpy(),
                 "g_sh": g_sh.double().cpu().numpy(), "g_e": None if g_e is None else g_e.double().cpu().numpy()}
        want = fp64_autograd(rawd, cam.camera_center.double().cpu().numpy(), grads, k, sgn)
        for ours, theirs in (("_scaling", "d_scaling"), ("_rotation", "d_rotation"), ("_opacity", "d_opacity"), ("_features_dc", "d_f_dc"),
                             ("_features_rest", "d_f_rest")):
            if want[theirs].numel():  # the rows below the clamp (gradients ~1e12 larger) apart from the rest
                _assert_rows(got[ours][4:], want[theirs][4:], (name, term, ours))
                _assert_rows(got[ours][:4], want[theirs][:4], (name, term, ours, "clamped rows"))
        assert torch.count_nonzero(got["_rotation"][:4]) > 0  # the clamped rows carry (large) gradients


# ---- 3. end to end against the reference graph -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMED + ["M25_D2_off", "M1_D0"])
def test_matches_the_reference_graph(dev, exact, name):
    from autovfx_b200 import rasterizer as R, renderer
    raw, cam, bg, D, mod, offset = _case(name, dev)
    w = _weights(cam, dev)
    res = {}
    for which in ("raw", "torch"):
        pc = _RawPC(raw, D, offset) if which == "raw" else _TorchPC(raw, D, offset)
        out = (renderer.render_raw if which == "raw" else renderer.render)(cam, pc, PIPE, bg, scaling_modifier=mod)
        node = out["depth"].grad_fn.next_functions[0][0]
        n_contrib = R.debug_views(node.saved_tensors[7:10], raw["_xyz"].shape[0], int(cam.image_width), int(cam.image_height))["n_contrib"]
        _loss(out, w, "all").backward()
        res[which] = (out, n_contrib.clone(), pc.grads())
    (ro, rn, rg), (to, tn, tg) = res["raw"], res["torch"]
    assert torch.equal(ro["radii"], to["radii"]), name
    assert torch.equal(rn, tn), name
    for k in ("render", "depth", "normal"):
        assert Hh.maxabs(ro[k], to[k]) <= 1e-5, (name, k, Hh.maxabs(ro[k], to[k]))
    assert sorted(rg) == sorted(RAW)
    _assert_e2e(rg, tg, name)


# ---- 4. edge cases --------------------------------------------------------------------------------------------------------------
def test_empty_scene(dev):
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, _ = _case("small_sh", dev)
    pc = _RawPC({k: v[:0] for k, v in raw.items()}, D)
    out = renderer.render_raw(cam, pc, PIPE, bg)
    assert out["radii"].numel() == 0
    (out["render"].sum() + out["depth"].sum() + out["normal"].sum()).backward()
    for k, v in pc.leaves.items():
        assert v.grad is None or v.grad.shape == v.shape, k


def test_override_color_gives_no_sh_gradient(dev, exact):
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, _ = _case("small_sh", dev)
    w = _weights(cam, dev)
    colors = torch.rand(raw["_xyz"].shape[0], 3, generator=torch.Generator().manual_seed(3)).to(dev)
    res = {}
    for which in ("raw", "torch"):
        pc = _RawPC(raw, D) if which == "raw" else _TorchPC(raw, D)
        ov = colors.clone().requires_grad_(True)
        out = (renderer.render_raw if which == "raw" else renderer.render)(cam, pc, PIPE, bg, override_color=ov)
        _loss(out, w, "all").backward()
        res[which] = (out, dict(pc.grads(), override=ov.grad))
    (ro, rg), (to, tg) = res["raw"], res["torch"]
    assert "_features_dc" not in rg and "_features_rest" not in rg
    assert torch.equal(ro["radii"], to["radii"])
    tg.pop("_features_dc", None), tg.pop("_features_rest", None)
    _assert_e2e(rg, tg, "override_color")


def test_loss_without_the_normal_image(dev, monkeypatch):
    """The normal image gets no gradient: the rotation gradient is F.normalize's Jacobian of the covariance path's alone."""
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, _ = _case("small_sh", dev, tiny=3)
    seen = _capture(monkeypatch)
    pc = _RawPC(raw, D)
    out = renderer.render_raw(cam, pc, PIPE, bg)
    (out["render"].sum() + out["depth"].sum()).backward()
    (_, _, _, g_r, g_e), = seen
    assert g_e is None
    rho = raw["_rotation"].double()
    n = rho.norm(dim=1, keepdim=True)
    r = rho / n.clamp_min(1e-12)
    g = g_r.double()
    want = torch.where(n >= 1e-12, (g - r * (r * g).sum(-1, keepdim=True)) / n, g / 1e-12)
    _assert_rows(pc.grads()["_rotation"], want, "rotation without normals")


def test_sh_gradient_is_zero_beyond_the_active_degree(dev):
    from autovfx_b200 import renderer
    raw, cam, bg, D, mod, offset = _case("M25_D2_off", dev)
    assert D == 2
    pc = _RawPC(raw, D, offset)
    _loss(renderer.render_raw(cam, pc, PIPE, bg, scaling_modifier=mod), _weights(cam, dev), "all").backward()
    g = pc.grads()["_features_rest"]
    assert g.shape == (raw["_xyz"].shape[0], 24, 3)
    assert torch.count_nonzero(g[:, 8:]) == 0 and torch.count_nonzero(g[:, :8]) > 0


def test_isotropic_rows_pick_the_lowest_axis(dev):
    """create_from_pcd leaves every Gaussian isotropic (three equal scales).  The kernels' rule, shared with gsr_axis_normals since
    it was written, is the lowest index: column 0, in the forward and in the backward.  torch.argsort on the GPU, which the
    reference's get_minimum_axis calls, is not stable: on an H100 it returned index 2 for every isotropic row of this case, so the
    reference shades such Gaussians with another axis than gsr_axis_normals does.  That difference predates render_raw and is
    left as it is."""
    from autovfx_b200 import edit, renderer
    from autovfx_b200.renderer import axis_normals
    raw, cam, bg, D, mod, _ = _case("small_sh", dev)
    raw["_scaling"] = raw["_scaling"][:, :1].expand(-1, 3).contiguous()
    act = edit.activate({k[1:].replace("features_", "f_"): v for k, v in raw.items()})
    assert torch.equal(act["scales"][:, 0], act["scales"][:, 1]) and torch.equal(act["scales"][:, 0], act["scales"][:, 2])
    n = axis_normals(act["means3D"], act["scales"], act["rotations"], cam.camera_center)
    col0 = WR.build_rotation(act["rotations"])[:, :, 0]
    assert Hh.maxabs(n.abs(), col0.abs()) <= 1e-6
    _, k, _ = _decisions(raw, cam.camera_center)
    assert (k == 0).all()
    # the backward differentiates through the same column: the normal image's gradient reaches _rotation
    pc = _RawPC(raw, D)
    out = renderer.render_raw(cam, pc, PIPE, bg)
    (out["normal"] * _weights(cam, dev)["normal"]).sum().backward()
    assert torch.count_nonzero(pc.grads()["_rotation"]) > 0
