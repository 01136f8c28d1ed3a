"""The differentiable product frame: rasterize_gaussians_multi and render() with gradients (run with -m gpu on an H100).

One autograd call renders the SH colours and a second colour set (the normals of render()) on one projection, binning, sort and
blend, and one blend backward takes the gradients of both images (gsr_backward_multi).  The graph it replaces is two
GaussianRasterizer calls on the same geometry, whose gradients autograd sums.  Checked here, in both image modes:

  1. the forward equals gsr_forward_multi and the two separate calls bit for bit, and keeps the single pass's n_contrib;
  2. every input gradient equals the two-call graph's per row within atomic-summation rounding, with the same non-zero rows,
     for each loss term alone and all together;
  3. against fp64 autograd of the two passes (tests/torch_ref.py), the GPU's per-row error stays within the CPU oracle's two
     backward passes summed;
  4. render() with gradients against the two-call graph built from GaussianRasterizer, on each of its colour/covariance paths;
  5. the empty scene, an extra image without gradient, an async-mode overflow and the C ABI's argument check.
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

pytestmark = pytest.mark.gpu

CASES = ["config1", "small_sh", "small_deg1_m25", "small_precomp", "big_splats", "dense_tile", "coplanar"]
FAMILIES = ["precomp", "M25_D2_off", "M16_D3"]  # colours and covariances precomputed; M = 25 rows 4 bytes off alignment
# the dense cases of tests/helpers.DENSE_CASES that CASES lacks: the backward's redo band, ballot block edge, top-row mask of
# partial footprints and deep termination
DENSE = ["skip_band", "faint_slab", "sort_regimes"]
TERMS = ("color", "depth", "alpha", "extra", "all")
NAMES = {"means3D": "dL_dmeans3D", "opacities": "dL_dopacity", "shs": "dL_dsh", "colors_precomp": "dL_dcolors", "scales": "dL_dscales",
         "rotations": "dL_drotations", "cov3D_precomp": "dL_dcov3D", "extra": "dL_dextra"}

# Fused against the two-call graph, per Gaussian row of every gradient tensor: ||fused - two|| <= ROW_REL ||two|| + ROW_ABS max ||two||,
# and the median of ||fused - two|| / ||two|| at most MED.  The two differ only in the order of fp32 sums (one set of atomics against
# two, whose results autograd adds).
ROW_REL = 5e-5
ROW_ABS = 1e-5
MED = 4e-6
# fused against fp64 autograd, per tensor: q50 and q99 of the per-row error within Q_FACTOR x the oracle's + Q_FLOOR
Q_FACTOR = 3.0
Q_FLOOR = 2e-6


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


def _extra(P, dev, seed=21):
    return torch.rand(P, 3, generator=torch.Generator().manual_seed(seed)).to(dev)


def _args(name, dev):
    return Hh.grad_args(name, dev) if name in Hh.GRAD_FAMILIES else Hh.dense_case(name, dev)


def _leaves(a, extra):
    """Fresh leaves for one graph; a 4-byte-offset shs keeps its offset (a view into a flat leaf)."""
    leaves, inputs = {}, {}
    for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"):
        t = a[k]
        if t is None:
            inputs[k] = None
        elif k == "shs" and t.data_ptr() % 16:
            buf = torch.zeros(t.numel() + 1, device=t.device)
            buf[1:] = t.reshape(-1)
            leaves[k] = buf.requires_grad_(True)
            inputs[k] = buf[1:].view(t.shape)
        else:
            leaves[k] = inputs[k] = t.detach().clone().requires_grad_(True)
    leaves["extra"] = inputs["extra"] = extra.detach().clone().requires_grad_(True)
    leaves["means2D"] = inputs["means2D"] = torch.zeros_like(a["means3D"], requires_grad=True)
    return leaves, inputs


def _grads(a, leaves):
    g = {}
    for k, v in leaves.items():
        if v.grad is None:
            continue
        g["dL_dmeans2D" if k == "means2D" else NAMES[k]] = (v.grad[1:].view(a[k].shape) if k == "shs" and v.dim() == 1 else v.grad).detach()
    return g


def _fused(a, extra, loss_imgs, tight=None):
    from autovfx_b200.rasterizer import rasterize_gaussians_multi
    leaves, x = _leaves(a, extra)
    out = rasterize_gaussians_multi(x["means3D"], x["means2D"], x["shs"], x["colors_precomp"], x["extra"], x["opacities"], x["scales"],
                                    x["rotations"], x["cov3D_precomp"], Hh.settings_from(a))
    if loss_imgs is not None:
        sum(((o * w).sum() for o, w in zip(out[:4], loss_imgs) if w is not None), torch.zeros((), device=extra.device)).backward()
    return out, _grads(a, leaves)


def _two_call(a, extra, loss_imgs):
    """The graph render() built before the fused call: two GaussianRasterizer calls on the same leaves."""
    from autovfx_b200.rasterizer import GaussianRasterizer
    leaves, x = _leaves(a, extra)
    rast = GaussianRasterizer(Hh.settings_from(a))
    geo = dict(opacities=x["opacities"], scales=x["scales"], rotations=x["rotations"], cov3D_precomp=x["cov3D_precomp"])
    c, d, al, radii = rast(x["means3D"], x["means2D"], shs=x["shs"], colors_precomp=x["colors_precomp"], **geo)
    e = rast(x["means3D"], x["means2D"], shs=None, colors_precomp=x["extra"], **geo)[0]
    out = (c, d, al, e, radii)
    if loss_imgs is not None:
        sum(((o * w).sum() for o, w in zip(out[:4], loss_imgs) if w is not None), torch.zeros((), device=extra.device)).backward()
    return out, _grads(a, leaves)


def _loss_imgs(a, term, dev, zeros=False):
    """Seeded gradients of the colour, depth, alpha and extra images; the images a term leaves out of the loss get None (so that
    they receive no gradient at all), or zeros."""
    dc, dd, da = Hh.image_grads(a, device=dev)
    de = Hh.extra_image_grad(a, "all", device=dev)
    keep = {"color": (1, 0, 0, 0), "depth": (0, 1, 0, 0), "alpha": (0, 0, 1, 0), "extra": (0, 0, 0, 1), "all": (1, 1, 1, 1)}[term]
    return tuple(g if k else (torch.zeros_like(g) if zeros else None) for g, k in zip((dc, dd, da, de), keep))


def _row_stats(got, want):
    """(worst row's share of its bound, median relative row error) of got against want, both [P, ...]."""
    g, w = got.double().cpu().reshape(want.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    d, n = (g - w).norm(dim=1), w.norm(dim=1)
    if float(n.max()) == 0.0:
        return (0.0 if not torch.count_nonzero(d) else math.inf), 0.0
    return float((d / (ROW_REL * n + ROW_ABS * n.max())).max()), float(np.median(Hh.row_errors(g, w)))


def assert_matches_two_call(got, want, what):
    """A tensor one side has no gradient for (an input whose image is not in the loss) must be exactly zero on the other."""
    bad = []
    for k in sorted(set(got) | set(want)):
        if k not in got or k not in want:
            if torch.count_nonzero(got[k] if k in got else want[k]):
                bad.append((k, "non-zero where the other graph has no gradient"))
            continue
        g, w = got[k], want[k]
        nz_g, nz_w = g.reshape(g.shape[0], -1).ne(0).any(dim=1), w.reshape(w.shape[0], -1).ne(0).any(dim=1)
        if not torch.equal(nz_g, nz_w):
            bad.append((k, "non-zero rows differ: %d fused only, %d two-call only" % (int((nz_g & ~nz_w).sum()), int((nz_w & ~nz_g).sum()))))
            continue
        excess, med = _row_stats(g, w)
        if excess > 1.0 or med > MED:
            bad.append((k, "worst row at %.3g of its bound, median relative error %.3g" % (excess, med)))
    assert not bad, (what, bad)


# ---- 1. forward ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("tight", [False, True], ids=["tight_off", "tight_on"])
def test_forward_equals_one_pass_and_two_calls(dev, exact, name, tight):
    from autovfx_b200 import rasterizer as R
    a = _args(name, dev)
    extra = _extra(a["means3D"].shape[0], dev)
    old = R.get_tight_tiles()
    R.set_tight_tiles(tight)
    try:
        (c, d, al, e, radii), _ = _fused(a, extra, None)
        assert c.grad_fn is not None  # a backward is pending: the forward kept its workspaces
        geom, binning, image = c.grad_fn.saved_tensors[7:10]
        n_contrib = R.debug_views((geom, binning, image), a["means3D"].shape[0], a["W"], a["H"])["n_contrib"]
        want = R.forward_multi(a["means3D"], a["shs"], a["colors_precomp"], extra, a["opacities"], a["scales"], a["rotations"],
                               a["cov3D_precomp"], Hh.settings_from(a), sync=True)
        for got, w, k in zip((c, d, al, e, radii), want[:5], ("color", "depth", "alpha", "extra", "radii")):
            assert torch.equal(got, w), k
        (c2, d2, al2, e2, radii2), _ = _two_call(a, extra, None)
        for got, w, k in zip((c, d, al, e, radii), (c2, d2, al2, e2, radii2), ("color", "depth", "alpha", "extra", "radii")):
            assert torch.equal(got, w), k
        one = Hh.run_ours(a, for_backward=True)
        assert torch.equal(n_contrib, one["views"]["n_contrib"])
    finally:
        R.set_tight_tiles(old)


# ---- 2. against the two-call graph ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES + FAMILIES + DENSE)
def test_gradients_match_the_two_call_graph(dev, exact, name):
    a = _args(name, dev)
    extra = _extra(a["means3D"].shape[0], dev)
    for term in TERMS:
        imgs = _loss_imgs(a, term, dev)
        (_, _, _, _, radii), got = _fused(a, extra, imgs)
        (_, _, _, _, radii2), want = _two_call(a, extra, imgs)
        assert torch.equal(radii, radii2)
        if term in ("color", "depth", "alpha"):
            assert "dL_dextra" not in got  # the extra image had no gradient: extra_colors gets none
            want.pop("dL_dextra", None)
        assert_matches_two_call(got, want, (name, term))


# ---- 3. against fp64 autograd of the two passes ---------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=FAMILIES)
def fp64_family(request, dev):
    """(name, a, extra, {term: fp64 gradients}, {term: the oracle's two passes summed}) for the terms 'extra' and 'all'."""
    a = Hh.grad_args(request.param, dev)
    extra = _extra(a["means3D"].shape[0], dev)
    b = Hh.extra_pass(a, extra)
    fa, fb = Hh.run_oracle(a), Hh.run_oracle(b)
    g64 = Hh.fp64_grads(a, fa, ("extra", "all"), extra=(b, fb))
    orc = {term: Hh.oracle_two_pass_grads(a, fa, b, fb, *(t.cpu() for t in _loss_imgs(a, term, dev, zeros=True))) for term in ("extra", "all")}
    return request.param, a, extra, g64, orc


@pytest.mark.parametrize("term", ["extra", "all"])
def test_gradients_against_fp64_two_passes(fp64_family, exact, term):
    name, a, extra, g64, orc = fp64_family
    dev = a["means3D"].device
    (_, _, _, _, radii), got = _fused(a, extra, _loss_imgs(a, term, dev))
    got = Hh.comparable_grads({k: v.cpu() for k, v in got.items()}, a)
    checked = 0
    for k, want in g64[term].items():
        if k not in got:
            continue
        if float(want.abs().max()) == 0.0:
            assert float(got[k].abs().max()) == 0.0, k
            continue
        e_gpu, e_orc = Hh.row_errors(got[k], want), Hh.row_errors(orc[term][k], want)
        for q in (0.5, 0.99):
            g, base = float(np.quantile(e_gpu, q)), float(np.quantile(e_orc, q))
            assert g <= Q_FACTOR * base + Q_FLOOR, "%s %s %s: q%g per-row error %.3g, oracle %.3g" % (name, term, k, 100 * q, g, base)
        checked += 1
    assert checked >= 5 and "dL_dextra" in got
    assert float(a["bg"].abs().max()) > 0  # the background term of both images is exercised


# ---- 4. render() with gradients -----------------------------------------------------------------------------------------------
class _PC:
    """Duck-typed GaussianModel with every activated parameter a leaf (scene/gaussian_model.py)."""

    def __init__(self, g, sh_degree, max_sh_degree=3):
        self._xyz, self._scales, self._rot, self._op, self._shs = (g[k].detach().clone().requires_grad_(True) for k in
                                                                   ("means3D", "scales", "rotations", "opacities", "shs"))
        self.active_sh_degree, self.max_sh_degree = sh_degree, max_sh_degree

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: s._scales)
    get_rotation = property(lambda s: s._rot)
    get_opacity = property(lambda s: s._op)
    get_features = property(lambda s: s._shs)

    def get_covariance(self, mod):
        return Hh.cov3d_from(self._scales, self._rot, mod)

    def get_normal(self, dir_pp_normalized=None):
        n, _ = WR.flip_align_view(WR.get_minimum_axis(self._scales, self._rot), dir_pp_normalized)
        return n / n.norm(dim=1, keepdim=True)


def _cam(cam, dev):
    return types.SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy), image_height=cam.image_height,
                                 image_width=cam.image_width, world_view_transform=cam.world_view_transform.to(dev),
                                 full_proj_transform=cam.full_proj_transform.to(dev), camera_center=cam.camera_center.to(dev))


def _render_two_call(cam, pc, pipe, bg, override_color=None):
    """render() with gradients as the reference writes it (GR/:83-218): two GaussianRasterizer calls, torch ops around them."""
    from autovfx_b200 import renderer
    from autovfx_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    xyz = pc.get_xyz
    means2D = torch.zeros_like(xyz, requires_grad=True) + 0
    means2D.retain_grad()
    H, W = int(cam.image_height), int(cam.image_width)
    s = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
                                      bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                                      sh_degree=pc.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False)
    rast = GaussianRasterizer(s)
    scales = rotations = cov3D = None
    if pipe.compute_cov3D_python:
        cov3D = pc.get_covariance(1.0)
    else:
        scales, rotations = pc.get_scaling, pc.get_rotation
    dir_pp = xyz - cam.camera_center.repeat(pc.get_features.shape[0], 1)
    dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
    shs = colors = None
    if override_color is not None:
        colors = override_color
    elif pipe.convert_SHs_python:
        shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
        colors = torch.clamp_min(renderer._eval_sh_torch(pc.active_sh_degree, shs_view, dir_pp_normalized) + 0.5, 0.0)
    else:
        shs = pc.get_features
    geo = dict(opacities=pc.get_opacity, scales=scales, rotations=rotations, cov3D_precomp=cov3D)
    img, depth, alpha, radii = rast(xyz, means2D, shs=shs, colors_precomp=colors, **geo)
    nn = pc.get_normal(dir_pp_normalized=dir_pp_normalized) * 0.5 + 0.5
    nimg = rast(xyz, means2D, shs=None, colors_precomp=nn, **geo)[0]
    depth = depth.squeeze(0)
    return {"render": torch.cat((img, alpha), 0), "depth": depth, "normal": WR.normal_image(nimg),
            "pseudo_normal": WR.pseudo_normal(depth, cam.world_view_transform, cam.FoVx, cam.FoVy), "viewspace_points": means2D,
            "radii": radii}


@pytest.mark.parametrize("path", ["plain", "convert_SHs_python", "compute_cov3D_python", "override_color"])
def test_render_with_gradients_matches_the_two_call_graph(dev, exact, path):
    from autovfx_b200 import renderer
    case = Hh.case_inputs("small_sh")
    g = {k: v.to(dev) for k, v in case["g"].items()}
    cam = _cam(case["cam"], dev)
    bg = torch.tensor(case["bg"], device=dev)
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=path == "compute_cov3D_python",
                                 convert_SHs_python=path == "convert_SHs_python")
    gen = torch.Generator().manual_seed(5)
    H, W = cam.image_height, cam.image_width
    w = {"render": torch.randn(4, H, W, generator=gen), "depth": torch.randn(H, W, generator=gen),
         "normal": torch.randn(H, W, 3, generator=gen), "pseudo_normal": torch.randn(H, W, 3, generator=gen)}
    w = {k: v.to(dev) for k, v in w.items()}
    res = {}
    for which in ("fused", "two"):
        pc = _PC(g, case["sh_degree"])
        override = None
        if path == "override_color":
            override = (torch.rand(g["means3D"].shape[0], 3, generator=torch.Generator().manual_seed(3)).to(dev)).requires_grad_(True)
        out = renderer.render(cam, pc, pipe, bg, override_color=override) if which == "fused" else _render_two_call(cam, pc, pipe, bg, override)
        sum((out[k] * w[k]).sum() for k in w).backward()
        grads = {"xyz": pc._xyz.grad, "scaling": pc._scales.grad, "rotation": pc._rot.grad, "opacity": pc._op.grad,
                 "viewspace_points": out["viewspace_points"].grad}
        if path != "override_color":
            grads["features"] = pc._shs.grad
        else:
            grads["override_color"] = override.grad
        res[which] = (out, grads)
    (fo, fg), (to, tg) = res["fused"], res["two"]
    for k in ("render", "depth", "normal"):
        assert fo[k].shape == to[k].shape and torch.equal(fo[k], to[k]), k
    assert Hh.maxabs(fo["pseudo_normal"], to["pseudo_normal"]) < 5e-3
    assert torch.equal(fo["radii"], to["radii"]) and torch.equal(fo["visibility_filter"], to["radii"] > 0)
    assert all(v is not None for v in fg.values()) and all(v is not None for v in tg.values())
    assert_matches_two_call({k: v.detach() for k, v in fg.items()}, {k: v.detach() for k, v in tg.items()}, path)


# ---- 5. edge cases --------------------------------------------------------------------------------------------------------------
def test_empty_scene_gives_empty_gradients(dev):
    from autovfx_b200.rasterizer import rasterize_gaussians_multi
    a = Hh.resolve(Hh.case_inputs("small_sh"), dev)
    z = lambda *s: torch.zeros(*s, device=dev, requires_grad=True)  # noqa: E731
    x = dict(means3D=z(0, 3), means2D=z(0, 3), shs=z(0, 16, 3), extra=z(0, 3), opacities=z(0, 1), scales=z(0, 3), rotations=z(0, 4))
    c, d, al, e, radii = rasterize_gaussians_multi(x["means3D"], x["means2D"], x["shs"], None, x["extra"], x["opacities"], x["scales"],
                                                   x["rotations"], None, Hh.settings_from(a))
    assert radii.numel() == 0 and float(e.abs().max()) == 0.0
    (c.sum() + d.sum() + al.sum() + e.sum()).backward()
    for k, v in x.items():
        assert v.grad is not None and v.grad.shape == v.shape, k


def test_extra_image_without_gradient_takes_the_plain_backward(dev, monkeypatch):
    from autovfx_b200 import rasterizer as R
    a = Hh.resolve(Hh.case_inputs("small_sh"), dev)
    extra = _extra(a["means3D"].shape[0], dev)
    calls = []
    for fn in ("gsr_backward", "gsr_backward_multi"):
        real = getattr(R._L, fn)
        monkeypatch.setattr(R._L, fn, lambda *args, _f=fn, _r=real: calls.append(_f) or _r(*args))
    dc, dd, da = Hh.image_grads(a, device=dev)
    (_, _, _, e, _), got = _fused(a, extra, (dc, dd, da, None))
    assert calls == ["gsr_backward"] and "dL_dextra" not in got and e.requires_grad
    calls.clear()
    _fused(a, extra, (None, None, None, torch.ones_like(e)))
    assert calls == ["gsr_backward_multi"]


def test_async_overflow_raises_like_the_single_pass(dev):
    from autovfx_b200 import rasterizer as R
    a = Hh.resolve(Hh.case_inputs("config1"), dev)
    extra = _extra(a["means3D"].shape[0], dev)
    st = R._state(dev)
    old = st.capacity
    errors = []
    try:
        R.set_sync_mode("async")
        st.ensure_capacity = lambda P, W=0, H=0: None  # keep a capacity far below R = 41671
        for run in (_fused, _two_call):
            st.capacity = 1000
            with pytest.raises(RuntimeError, match="overflowed its binning buffer") as ex:
                run(a, extra, _loss_imgs(a, "all", dev))
            errors.append(str(ex.value))
    finally:
        R.set_sync_mode("safe")
        del st.ensure_capacity
        st.capacity = max(old, st.capacity)
    assert errors[0] == errors[1]


def test_partly_null_extra_arguments_are_rejected(dev):
    import ctypes as C
    from autovfx_b200 import _lib
    from autovfx_b200 import rasterizer as R
    a = Hh.resolve(Hh.case_inputs("small_sh"), dev)
    P, H, W = a["means3D"].shape[0], a["H"], a["W"]
    extra = _extra(P, dev)
    o = R.forward_raw(a["means3D"], a["shs"], None, a["opacities"], a["scales"], a["rotations"], None, Hh.settings_from(a),
                      for_backward=True, sync=True, extra=extra, extra_out=torch.empty(3, H, W, device=dev))
    color, depth, alpha, radii, (geom, binning, image), _, keep = o
    fr = _lib.gsr_frame()
    R._fill_frame(fr, P, a["sh_degree"], a["shs"].shape[1], W, H, Hh.settings_from(a), keep[7], keep[0], keep[1], None, None, keep[4],
                  keep[5], None, keep[8], keep[9], keep[10])
    ws = _lib.gsr_workspace(geom.data_ptr(), geom.numel(), binning.data_ptr(), binning.numel(), image.data_ptr(), image.numel())
    f = lambda *s: torch.empty(*s, device=dev)  # noqa: E731
    bufs = dict(m2=f(P, 3), co=f(P, 4), op=f(P), col=f(P, 3), dep=f(P), m3=f(P, 3), cov=f(P, 6), sh=f(P, 16, 3), sc=f(P, 3), rot=f(P, 4))
    gr = _lib.gsr_grads(*(t.data_ptr() for t in bufs.values()))
    dc, dd, da = Hh.image_grads(a, device=dev)
    de, dx = torch.randn(3, H, W, device=dev), torch.full((P, 3), float("nan"), device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def call(e, g, d):
        return _lib.lib.gsr_backward_multi(C.byref(fr), C.byref(ws), radii.data_ptr(), alpha.data_ptr(), dc.data_ptr(), dd.data_ptr(),
                                           da.data_ptr(), e, g, d, C.byref(gr), stream)
    for e, g, d in ((extra.data_ptr(), None, None), (None, de.data_ptr(), dx.data_ptr()), (extra.data_ptr(), de.data_ptr(), None)):
        assert call(e, g, d) == -1  # GSR_ERR_INVALID
        assert b"all given or all NULL" in _lib.lib.gsr_last_error()
    assert torch.isnan(dx).all()  # a rejected call writes nothing
    assert call(extra.data_ptr(), de.data_ptr(), dx.data_ptr()) == 0
    torch.cuda.synchronize(dev)
    assert torch.isfinite(dx).all() and torch.count_nonzero(dx[radii == 0]) == 0 and torch.count_nonzero(dx) > 0
