"""The trainers' remaining loss terms in CUDA on an H100, run with -m gpu: autovfx_b200.losses.depth_loss / opacity_loss /
sparsity_loss / entropy_loss and autovfx_b200.sugar_field.density_estimation_loss.  Every value and every gradient element is held
to the per-element float32 error bound tests/loss_terms_ref.py derives around its fp64 restatement, and the reference lines' own
float32 torch graph (restated below) is held to the same bound.  Also: the edge cases of each term, bit-identical repeats (with
and without torch.use_deterministic_algorithms), no host synchronisation in the objectives that use them, and the torch lines'
synchronisations that the drop-ins remove."""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import loss_terms_ref as TR  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import losses  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


# -- the reference lines in float32 torch ------------------------------------------------------------------------------------------
def torch_depth_loss(network_output, gt, scene_scale=5.0):
    """loss_utils.depth_loss and compute_scale_and_shift (LU/:65-111), its det == 0 branch left out."""
    network_output = network_output.view(-1)
    gt = gt.view(-1)
    depth_2d = gt / 25
    mask = depth_2d > 0
    weight = torch.zeros_like(depth_2d)
    weight[mask] = 1.
    prediction, target = network_output[mask].detach(), depth_2d[mask]
    a_00 = torch.sum(prediction * prediction)
    a_01 = torch.sum(prediction)
    a_11 = torch.sum(torch.ones_like(prediction))
    b_0 = torch.sum(prediction * target)
    b_1 = torch.sum(target)
    det = a_00 * a_11 - a_01 * a_01
    if det != 0:
        x_0 = (a_11 * b_0 - a_01 * b_1) / det
        x_1 = (-a_01 * b_0 + a_00 * b_1) / det
    else:
        raise ZeroDivisionError("det == 0")
    return torch.mean(weight * torch.exp(-network_output.detach() / scene_scale) * (x_0 * network_output + x_1 - depth_2d) ** 2)


def torch_opacity_loss(network_output):
    return torch.mean(network_output)


def torch_sparsity_loss(network_output):
    val = torch.clamp(network_output, 1e-3, 1 - 1e-3)
    return torch.mean(torch.log(val) + torch.log(1 - val))


def torch_entropy(opacities, radii):
    visibility_filter = radii > 0
    vis_opacities = opacities[visibility_filter]
    return (- vis_opacities * torch.log(vis_opacities + 1e-10) - (1 - vis_opacities) * torch.log(1 - vis_opacities + 1e-10)).mean()


def torch_density(densities, beta, sdf_estimation, squared=False):
    target_densities = torch.exp(-0.5 * sdf_estimation.pow(2) / beta.pow(2))
    return ((densities - target_densities).pow(2) if squared else (densities - target_densities).abs()).mean()


def _run(fn, leaves, *rest):
    """(value, gradients) of fn on fresh leaves."""
    ls = [t.detach().clone().requires_grad_(True) for t in leaves]
    v = fn(*ls, *rest)
    v.backward()
    return v.detach(), [t.grad for t in ls]


def _assert_within(got, want, bound, what):
    err = (got.double() - want.double()).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), float((err / bound.clamp_min(1e-300)).max()))


def _value_within(got, want, bound, what):
    assert abs(float(got) - float(want)) <= bound, (what, float(got) - float(want), bound)


def _same_bits(a, b):
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


# -- depth_loss -----------------------------------------------------------------------------------------------------------------
def _depth_case(kind, dev):
    gen = torch.Generator().manual_seed(len(kind))
    H, W = (1080, 1920) if kind == "1080p" else (480, 640)
    if kind == "near_flat":
        p = 1.0 + 0.05 * torch.rand(H, W, generator=gen)
    else:
        p = 1.0 + 4.0 * torch.rand(H, W, generator=gen)
    # omnidata-like monocular depth: an affine image of the render with noise, half of it missing (0)
    gt = 25 * (0.3 * p + 0.2 + 0.05 * torch.randn(H, W, generator=gen)).clamp_min(0.01)
    gt[torch.rand(H, W, generator=gen) < 0.5] = 0.0
    frame = torch.rand(H, W, 5, generator=gen)  # the render's depth as a strided channel of a frame
    frame[..., 4] = p
    return frame.to(dev)[..., 4], gt.to(dev).unsqueeze(0)


@pytest.mark.parametrize("kind", ["1080p", "near_flat"])
def test_depth_loss_values_and_gradients(dev, kind):
    from autovfx_b200 import losses as L
    p, gt = _depth_case(kind, dev)
    r = TR.depth64(p, gt, 5.0)
    assert r["cond"] < 0.5, r["cond"]
    if kind == "near_flat":  # the fit really is ill-conditioned: the sums' errors are amplified by about 1e3 in det
        assert r["cond"] > 1e3 * TR.K_SUM * TR.U32, r["cond"]
    v, (g,) = _run(L.depth_loss, [p], gt)
    assert v.dim() == 0 and v.dtype == torch.float32 and g.shape == p.shape
    _value_within(v, r["val"], r["vb"], (kind, "library value"))
    _assert_within(g, r["grad"], r["gb"], (kind, "library gradient"))
    tv, (tg,) = _run(torch_depth_loss, [p.contiguous()], gt)
    _value_within(tv, r["val"], r["vb"], (kind, "torch value"))
    _assert_within(tg, r["grad"], r["gb"], (kind, "torch gradient"))


def test_torch_divides_by_a_python_number_as_a_reciprocal_multiply(dev):
    """gt / 25 and -p / scene_scale in the reference are a float32 CUDA tensor over a Python number, which torch computes as
    x * float32(1 / b): the rule gsr_depth_loss follows."""
    x = (torch.rand(1 << 20, generator=torch.Generator().manual_seed(3)) * 60).to(dev)
    for b in (25, 5.0, 3.7):
        inv = float(np.float32(1.0) / np.float32(b))
        assert torch.equal(x / b, x * inv), b


@pytest.mark.parametrize("kind", ["empty_mask", "constant_depth"])
def test_depth_loss_det_zero_gives_nan(dev, kind):
    from autovfx_b200 import losses as L
    p = (1.0 + torch.rand(64, 80, generator=torch.Generator().manual_seed(1))).to(dev)
    gt = torch.rand(64, 80, generator=torch.Generator().manual_seed(2)).to(dev) * 50
    if kind == "empty_mask":
        gt = gt * 0.0 - 1.0
    else:
        p = torch.full_like(p, 2.0)
    v, (g,) = _run(L.depth_loss, [p], gt)
    assert torch.isnan(v) and torch.isnan(g).all()
    with pytest.raises((RuntimeError, ZeroDivisionError)):  # the reference fails (its 0-element tensors do not broadcast)
        torch_depth_loss(p.clone().requires_grad_(True), gt)


# -- opacity_loss and sparsity_loss --------------------------------------------------------------------------------------------
def _opacities(dev, P=1_000_000):
    gen = torch.Generator().manual_seed(4)
    x = torch.sigmoid(torch.randn(P, 1, generator=gen) * 3)
    edge = [TR.SPARSE_LO, TR.SPARSE_HI, 0.0, 1.0, -0.5, 1.5, float(np.nextafter(np.float32(TR.SPARSE_LO), np.float32(0))),
            float(np.nextafter(np.float32(TR.SPARSE_HI), np.float32(1)))]
    x[:len(edge), 0] = torch.tensor(edge)
    return x.to(dev)


@pytest.mark.parametrize("term", ["opacity", "sparsity"])
def test_opacity_terms_values_and_gradients(dev, term):
    from autovfx_b200 import losses as L
    x = _opacities(dev)
    lib, ref, fn64 = {"opacity": (L.opacity_loss, torch_opacity_loss, TR.opacity64),
                      "sparsity": (L.sparsity_loss, torch_sparsity_loss, TR.sparsity64)}[term]
    r = fn64(x)
    v, (g,) = _run(lib, [x])
    assert v.dim() == 0 and g.shape == x.shape
    _value_within(v, r["val"], r["vb"], (term, "library value"))
    _assert_within(g, r["grad"], r["gb"], (term, "library gradient"))
    tv, (tg,) = _run(ref, [x])
    _value_within(tv, r["val"], r["vb"], (term, "torch value"))
    _assert_within(tg, r["grad"], r["gb"], (term, "torch gradient"))
    if term == "sparsity":  # exactly on both bounds the gradient passes; one ulp outside, and outside [0, 1], it is zero
        assert (g[:2] != 0).all() and (g[2:8] == 0).all() and torch.equal(g[:8] != 0, tg[:8] != 0)


def test_opacity_terms_on_a_strided_view(dev):
    from autovfx_b200 import losses as L
    x = _opacities(dev, 10_000)
    buf = torch.rand(10_000, 3, device=dev)
    buf[:, 1:2] = x
    view = buf[:, 1:2]
    assert not view.is_contiguous()
    for lib in (L.opacity_loss, L.sparsity_loss):
        a, (ga,) = _run(lib, [x])
        leaf = buf.detach().clone().requires_grad_(True)
        v = lib(leaf[:, 1:2])
        v.backward()
        assert torch.equal(v.detach(), a) and torch.equal(leaf.grad[:, 1:2], ga) and (leaf.grad[:, ::2] == 0).all()


# -- the entropy term ------------------------------------------------------------------------------------------------------------
def _entropy_case(dev, P=3_000_000, layout="P1", visible=0.7):
    gen = torch.Generator().manual_seed(6)
    o = torch.sigmoid(torch.randn(P, generator=gen) * 2)
    o[:4] = torch.tensor([0.0, 1.0, 0.0, 1.0])
    radii = torch.where(torch.rand(P, generator=gen) < visible, torch.randint(1, 40, (P,), generator=gen, dtype=torch.int32),
                        torch.zeros(P, dtype=torch.int32))
    radii[:4] = torch.tensor([3, 3, 0, 0], dtype=torch.int32)
    o = o.unsqueeze(1) if layout == "P1" else o
    return o.to(dev), radii.to(dev)


@pytest.mark.parametrize("layout", ["P", "P1"])
def test_entropy_values_and_gradients(dev, layout):
    from autovfx_b200 import losses as L
    o, radii = _entropy_case(dev, layout=layout)
    r = TR.entropy64(o, radii)
    v, (g,) = _run(L.entropy_loss, [o], radii)
    assert v.dim() == 0 and g.shape == o.shape
    _value_within(v, r["val"], r["vb"], (layout, "library value"))
    _assert_within(g, r["grad"], r["gb"], (layout, "library gradient"))
    tv, (tg,) = _run(torch_entropy, [o], radii)
    _value_within(tv, r["val"], r["vb"], (layout, "torch value"))
    _assert_within(tg, r["grad"], r["gb"], (layout, "torch gradient"))
    gf = g.view(-1)
    assert torch.isfinite(gf[:2]).all() and (gf[2:4] == 0).all() and (gf[radii <= 0] == 0).all()  # o in {0, 1}: finite


def test_entropy_no_visible_gaussian_is_nan(dev):
    from autovfx_b200 import losses as L
    o, radii = _entropy_case(dev, P=5000, visible=0.0)
    radii[:4] = 0
    v, (g,) = _run(L.entropy_loss, [o], radii)
    tv, (tg,) = _run(torch_entropy, [o], radii)
    assert torch.isnan(v) and torch.isnan(tv) and (g == 0).all() and (tg == 0).all()


# -- the density-mode SDF estimation -----------------------------------------------------------------------------------------------
def _density_case(dev, N=1_000_000):
    gen = torch.Generator().manual_seed(8)
    d = torch.rand(N, generator=gen)
    b = 0.02 + 0.1 * torch.rand(N, generator=gen)
    s = 0.1 * torch.randn(N, generator=gen)
    # s = 0 with d equal to its target 1 and beta tiny: abs's sign(0) (and 2 * 0) zero every gradient; then a few exact ties at s != 0
    s[:4], b[:4], d[:4] = 0.0, torch.tensor([1e-12, 1e-6, 0.05, 1.0]), 1.0
    d, b, s = d.to(dev), b.to(dev), s.to(dev)
    d[4:8] = torch.exp(-0.5 * s[4:8].pow(2) / b[4:8].pow(2))  # torch's float32 targets at s != 0
    return d, b, s


@pytest.mark.parametrize("squared", [False, True], ids=["abs", "squared"])
def test_density_estimation_values_and_gradients(dev, squared):
    from autovfx_b200.sugar_field import density_estimation_loss
    d, b, s = _density_case(dev)
    r = TR.density64(d, b, s, squared)
    v, gs = _run(density_estimation_loss, [d, b, s], squared)
    assert v.dim() == 0 and all(g.shape == d.shape for g in gs)
    _value_within(v, r["val"], r["vb"], (squared, "library value"))
    tv, tgs = _run(torch_density, [d, b, s], squared)
    _value_within(tv, r["val"], r["vb"], (squared, "torch value"))
    for name, g, tg, want, bound in zip(("densities", "beta", "sdf_estimation"), gs, tgs, r["grads"], r["gbs"]):
        _assert_within(g, want, bound, (squared, "library", name))
        _assert_within(tg, want, bound, (squared, "torch", name))
        assert (g[:4] == 0).all() and (tg[:4] == 0).all(), name  # s = 0, d = target, beta tiny


def test_density_estimation_on_strided_inputs(dev):
    """The field's density and beta as columns of one buffer, the estimate contiguous: read in place, same bits."""
    from autovfx_b200.sugar_field import density_estimation_loss
    d, b, s = _density_case(dev, 4096)
    buf = torch.stack([d, b, torch.zeros_like(d)], 1)
    a, ga = _run(density_estimation_loss, [d, b, s])
    leaf = buf.clone().requires_grad_(True)
    sl = s.clone().requires_grad_(True)
    v = density_estimation_loss(leaf[:, 0], leaf[:, 1], sl)
    v.backward()
    assert torch.equal(v.detach(), a) and torch.equal(leaf.grad[:, 0], ga[0]) and torch.equal(leaf.grad[:, 1], ga[1])
    assert torch.equal(sl.grad, ga[2])


# -- determinism -----------------------------------------------------------------------------------------------------------------
def _all_terms(dev):
    from autovfx_b200 import losses as L
    from autovfx_b200.sugar_field import density_estimation_loss
    p, gt = _depth_case("1080p", dev)
    x = _opacities(dev)
    o, radii = _entropy_case(dev)
    d, b, s = _density_case(dev)
    out = []
    for fn, leaves, rest in ((L.depth_loss, [p], [gt]), (L.opacity_loss, [x], []), (L.sparsity_loss, [x], []),
                             (L.entropy_loss, [o], [radii]), (density_estimation_loss, [d, b, s], [False]),
                             (density_estimation_loss, [d, b, s], [True])):
        v, gs = _run(fn, leaves, *rest)
        out += [v] + gs
    return out


def test_bit_identical_repeats_with_and_without_deterministic_mode(dev):
    a = _all_terms(dev)
    b = _all_terms(dev)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = _all_terms(dev)
    finally:
        torch.use_deterministic_algorithms(prev)
    for u, v, w in zip(a, b, c):
        assert _same_bits(u, v) and _same_bits(u, w)


def test_no_grad_keeps_nothing(dev):
    from autovfx_b200 import losses as L
    from autovfx_b200.sugar_field import density_estimation_loss
    p, gt = _depth_case("near_flat", dev)
    o, radii = _entropy_case(dev, P=1000)
    leaves = [t.clone().requires_grad_(True) for t in (p, o)]
    with torch.no_grad():
        for v in (L.depth_loss(leaves[0], gt), L.opacity_loss(leaves[1]), L.sparsity_loss(leaves[1]),
                  L.entropy_loss(leaves[1], radii), density_estimation_loss(leaves[1], leaves[1], leaves[1])):
            assert v.grad_fn is None and not v.requires_grad


# -- no host synchronisation ----------------------------------------------------------------------------------------------------
def _no_sync(objective, leaves):
    """objective() and its backward() under torch.cuda.set_sync_debug_mode("error")."""
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        objective().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(t.grad is not None and torch.isfinite(t.grad).all() for t in leaves)


def _raises_under_sync_error(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with pytest.raises(RuntimeError):
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_train_objective_has_no_host_sync(dev):
    """GS/train.py:98-132 with every lambda > 0 on render_raw outputs: the objective's leaves are the render's outputs and the
    activated opacities and scales, detached, so only the objective and its backward are checked."""
    from autovfx_b200 import losses as L, renderer
    from tests.test_gpu_raw_render import PIPE, _RawPC, _case
    raw, cam, bg, D, mod, offset = _case("small_sh", dev)
    H, W = int(cam.image_height), int(cam.image_width)
    pc = _RawPC(raw, D, offset)
    out = renderer.render_raw(cam, pc, PIPE, bg, scaling_modifier=mod)
    gen = torch.Generator().manual_seed(1)
    gt_image = torch.rand(4, H, W, generator=gen).to(dev)
    gt_depth = (25 * (0.3 * out["depth"].detach().cpu() + 0.2 + 0.05 * torch.randn(H, W, generator=gen))).clamp_min(0).to(dev)
    gt_normal = torch.randn(H, W, 3, generator=gen).to(dev)
    image, depth, normal = (out[k].detach().clone().requires_grad_(True) for k in ("render", "depth", "normal"))
    pseudo_normal = out["pseudo_normal"].detach()
    opacity = torch.sigmoid(pc._opacity).detach().requires_grad_(True)
    scaling = torch.exp(pc._scaling).detach().requires_grad_(True)
    leaves = [image, depth, normal, opacity, scaling]

    def objective():
        loss = L.photometric_loss(image, gt_image, 0.2)
        loss = loss + 0.1 * L.depth_loss(depth, gt_depth)
        loss = loss + 0.05 * L.normal_loss(normal, gt_normal)
        loss = loss + 0.01 * L.normal_loss(normal, pseudo_normal)
        loss_alpha = L.opacity_loss(opacity)
        loss_alpha = L.sparsity_loss(opacity)
        loss = loss + 0.01 * loss_alpha
        return loss + 0.1 * L.anisotropic_loss(scaling)

    _no_sync(objective, leaves)
    _raises_under_sync_error(lambda: torch_depth_loss(depth, gt_depth))


def _sugar_render(dev):
    from autovfx_b200 import renderer
    from tests.test_gpu_sugar_render import _scene
    model = _scene(dev)
    out = renderer.render_sugar_raw(model, camera_indices=1, bg_color=torch.tensor([0.1, 0.2, 0.3], device=dev), sh_deg=3,
                                    return_2d_radii=True, return_opacities=True)
    image = out["image"].detach().clone().requires_grad_(True)
    gt = torch.rand(image.shape, generator=torch.Generator().manual_seed(2)).to(dev)
    return out, image, gt


def test_coarse_density_entropy_phase_has_no_host_sync(dev):
    """coarse_density's objective in the entropy phase (iterations 7000-9000): L1 + D-SSIM on the image and the entropy term on a
    SuGaR stand-in's render_sugar_raw outputs."""
    from autovfx_b200 import losses as L
    out, image, gt = _sugar_render(dev)
    radii = out["radii"]
    opacities = out["opacities"].detach().clone().requires_grad_(True)
    assert int((radii > 0).sum()) > 0

    def objective():
        loss = L.photometric_loss(image.permute(2, 0, 1), gt.permute(2, 0, 1), 0.2)
        return loss + 0.1 * L.entropy_loss(opacities, radii)

    _no_sync(objective, [image, opacities])
    _raises_under_sync_error(lambda: torch_entropy(opacities, radii))


def test_coarse_density_sdf_phase_has_no_host_sync(dev):
    """coarse_density's objective in the SDF phase (after iteration 9000): L1 + D-SSIM on the stand-in's image and the density-mode
    estimation loss on seeded field outputs and estimate."""
    from autovfx_b200 import losses as L
    from autovfx_b200.sugar_field import density_estimation_loss
    out, image, gt = _sugar_render(dev)
    d, b, s = (t[:20_000].clone().requires_grad_(True) for t in _density_case(dev, 20_000))
    proj_mask = torch.ones_like(s, dtype=torch.bool)

    def objective():
        loss = L.photometric_loss(image.permute(2, 0, 1), gt.permute(2, 0, 1), 0.2)
        return loss + 0.2 * density_estimation_loss(d, b, s)

    _no_sync(objective, [image, d, b, s])
    _raises_under_sync_error(lambda: torch_density(d[proj_mask], b[proj_mask], s))
