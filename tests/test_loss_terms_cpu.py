"""CPU checks of the remaining loss terms (autovfx_b200.losses.depth_loss / opacity_loss / sparsity_loss / entropy_loss and
autovfx_b200.sugar_field.density_estimation_loss): the fp64 restatement of tests/loss_terms_ref.py against fp64 autograd of the
reference lines, the conditioning the depth bound carries, every argument error, CPU tensors, and the new C-ABI exports."""
from __future__ import annotations

import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402
import torch  # noqa: E402

from tests import loss_terms_ref as TR  # noqa: E402


# -- the reference lines, in fp64 --------------------------------------------------------------------------------------------------
def ref_depth_loss(network_output, gt, scene_scale=5.0):
    """loss_utils.depth_loss with compute_scale_and_shift (without the .cuda() of its weight)."""
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
    scale = (a_11 * b_0 - a_01 * b_1) / det
    shift = (-a_01 * b_0 + a_00 * b_1) / det
    return torch.mean(weight * torch.exp(-network_output.detach() / scene_scale) * (scale * network_output + shift - depth_2d) ** 2)


def ref_sparsity_loss(network_output):
    val = torch.clamp(network_output, 1e-3, 1 - 1e-3)
    return torch.mean(torch.log(val) + torch.log(1 - val))


def ref_entropy(opacities, radii):
    vis_opacities = opacities[radii > 0]
    return (- vis_opacities * torch.log(vis_opacities + 1e-10) - (1 - vis_opacities) * torch.log(1 - vis_opacities + 1e-10)).mean()


def ref_density(densities, beta, sdf_estimation, squared):
    target_densities = torch.exp(-0.5 * sdf_estimation.pow(2) / beta.pow(2))
    return ((densities - target_densities).pow(2) if squared else (densities - target_densities).abs()).mean()


def _depth_maps(H, W, seed, flat=False):
    gen = torch.Generator().manual_seed(seed)
    p = 1.0 + 0.03 * torch.rand(H, W, generator=gen, dtype=torch.float64) if flat else \
        1.0 + 4.0 * torch.rand(H, W, generator=gen, dtype=torch.float64)
    gt = 25 * (0.3 * p + 0.2 + 0.05 * torch.randn(H, W, generator=gen, dtype=torch.float64)).clamp_min(0.01)
    gt[:, : W // 2] = 0.0  # half the monocular depth missing
    return p, gt


@pytest.mark.parametrize("flat", [False, True], ids=["spread", "near_flat"])
def test_depth_restatement_matches_fp64_autograd(flat):
    p, gt = _depth_maps(17, 23, 4, flat)
    pr = p.clone().requires_grad_(True)
    ref = ref_depth_loss(pr, gt, 5.0)
    ref.backward(torch.tensor(0.7, dtype=torch.float64))
    r = TR.depth64(p, gt, 5.0, g_out=0.7)
    assert abs(float(r["val"]) - float(ref.detach())) <= 1e-12 * abs(float(ref.detach()))
    torch.testing.assert_close(r["grad"], pr.grad, rtol=1e-9, atol=1e-18)
    assert r["count"] == 17 * (23 - 23 // 2)


def test_depth_bound_carries_the_conditioning():
    """The near-flat map's fit is ill-conditioned: its scale bound, relative to the scale, is orders above the spread map's."""
    spread, flat = TR.depth64(*_depth_maps(64, 64, 1)), TR.depth64(*_depth_maps(64, 64, 1, flat=True))
    assert flat["cond"] > 50 * spread["cond"]
    assert flat["bx0"] / abs(flat["x0"]) > 50 * spread["bx0"] / abs(spread["x0"])
    assert flat["cond"] < 0.5 and all(torch.isfinite(flat["gb"]).view(-1))


def test_depth_restatement_det_zero_is_nan():
    p = torch.rand(4, 5, dtype=torch.float64)
    r = TR.depth64(p, torch.zeros(4, 5, dtype=torch.float64))
    assert r["count"] == 0 and torch.isnan(r["val"]) and torch.isnan(r["grad"]).all()
    r = TR.depth64(torch.full((4, 5), 2.0, dtype=torch.float64), torch.ones(4, 5, dtype=torch.float64))  # constant p: det == 0
    assert r["det"] == 0.0 and torch.isnan(r["val"])


def test_opacity_and_sparsity_restatements_match_fp64_autograd():
    gen = torch.Generator().manual_seed(9)
    x = torch.rand(300, 1, generator=gen, dtype=torch.float64) * 1.2 - 0.1
    x[:4, 0] = torch.tensor([TR.SPARSE_LO, TR.SPARSE_HI, 0.0, 1.0], dtype=torch.float64)
    xr = x.clone().requires_grad_(True)
    torch.mean(xr).backward()
    r = TR.opacity64(x)
    assert abs(float(r["val"]) - float(x.mean())) < 1e-15 and torch.equal(r["grad"], xr.grad)
    # torch's clamp compares against the float32 bounds when the input is float32; in fp64 it would use the doubles, so the
    # reference is evaluated with the float32 bounds spelled out
    xr = x.clone().requires_grad_(True)
    val = torch.clamp(xr, TR.SPARSE_LO, TR.SPARSE_HI)
    ref = torch.mean(torch.log(val) + torch.log(1 - val))
    ref.backward()
    r = TR.sparsity64(x)
    assert abs(float(r["val"]) - float(ref.detach())) < 1e-13
    torch.testing.assert_close(r["grad"], xr.grad, rtol=1e-12, atol=0.0)
    assert xr.grad[0, 0] != 0 and xr.grad[1, 0] != 0 and xr.grad[2, 0] == 0 and xr.grad[3, 0] == 0  # both bounds pass


def test_sparsity_bounds_are_torchs_float32_bounds():
    x = torch.tensor([TR.SPARSE_LO, TR.SPARSE_HI], dtype=torch.float32)
    assert torch.equal(torch.clamp(x, 1e-3, 1 - 1e-3), x)
    assert float(torch.nextafter(x[1], torch.tensor(2.0))) > TR.SPARSE_HI
    xr = x.clone().requires_grad_(True)
    ref_sparsity_loss(xr).backward()
    assert (xr.grad != 0).all()


@pytest.mark.parametrize("layout", ["P", "P1"])
def test_entropy_restatement_matches_fp64_autograd(layout):
    gen = torch.Generator().manual_seed(2)
    o = torch.rand(200, generator=gen, dtype=torch.float64)
    o[:2] = torch.tensor([0.0, 1.0], dtype=torch.float64)
    radii = torch.randint(-1, 3, (200,), generator=gen, dtype=torch.int32)
    radii[:2] = 1
    if layout == "P1":
        o = o.unsqueeze(1)
    orr = o.clone().requires_grad_(True)
    ref = ref_entropy(orr, radii.view(-1, 1) if layout == "P1" else radii)
    ref.backward()
    r = TR.entropy64(o, radii)
    assert r["count"] == int((radii > 0).sum())
    assert abs(float(r["val"]) - float(ref.detach())) < 1e-13
    torch.testing.assert_close(r["grad"], orr.grad, rtol=1e-12, atol=1e-300)


def test_entropy_restatement_no_visible_gaussian_is_nan():
    o = torch.rand(10, dtype=torch.float64)
    r = TR.entropy64(o, torch.zeros(10, dtype=torch.int32))
    assert torch.isnan(r["val"]) and (r["grad"] == 0).all() and torch.isnan(ref_entropy(o, torch.zeros(10, dtype=torch.int32)))


@pytest.mark.parametrize("squared", [False, True])
def test_density_restatement_matches_fp64_autograd(squared):
    gen = torch.Generator().manual_seed(5)
    n = 400
    d = torch.rand(n, generator=gen, dtype=torch.float64)
    b = 0.02 + 0.1 * torch.rand(n, generator=gen, dtype=torch.float64)
    s = 0.1 * torch.randn(n, generator=gen, dtype=torch.float64)
    s[:3], b[:3], d[:3] = 0.0, 1e-12, 1.0  # s = 0, d = target, beta tiny: torch's sign(0) zeroes every gradient
    leaves = [t.clone().requires_grad_(True) for t in (d, b, s)]
    ref = ref_density(*leaves, squared)
    ref.backward()
    r = TR.density64(d, b, s, squared)
    assert abs(float(r["val"]) - float(ref.detach())) < 1e-13
    for got, leaf in zip(r["grads"], leaves):
        torch.testing.assert_close(got, leaf.grad, rtol=1e-10, atol=1e-300)
        assert (leaf.grad[:3] == 0).all() and (got[:3] == 0).all()


# -- argument errors -------------------------------------------------------------------------------------------------------------
def test_depth_loss_argument_errors():
    from autovfx_b200 import losses as L
    p, g = torch.rand(6, 8), torch.rand(6, 8)
    with pytest.raises(ValueError, match="network_output"):
        L.depth_loss(p.double(), g)
    with pytest.raises(ValueError, match="gt"):
        L.depth_loss(p, g.half())
    with pytest.raises(ValueError, match="gt has 42 elements"):
        L.depth_loss(p, torch.rand(6, 7))
    with pytest.raises(ValueError, match="gt requires grad"):
        L.depth_loss(p, g.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="empty"):
        L.depth_loss(torch.rand(0), torch.rand(0))
    with pytest.raises(ValueError, match="scene_scale"):
        L.depth_loss(p, g, scene_scale="5")
    L_ = L.depth_loss
    with pytest.raises(RuntimeError, match="CUDA"):
        L_(p, g)
    with pytest.raises(RuntimeError, match="CUDA"):
        L_(p.view(1, 6, 8), g)  # same count, other shape: accepted up to the device check, as the reference flattens both


def test_opacity_sparsity_argument_errors():
    from autovfx_b200 import losses as L
    for fn in (L.opacity_loss, L.sparsity_loss):
        with pytest.raises(ValueError, match="network_output"):
            fn(torch.rand(5, 1).double())
        with pytest.raises(ValueError, match="network_output"):
            fn([0.5])
        with pytest.raises(ValueError, match="empty"):
            fn(torch.rand(0, 1))
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(torch.rand(5, 1))


def test_entropy_loss_argument_errors():
    from autovfx_b200 import losses as L
    o, r = torch.rand(7, 1), torch.ones(7, dtype=torch.int32)
    with pytest.raises(ValueError, match="opacities"):
        L.entropy_loss(o.double(), r)
    with pytest.raises(ValueError, match="opacities"):
        L.entropy_loss(torch.rand(7, 2), r)
    with pytest.raises(ValueError, match="radii"):
        L.entropy_loss(o, r.long())
    with pytest.raises(ValueError, match="radii"):
        L.entropy_loss(o, torch.ones(6, dtype=torch.int32))
    with pytest.raises(ValueError, match="empty"):
        L.entropy_loss(torch.rand(0), torch.ones(0, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        L.entropy_loss(o, r)


def test_density_estimation_loss_argument_errors():
    from autovfx_b200.sugar_field import density_estimation_loss as D
    a = torch.rand(9)
    with pytest.raises(ValueError, match="densities"):
        D(a.double(), a, a)
    with pytest.raises(ValueError, match="beta"):
        D(a, a.half(), a)
    with pytest.raises(ValueError, match="sdf_estimation has shape"):
        D(a, a, torch.rand(8))
    with pytest.raises(ValueError, match="beta has shape"):
        D(a, a.view(3, 3), a)
    with pytest.raises(ValueError, match="empty"):
        D(torch.rand(0), torch.rand(0), torch.rand(0))
    with pytest.raises(RuntimeError, match="CUDA"):
        D(a, a, a.clone().requires_grad_(True))


@pytest.mark.skipif(not torch.cuda.is_available(), reason="mixed devices need a CUDA device")
def test_mixed_devices_raise_value_error():
    from autovfx_b200 import losses as L
    from autovfx_b200.sugar_field import density_estimation_loss as D
    c = torch.rand(8, device="cuda")
    with pytest.raises(ValueError, match="gt"):
        L.depth_loss(c, torch.rand(8))
    with pytest.raises(ValueError, match="radii"):
        L.entropy_loss(c, torch.ones(8, dtype=torch.int32))
    with pytest.raises(ValueError, match="beta"):
        D(c, torch.rand(8), c)


# -- the C ABI -------------------------------------------------------------------------------------------------------------------
NEW_EXPORTS = ("gsr_depth_loss", "gsr_depth_loss_backward", "gsr_opacity_loss", "gsr_opacity_loss_backward", "gsr_sparsity_loss",
               "gsr_sparsity_loss_backward", "gsr_entropy_loss", "gsr_entropy_loss_backward", "gsr_density_estimation_loss",
               "gsr_density_estimation_loss_backward")


def test_new_exports_are_declared_and_bound():
    from autovfx_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    for n in NEW_EXPORTS:
        assert n in _lib.EXPORTS and hasattr(_lib.lib, n)
        assert ("int %s(" % n) in hdr


def test_new_entry_points_refuse_bad_arguments():
    """Null pointers or n <= 0 give GSR_ERR_INVALID (-1) and a missing workspace GSR_ERR_WORKSPACE (-2), before any launch."""
    from autovfx_b200 import _lib
    lib = _lib.lib
    assert lib.gsr_depth_loss(0, 8, 1, 8, 1, 0.2, 8, None, 0, None) == -1
    assert b"gsr_depth_loss" in lib.gsr_last_error()
    assert lib.gsr_depth_loss(4, 8, 1, 8, 1, 0.2, 8, None, 0, None) == -2
    assert lib.gsr_depth_loss_backward(4, 8, 1, 8, 1, 0.2, None, 8, None, 0, None) == -1
    assert lib.gsr_depth_loss_backward(4, 8, 1, 8, 1, 0.2, 8, 8, 8, 16, None) == -2  # workspace too small
    assert lib.gsr_opacity_loss(4, None, 1, 8, None, 0, None) == -1
    assert lib.gsr_opacity_loss(4, 8, 1, 8, None, 0, None) == -2
    assert lib.gsr_opacity_loss_backward(0, 8, 8, None) == -1
    assert lib.gsr_sparsity_loss(-1, 8, 1, 8, None, 0, None) == -1
    assert lib.gsr_sparsity_loss_backward(4, None, 1, 8, 8, None) == -1
    assert lib.gsr_entropy_loss(4, 8, 1, None, 1, 8, None, 0, None) == -1
    assert lib.gsr_entropy_loss(4, 8, 1, 8, 1, 8, None, 0, None) == -2
    assert lib.gsr_entropy_loss_backward(4, 8, 1, 8, 1, 8, 8, None, 0, None) == -2
    assert lib.gsr_density_estimation_loss(4, 8, 1, None, 1, 8, 1, 0, 8, None, 0, None) == -1
    assert lib.gsr_density_estimation_loss(4, 8, 1, 8, 1, 8, 1, 0, 8, None, 0, None) == -2
    assert lib.gsr_density_estimation_loss_backward(4, 8, 1, 8, 1, 8, 1, 0, 8, 8, None, 8, None) == -1
    assert b"gsr_density_estimation_loss_backward" in lib.gsr_last_error()
    ws = (C.c_uint8 * 64)()
    assert lib.gsr_entropy_loss(4, 8, 1, 8, 1, 8, C.addressof(ws), 64, None) == -2
