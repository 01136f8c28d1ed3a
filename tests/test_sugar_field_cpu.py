"""CPU tests of SuGaR's field restatement (tests/sugar_field_ref.py) and of the host side of autovfx_b200.sugar_field: the
restatement's quirks in float64, the wrapper's argument errors (raised before any device is touched) and the C-ABI validation."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from tests import sugar_field_ref as SF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _getters(P=6, dtype=torch.float64, seed=0):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(P, 3, generator=g, dtype=dtype)
    sc = torch.rand(P, 3, generator=g, dtype=dtype) * 0.5 + 0.1
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g, dtype=dtype), dim=-1)
    st = torch.rand(P, 1, generator=g, dtype=dtype)
    knn = torch.stack([torch.roll(torch.arange(P), -s) for s in range(4)], 1)
    return SF.Getters(pts, sc, q, st, knn)


def test_density_is_cloned_before_the_normalisation():
    m = _getters()
    m.strengths = torch.ones_like(m.strengths)
    x = m.points[:3].clone()  # at the centres: the own Gaussian gives 1, so d >= 1
    f = m.get_field_values(x, torch.arange(3), return_sdf=True, return_beta=True)
    assert (f["density"] >= 1).all()
    # the sdf used the normalised value: d / (d + 1e-12) < 1 in float64, so the sdf is beta * sqrt(-2 log(~1)) ~ 0
    assert (f["sdf"].abs() < 1e-5).all() and (f["sdf"] > 0).all()


def test_normalised_density_is_exactly_one_in_float32():
    for d in (1.0, 1.5, 16.0, 3.0e4):
        t = torch.tensor([d], dtype=torch.float32)
        assert (t / (t.detach() + 1e-12)).item() == 1.0
    # so sqrt(-2 log 1) = 0 and, with density_threshold = 1, the sdf is 0 (beta * (0 - 0)) in float32
    m = _getters(dtype=torch.float32)
    m.strengths = torch.ones_like(m.strengths)
    f = m.get_field_values(m.points[:3].clone(), torch.arange(3), return_sdf=True)
    assert (f["sdf"] == 0).all()


def test_sdf_offset_for_a_threshold_below_one():
    m = _getters()
    x = m.points[:4] + 0.05
    a = m.get_field_values(x, torch.arange(4), density_threshold=1.0)["sdf"]
    b = m.get_field_values(x, torch.arange(4), density_threshold=0.3)["sdf"]
    beta = m.get_field_values(x, torch.arange(4), return_sdf=False, return_beta=True)["beta"]
    c = np.sqrt(-2.0 * np.log(0.3))
    torch.testing.assert_close(a - b, beta * c, rtol=1e-12, atol=1e-14)
    assert np.sqrt(-2.0 * np.log(min(5.0, 1.0))) == 0  # thresholds above 1 are capped at 1


def test_clamp_boundaries():
    # q is clamped to [0, 1e8]: a sample at the centre of a tiny Gaussian gives q = 0 (o = strength), a far one gives exp(-5e7) = 0
    m = _getters(P=2)
    m.scaling = torch.full((2, 3), 1e-9, dtype=torch.float64)  # below the 1e-8 clamp: 1 / 1e-8, not 1 / 1e-9
    m.knn_idx = torch.tensor([[0, 1], [1, 0]])
    x = torch.stack([m.points[0], m.points[0] + 1e-8 * torch.tensor([1.0, 0, 0], dtype=torch.float64)])
    o = m.get_field_values(x, torch.tensor([0, 0]), return_sdf=False, return_closest_gaussian_opacities=True)["closest_gaussian_opacities"]
    assert o[0, 0] == m.strengths[0, 0] and o[0, 1] == 0
    # |shift| = 1e-8 under 1/1e-8 (the clamp) gives q = 1 -> exp(-0.5); under 1/1e-9 it would be q = 100
    torch.testing.assert_close(o[1, 0], m.strengths[0, 0] * np.exp(-0.5), rtol=1e-6, atol=0)
    # an empty density is clamped to opacity_min_clamp before the log
    f = m.get_field_values(x[:1] + 10.0, torch.tensor([0]), return_sdf=True, opacity_min_clamp=1e-16)
    beta = 1e-9
    torch.testing.assert_close(f["sdf"], torch.tensor([beta * np.sqrt(-2 * np.log(1e-16))], dtype=torch.float64))


def test_min_scale_gradient_goes_to_the_lowest_index_on_ties():
    m = _getters(P=3)
    s = torch.tensor([[0.2, 0.2, 0.2], [0.5, 0.3, 0.3], [0.4, 0.4, 0.1]], dtype=torch.float64, requires_grad=True)
    m.scaling = s
    m.knn_idx = torch.tensor([[0, 1, 2]])
    beta = m.get_field_values(m.points[:1] + 5.0, torch.tensor([0]), return_sdf=False, return_beta=True)["beta"]
    beta.sum().backward()
    want = torch.zeros(3, 3, dtype=torch.float64)
    want[0, 0] = want[1, 1] = want[2, 2] = 1.0 / 3
    # q is clamped for this far sample, so beta is the only path to the scales
    torch.testing.assert_close(s.grad, want)


def test_compute_density_equals_the_field_density():
    m = _getters()
    idx = m.knn_idx[torch.arange(5) % 6]
    x = m.points[:5] + 0.1
    d, o = m.compute_density(x, idx, density_factor=0.5, return_closest_gaussian_opacities=True)
    f = m.get_field_values(x, closest_gaussians_idx=idx, density_factor=0.5, return_sdf=False, return_closest_gaussian_opacities=True)
    assert torch.equal(d, f["density"]) and torch.equal(o, f["closest_gaussian_opacities"])
    assert torch.equal(m.compute_density(x), m.compute_density(x, m.get_gaussians_closest_to_samples(x)))


# ------------------------------------------------------------------------------------------------ the wrapper's errors
def _cpu_model(P=8, K=4):
    m = _getters(P=P, dtype=torch.float32)
    m.knn_idx = m.knn_idx[:, :K].contiguous()
    return m


@pytest.mark.parametrize("kwargs, match", [
    (dict(return_sdf_grad=True), "return_sdf_grad"),
    (dict(gaussian_strengths=torch.ones(8, 1)), "gaussian_strengths"),
    (dict(gaussian_centers=torch.ones(8, 3)), "gaussian_centers"),
    (dict(gaussian_inv_scaled_rotation=torch.ones(8, 3, 3)), "gaussian_inv_scaled_rotation"),
    (dict(gaussian_idx=None), "both None"),
    (dict(x=torch.ones(3, 3, dtype=torch.float64)), "x must be torch.float32"),
    (dict(x=torch.ones(3, 4)), "x must have shape"),
    (dict(gaussian_idx=torch.arange(3, dtype=torch.int32)), "gaussian_idx must be torch.int64"),
    (dict(gaussian_idx=torch.arange(4)), "gaussian_idx has 4 entries"),
    (dict(gaussian_idx=None, closest_gaussians_idx=torch.zeros(3, 33, dtype=torch.int64)), "K = 33"),
    (dict(gaussian_idx=None, closest_gaussians_idx=torch.zeros(2, 4, dtype=torch.int64)), "2 rows for 3 samples"),
    (dict(gaussian_idx=None, closest_gaussians_idx=torch.zeros(3, 4, dtype=torch.float32)), "closest_gaussians_idx must be torch.int64"),
    (dict(density_factor="1"), "density_factor"),
])
def test_get_field_values_rejects_what_no_caller_uses(kwargs, match):
    from autovfx_b200.sugar_field import get_field_values
    m = _cpu_model()
    args = dict(x=torch.zeros(3, 3), gaussian_idx=torch.arange(3))
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        get_field_values(m, **args)


@pytest.mark.parametrize("mode, match", [("learnable", "beta_mode = 'learnable'"), ("weighted_average", "weighted_average"),
                                         (None, "Unknown beta_mode."), ("avg", "Unknown beta_mode.")])
def test_beta_modes_other_than_average_raise(mode, match):
    from autovfx_b200.sugar_field import get_field_values
    m = _cpu_model()
    m.beta_mode = mode
    for kw in (dict(return_sdf=True), dict(return_sdf=False, return_beta=True)):
        with pytest.raises(ValueError, match=match):
            get_field_values(m, torch.zeros(3, 3), torch.arange(3), **kw)
    # density alone does not read beta_mode; on CPU tensors it then fails for want of a device
    with pytest.raises(RuntimeError, match="no CPU path"):
        get_field_values(m, torch.zeros(3, 3), torch.arange(3), return_sdf=False)


def test_model_tensors_are_checked():
    from autovfx_b200.sugar_field import compute_density
    m = _cpu_model()
    m.quaternions = torch.ones(8, 3)
    with pytest.raises(ValueError, match="self.quaternions"):
        compute_density(m, torch.zeros(3, 3), torch.zeros(3, 4, dtype=torch.int64))
    m = _cpu_model()
    m.strengths = torch.ones(8, 2)
    with pytest.raises(ValueError, match="self.strengths"):
        compute_density(m, torch.zeros(3, 3), torch.zeros(3, 4, dtype=torch.int64))


def test_cpu_tensors_raise_runtime_error():
    from autovfx_b200.sugar_field import compute_density, get_field_values
    m = _cpu_model()
    with pytest.raises(RuntimeError, match="no CPU path"):
        get_field_values(m, torch.zeros(3, 3), torch.arange(3))
    with pytest.raises(RuntimeError, match="no CPU path"):
        compute_density(m, torch.zeros(3, 3), torch.zeros(3, 4, dtype=torch.int64), return_closest_gaussian_opacities=True)
    with pytest.raises(RuntimeError, match="no CPU path"):
        compute_density(m, torch.zeros(3, 3))  # through the model's own neighbour search


# ------------------------------------------------------------------------------------------------ exports and the C ABI
def test_sugar_field_exports():
    from autovfx_b200 import _lib, sugar_field
    names = {"gsr_sugar_field_bytes", "gsr_sugar_field", "gsr_sugar_field_backward"}
    assert names <= set(_lib.EXPORTS) and _lib.ABI_VERSION == 4
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsr_b200.h")).read(), flags=re.S)
    for n in names:
        assert re.search(r"\b%s\(" % n, hdr)
    L = _lib.lib
    assert L.gsr_abi_version() == 4
    assert len(L.gsr_sugar_field.argtypes) == 21 and len(L.gsr_sugar_field_backward.argtypes) == 26
    assert L.gsr_sugar_field_bytes(1000) == 64 * 1000 and L.gsr_sugar_field_bytes(0) == 0 and L.gsr_sugar_field_bytes(-3) == 0
    assert set(sugar_field.__all__) >= {"get_field_values", "compute_density"}


def _fwd(L, N=10, K=16, P=100, R=None, x=256, rows=256, row_idx=None, pts=256, sc=256, q=256, st=256, outs=(256, None, None, None),
         ws=256, nbytes=1 << 30):
    R = N if R is None else R
    return L.gsr_sugar_field(N, K, P, R, x, rows, row_idx, pts, sc, q, st, 1.0, 1e-16, 0.0, *outs, ws, nbytes, None)


def test_c_abi_rejects_bad_arguments_before_any_launch():
    from autovfx_b200 import _lib
    L = _lib.lib
    # every call below fails validation (or is a no-op) before anything is launched or dereferenced
    for kw, msg in [(dict(N=-1, R=-1), b"negative"), (dict(P=-2), b"negative"), (dict(K=0), b"K = 0"), (dict(K=33), b"K = 33"),
                    (dict(R=7), b"R == N"), (dict(x=None), b"without its inputs"), (dict(rows=None), b"without its inputs"),
                    (dict(st=None), b"without its inputs"), (dict(sc=None, outs=(256, None, 256, 256)), b"sdf needs beta")]:
        assert _fwd(L, **kw) == -1, kw
        assert msg in L.gsr_last_error(), (kw, L.gsr_last_error())
    assert _fwd(L, ws=None) == -2 and b"workspace" in L.gsr_last_error()
    assert _fwd(L, ws=264) == -2 and b"aligned" in L.gsr_last_error()
    assert _fwd(L, nbytes=64 * 100 - 1) == -2
    assert _fwd(L, N=0, R=0, x=None, rows=None, pts=None, sc=None, q=None, st=None, ws=None) == 0  # N = 0 is a no-op
    assert _fwd(L, N=0, R=5, row_idx=256, ws=None) == 0
    n = [None] * 4
    bw = lambda **kw: L.gsr_sugar_field_backward(kw.get("N", 10), 16, 100, 10, 256, 256, None, 256, 256, 256, 256, 1.0, 1e-16, 0.0,
                                                 256, None, None, None, 256, *kw.get("outs", [256] * 4), 256,
                                                 kw.get("nbytes", 1 << 30), None)
    assert bw(outs=n) == -1 and b"required" in L.gsr_last_error()
    assert bw(nbytes=64 * 100) == -2 and b"workspace" in L.gsr_last_error()  # the backward needs twice the forward's bytes
    assert bw(N=-1) == -1
