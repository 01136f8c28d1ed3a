"""CPU tests that the checks of tests/test_gpu_sugar_field_coverage.py have teeth: the float32 and float64 restatements of the
field (tests/sugar_field_ref.py) run on the CPU, and the checkers must accept a clean float32 result and reject planted errors
of the kinds a kernel could make: a beta with one extra term, a min-scale gradient moved to the other tied axis, and one wrong
Gaussian row among 3000 (which only the 100th percentile sees)."""
import math

import pytest
import torch

from tests import sugar_field_ref as SF
from tests.test_gpu_sugar_field import _bound, _check_fields
from tests.test_gpu_sugar_field_coverage import _grad_rule

P, K, N = 3000, 8, 4000


def _scene():
    """A SuGaR-like scene on the CPU: the edge cases of the GPU scenes (scales below the 1e-8 clamp, three-way ties, two-way
    ties of the min at indices 1 and 2), brute-force neighbours, samples drawn around the Gaussians."""
    g = torch.Generator().manual_seed(0)
    points = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([1.0, 1.0, 0.3])
    log_s = math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g)
    log_s[20:40] = math.log(1e-9)
    log_s[40:80] = log_s[40:80, :1]
    log_s[120:160, 2] = log_s[120:160, 1]
    log_s[120:160, 0] = log_s[120:160, 1] + 0.4
    scaling = torch.exp(log_s)
    quats = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    strengths = torch.sigmoid(2 * torch.randn(P, 1, generator=g))
    knn = torch.cdist(points, points).topk(K, dim=1, largest=False).indices
    idx = torch.randint(0, P, (N,), generator=g)
    x = points[idx] + (SF.quaternion_to_matrix(quats[idx]) @ (1.5 * scaling[idx] * torch.randn(N, 3, generator=g))[..., None])[..., 0]
    return [points, scaling, quats, strengths], knn, x, idx


@pytest.fixture(scope="module")
def scene():
    return _scene()


KW = dict(return_sdf=True, return_beta=True, return_closest_gaussian_opacities=True, density_factor=0.9 / K)


def _grads(t, knn, x, idx, dtype, flip=False):
    """Gradients of a fixed random functional of every field with respect to x, points, scaling, quaternions, strengths.  flip:
    each row's neighbours in reverse order, another summation order of the same float32 arithmetic."""
    leaves = [v.to(dtype).clone().requires_grad_(True) for v in (x, *t)]
    m = SF.Getters(*leaves[1:], knn)
    rows = knn[idx].flip(1) if flip else knn[idx]
    f = m.get_field_values(leaves[0], closest_gaussians_idx=rows, **KW)
    if flip:
        f["closest_gaussian_opacities"] = f["closest_gaussian_opacities"].flip(1)
    gen = torch.Generator().manual_seed(3)
    loss = sum((torch.randn(f[k].shape, generator=gen).to(dtype) * f[k]).sum() for k in sorted(f))
    loss.backward()
    return [v.grad for v in leaves]


@pytest.fixture(scope="module")
def grads(scene):
    t, knn, x, idx = scene
    return {name: _grads(t, knn, x, idx, dtype, flip) for name, dtype, flip in
            (("f64", torch.float64, False), ("torch32", torch.float32, False), ("other32", torch.float32, True))}


def test_forward_bound_rejects_a_beta_with_one_extra_term(scene):
    t, knn, x, idx = scene
    rows = knn[idx]
    m32 = SF.Getters(*t, knn)
    m64 = SF.Getters(*(v.double() for v in t), knn)
    want = SF.get_field_values(m64, x.double(), closest_gaussians_idx=rows, **KW)
    b = _bound(m64, x, rows, KW["density_factor"])
    clean = SF.get_field_values(m32, x, closest_gaussians_idx=rows.flip(1), **KW)
    clean["closest_gaussian_opacities"] = clean["closest_gaussian_opacities"].flip(1)
    _check_fields(clean, want, b, "clean")
    smin = t[1].min(-1)[0]
    planted = dict(clean)
    planted["beta"] = (smin[rows].sum(1) + smin[rows[:, 0]]) / K  # a ninth term, as from an idle lane that is not zero
    with pytest.raises(AssertionError, match="beta"):
        _check_fields(planted, want, b, "planted")


def test_gradient_rule_accepts_another_float32_order(grads):
    for i in range(5):
        _grad_rule("clean %d" % i, grads["other32"][i], grads["torch32"][i], grads["f64"][i])


def test_gradient_rule_rejects_a_min_scale_gradient_on_the_other_tied_axis(grads, scene):
    ds = grads["other32"][2].clone()
    tie = torch.arange(120, 160)
    assert (scene[0][1][tie, 1] == scene[0][1][tie, 2]).all() and (ds[tie, 1] != 0).all()
    ds[tie, 2], ds[tie, 1] = ds[tie, 1].clone(), ds[tie, 2].clone()  # the highest index of the tie instead of the lowest
    with pytest.raises(AssertionError, match="planted tie: q"):
        _grad_rule("planted tie", ds, grads["torch32"][2], grads["f64"][2])


def test_gradient_rule_rejects_one_wrong_row_among_3000(grads):
    for i in (1, 3, 4):  # points, quaternions, strengths
        g = grads["other32"][i].clone()
        r = int(g.reshape(P, -1).norm(dim=1).argmax())
        g[r] = g[r] * 1.01
        with pytest.raises(AssertionError, match="q100"):
            _grad_rule("planted row", g, grads["torch32"][i], grads["f64"][i])
