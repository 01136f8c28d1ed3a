"""CPU tests of SuGaR's sample_points_in_gaussians and the drop-in's restatement (tests/sugar_sample_ref.py): SuGaR draws row k
with probability proportional to the cumulative weight C_k, not to w_k; given the same u and z the drop-in's float64 search and
float32 placement agree with SuGaR's own computation; the C entry points are declared and bound; argument validation."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from tests import sugar_sample_ref as SR


def _scene(P, seed=0):
    g = torch.Generator().manual_seed(seed)
    points = torch.randn(P, 3, generator=g)
    scaling = torch.exp(math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g))
    quats = torch.randn(P, 4, generator=g)
    strengths = torch.rand(P, 1, generator=g)
    return points, scaling, quats, strengths


def _chi2_pvalue(counts, p, min_expected=5.0):
    """Chi-square p-value of observed counts against probabilities p, pooling consecutive bins until each expects >= 5."""
    n = counts.sum()
    exp = p * n
    obs_b, exp_b, o, e = [], [], 0.0, 0.0
    for ci, ei in zip(counts.tolist(), exp.tolist()):
        o, e = o + ci, e + ei
        if e >= min_expected:
            obs_b.append(o), exp_b.append(e)
            o, e = 0.0, 0.0
    if e > 0:
        obs_b[-1] += o
        exp_b[-1] += e
    return stats.chisquare(np.array(obs_b), np.array(exp_b)).pvalue


@pytest.mark.parametrize("volume", [False, True])
def test_sugar_draws_rows_proportional_to_the_cumulative_weight(volume):
    """SuGaR's method, literally, with torch.multinomial: the counts fit p_k ~ C_k; with uniform weights they do not fit p_k ~ w_k."""
    P, N = 40, 400_000
    points, scaling, quats, strengths = _scene(P)
    model = SR.Getters(points, scaling, quats, strengths)
    gen = torch.Generator().manual_seed(7)
    _, idx = SR.sample_points_in_gaussians(model, N, 1.5, probabilities_proportional_to_volume=volume, generator=gen)
    counts = torch.bincount(idx, minlength=P).double().numpy()
    w = SR.weights(scaling, volume=volume).double()
    c = w.cumsum(0)
    assert _chi2_pvalue(counts, (c / c.sum()).numpy()) > 1e-3
    if not volume:
        assert _chi2_pvalue(counts, (w / w.sum()).numpy()) < 1e-12


def test_sugar_mask_selects_rows_in_order():
    """With a mask the ramp runs over the selected rows in row order; unselected rows never appear."""
    P, N = 30, 300_000
    points, scaling, quats, strengths = _scene(P, seed=1)
    mask = torch.rand(P, generator=torch.Generator().manual_seed(2)) < 0.6
    mask[:3] = False
    model = SR.Getters(points, scaling, quats, strengths)
    gen = torch.Generator().manual_seed(8)
    _, idx = SR.sample_points_in_gaussians(model, N, 1.0, mask=mask, probabilities_proportional_to_volume=False, generator=gen)
    counts = torch.bincount(idx, minlength=P).double()
    assert (counts[~mask] == 0).all()
    T = SR.prefix(SR.weights(scaling, mask=mask, volume=False), mask)
    p = torch.diff(T, prepend=T.new_zeros(1)) / T[-1]
    assert _chi2_pvalue(counts[mask].numpy(), p[mask].numpy()) > 1e-3


@pytest.mark.parametrize("opacity,volume,masked", [(False, True, True), (True, True, False), (True, False, True), (False, False, False)])
def test_restatements_agree_given_the_draws(opacity, volume, masked):
    """Given u and z: SuGaR's float32 cum_probs, searched as torch.multinomial searches its weights, and the drop-in's float64
    search pick the same rows except where u lies within a float32 rounding band of a boundary; the placements are bit-equal."""
    P, N, f = 500, 100_000, 1.5
    points, scaling, quats, strengths = _scene(P, seed=3)
    scaling[5:9] = 0.0  # zero-volume rows
    mask = None
    if masked:
        mask = torch.rand(P, generator=torch.Generator().manual_seed(4)) < 0.7
        mask[:10] = False
    u, z = SR.draws(N, "cpu", seed=5)
    s = strengths if opacity else None
    T = SR.prefix(SR.weights(scaling, s, mask, volume), mask)
    rows, total = SR.select_rows(T, u)
    # SuGaR's path in float32: areas over the selected rows, cum_probs, then the inverse CDF of those weights
    sel = torch.arange(P) if mask is None else torch.arange(P)[mask]
    areas = SR.weights(scaling[sel], None if s is None else s[sel], None, volume)
    cum_probs = areas.cumsum(-1) / areas.sum(-1, keepdim=True)
    cdf = cum_probs.cumsum(-1) / cum_probs.sum()
    rows32 = sel[torch.searchsorted(cdf, u.float(), right=True).clamp(max=sel.numel() - 1)]
    off = rows != rows32
    assert (T[rows] > torch.cat([T.new_zeros(1), T[:-1]])[rows]).all()  # no zero-weight row
    band = 64 * 2.0 ** -24 * P  # float32 cumsums of P positive terms, twice
    lo = torch.minimum(rows, rows32)[off]
    assert ((u[off] - T[lo] / total).abs() <= band).all()
    assert off.sum() <= 0.01 * N
    a = SR.place(points, scaling, quats, rows, z, f)
    b = SR.place_pytorch3d(points, scaling, quats, rows, z, f)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_non_unit_quaternions_scale_by_the_squared_norm():
    """pytorch3d's quaternion_apply multiplies by the conjugate: a quaternion of norm r scales the offset by r^2."""
    q = torch.tensor([[0.3, -1.2, 0.5, 2.0]], dtype=torch.float64)
    v = torch.tensor([[0.1, 0.2, -0.3]], dtype=torch.float64)
    out = SR.quaternion_apply(q, v)
    qn = q / q.norm()
    assert torch.allclose(out, SR.quaternion_apply(qn, v) * q.norm() ** 2, rtol=1e-12, atol=0)


def test_select_rows_skips_zero_weight_rows_and_stays_in_range():
    w = torch.tensor([0.0, 0.0, 1.0, 0.0, 2.0, 0.0])
    mask = torch.tensor([True, True, True, False, True, False])
    T = SR.prefix(w, mask)
    u = torch.tensor([0.0, 0.5, 1.0 - 2.0 ** -53, 0.999999], dtype=torch.float64)
    rows, total = SR.select_rows(T, u)
    assert total == 4  # C = [0, 0, 1, 1, 3, 3], t = mask C = [0, 0, 1, 0, 3, 0], T = [0, 0, 1, 1, 4, 4]
    assert rows.tolist() == [2, 4, 4, 4]


# ------------------------------------------------------------------------------------------------ C ABI and Python surface
def test_exports_declared_and_bound():
    from autovfx_b200 import _lib
    for n in ("gsr_sugar_sample_bytes", "gsr_sugar_sample", "gsr_sugar_sample_backward"):
        assert n in _lib.EXPORTS and hasattr(_lib.lib, n)
    L = _lib.lib
    nb = (3_000_000 + 1023) // 1024
    assert L.gsr_sugar_sample_bytes(3_000_000) == 8 * 3_000_000 + 2 * 16 * ((8 * nb + 15) // 16)
    assert L.gsr_sugar_sample(1, 0, 1.0, 1, *([None] * 10), None, 0, None) != 0
    assert b"P = 0" in L.gsr_last_error()
    assert L.gsr_sugar_sample_backward(1, 4, 1.0, *([None] * 10)) != 0


def test_drop_in_signature_matches_sugar():
    import inspect
    from autovfx_b200.sugar_field import sample_points_in_gaussians
    a = inspect.signature(sample_points_in_gaussians)
    b = inspect.signature(SR.sample_points_in_gaussians)
    assert list(a.parameters)[:6] == list(b.parameters)[:6]
    assert all(a.parameters[k].default == b.parameters[k].default for k in list(a.parameters)[1:6])


def _model(P=6, **over):
    points, scaling, quats, strengths = _scene(P)
    d = dict(points=points, scaling=scaling, quaternions=quats, strengths=strengths)
    d.update(over)
    return SR.Getters(d["points"], d["scaling"], d["quaternions"], d["strengths"])


@pytest.mark.parametrize("kw,model_over,match", [
    ({"num_samples": 0}, {}, "num_samples"),
    ({"num_samples": 2.5}, {}, "num_samples"),
    ({"num_samples": True}, {}, "num_samples"),
    ({"sampling_scale_factor": "1"}, {}, "sampling_scale_factor"),
    ({"mask": torch.ones(6, dtype=torch.uint8)}, {}, "mask"),
    ({"mask": torch.ones(5, dtype=torch.bool)}, {}, "mask"),
    ({}, {"points": torch.zeros(6, 3, dtype=torch.float64)}, "self.points"),
    ({}, {"points": torch.zeros(0, 3)}, "no rows"),
    ({}, {"scaling": torch.zeros(6, 2)}, "self.scaling"),
    ({}, {"quaternions": torch.zeros(5, 4)}, "self.quaternions"),
    ({"probabilities_proportional_to_opacity": True}, {"strengths": torch.zeros(6, 2)}, "self.strengths"),
    ({"probabilities_proportional_to_opacity": True}, {"strengths": torch.zeros(6, 1, dtype=torch.float64)}, "self.strengths"),
])
def test_argument_validation(kw, model_over, match):
    from autovfx_b200.sugar_field import sample_points_in_gaussians
    args = {"num_samples": 4}
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        sample_points_in_gaussians(_model(**model_over), **args)


def test_cpu_tensors_raise():
    from autovfx_b200.sugar_field import sample_points_in_gaussians
    with pytest.raises(RuntimeError, match="CUDA"):
        sample_points_in_gaussians(_model(), 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        sample_points_in_gaussians(_model(), 4, mask=torch.ones(6, dtype=torch.bool), probabilities_proportional_to_opacity=True)
