"""GPU tests of autovfx_b200.sugar_field.sample_points_in_gaussians (gsr_sugar_sample and its backward) against the restatements
of tests/sugar_sample_ref.py: given the draws, the rows equal the float64 search and the samples are bit-identical to the float32
placement; the distribution (chi-square, fixed seeds); gradients against float64 autograd; no host synchronisation; an empty
selection; coarse_density's block end to end; one full-size call."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from tests import sugar_normal_ref as SN
from tests import sugar_sample_ref as SR

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24


def _sample():
    from autovfx_b200.sugar_field import sample_points_in_gaussians
    return sample_points_in_gaussians


def _scene(P, seed=0, zero_volume=True, unit=False):
    g = torch.Generator().manual_seed(seed)
    points = torch.randn(P, 3, generator=g)
    scaling = torch.exp(math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g))
    if zero_volume and P > 8:
        scaling[:3, 1] = 0.0          # leading zero-volume rows: C = 0, never drawn with volume weights
        scaling[P // 2, 2] = 0.0
    quats = torch.randn(P, 4, generator=g)  # not unit: quaternion_apply scales by |q|^2
    if unit:
        quats = torch.nn.functional.normalize(quats, dim=-1)
    strengths = torch.rand(P, 1, generator=g)
    strengths[P - 1] = 0.0
    return [t.to(DEV).contiguous() for t in (points, scaling, quats, strengths)]


def _mask(P, seed=1):
    m = torch.rand(P, generator=torch.Generator().manual_seed(seed)) < 0.7
    m[: max(1, P // 8)] = False  # leading rows unselected
    m[-1] = True
    return m.to(DEV)


def _expected(scaling, strengths, mask, volume, opacity):
    w = SR.weights(scaling, strengths if opacity else None, mask, volume)
    T = SR.prefix(w, mask)
    return T, torch.diff(T, prepend=T.new_zeros(1))


def _call(model, N, f, mask, opacity, volume, seed):
    torch.manual_seed(seed)
    return _sample()(model, N, f, mask=mask, probabilities_proportional_to_opacity=opacity,
                     probabilities_proportional_to_volume=volume)


def _chi2_pvalue(counts, p, min_expected=5.0):
    exp = p * counts.sum()
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


def _check_rows(rows, ref_rows, T, u):
    """Rows equal the float64 search, except where u * total lies within a float64 rounding band of the boundary between the
    two rows (the kernel's scan adds in another order than torch's cumsum); count those."""
    off = rows != ref_rows
    total = T[-1]
    lo = torch.minimum(rows, ref_rows)[off]
    assert ((u[off] * total - T[lo]).abs() <= 1e-12 * total).all()
    assert off.sum().item() <= 4
    prev = torch.cat([T.new_zeros(1), T[:-1]])
    assert (T[rows] > prev[rows]).all()  # never a row of zero weight or an unselected row


CASES = [(v, o, m) for v in (False, True) for o in (False, True) for m in (False, True)]


@pytest.mark.parametrize("P", [8, 257, 4096])
@pytest.mark.parametrize("volume,opacity,masked", CASES)
def test_given_the_draws_rows_and_samples_match(P, volume, opacity, masked):
    points, scaling, quats, strengths = _scene(P)
    mask = _mask(P) if masked else None
    N, f, seed = 20_000, 1.5, 11
    model = SR.Getters(points, scaling, quats, strengths)
    x, idx = _call(model, N, f, mask, opacity, volume, seed)
    u, z = SR.draws(N, DEV, seed)
    T, _ = _expected(scaling, strengths, mask, volume, opacity)
    ref_rows, _ = SR.select_rows(T, u)
    assert idx.dtype == torch.int64 and x.dtype == torch.float32 and x.shape == (N, 3)
    _check_rows(idx, ref_rows, T, u)
    ref = SR.place(points, scaling, quats, idx, z, f)
    assert torch.equal(x.view(torch.int32), ref.view(torch.int32))
    assert torch.equal(x.view(torch.int32), SR.place_pytorch3d(points, scaling, quats, idx, z, f).view(torch.int32))


@pytest.mark.parametrize("P", [8, 257, 4096])
@pytest.mark.parametrize("volume,opacity,masked", CASES)
def test_distribution(P, volume, opacity, masked):
    """Chi-square of the row counts against p_k ~ mask_k C_k, fixed seed; rows with p = 0 never appear."""
    points, scaling, quats, strengths = _scene(P, seed=2)
    mask = _mask(P, seed=3) if masked else None
    N = 400_000 if P == 4096 else 100_000
    _, idx = _call(SR.Getters(points, scaling, quats, strengths), N, 1.0, mask, opacity, volume, seed=21)
    _, t = _expected(scaling, strengths, mask, volume, opacity)
    p = (t / t.sum()).cpu()
    counts = torch.bincount(idx, minlength=P).double().cpu()
    assert (counts[p == 0] == 0).all()
    if mask is not None:
        assert (counts[~mask.cpu()] == 0).all()
    assert _chi2_pvalue(counts[p > 0].numpy(), p[p > 0].numpy()) > 1e-4


def _row_bound(scaling, quats, z, g, idx, f, P):
    """Per-row bound of a float32 gradient against float64: each sample's terms have magnitude at most
    S_n = |g|_1 (1 + |q|^2)(1 + |v|_1 + f |z|_1) and about a dozen roundings, and the row sums `hits` of them with atomics, so
    (64 + hits) U times the sum of the row's S_n."""
    q2 = (quats.double() ** 2).sum(-1)[idx]
    zd = z.double()
    v1 = (f * scaling.double()[idx] * zd).abs().sum(-1)
    mag = g.double().abs().sum(-1) * (1 + q2) * (1 + v1 + f * zd.abs().sum(-1))
    hits = torch.bincount(idx, minlength=P).double()
    S = torch.zeros(P, dtype=torch.float64, device=idx.device).index_add_(0, idx, mag)
    return (64 + hits) * U * S + 1e-30, hits


def _grad_case(P, N, f, seed, masked=True):
    points, scaling, quats, strengths = _scene(P, seed=seed, zero_volume=False)
    mask = _mask(P, seed=seed + 1) if masked else None
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats)]
    model = SR.Getters(*leaves, strengths)
    x, idx = _call(model, N, f, mask, False, True, seed=31)
    g = torch.randn(N, 3, generator=torch.Generator().manual_seed(seed + 2)).to(DEV)
    (x * g).sum().backward()
    _, z = SR.draws(N, DEV, 31)
    l64 = [t.detach().double().requires_grad_(True) for t in (points, scaling, quats)]
    x64 = SR.place_pytorch3d(*l64, idx, z.double(), f)
    (x64 * g.double()).sum().backward()
    bound, hits = _row_bound(l64[1].detach(), l64[2].detach(), z, g, idx, f, P)
    for a, b in zip(leaves, l64):
        err = (a.grad.double() - b.grad).abs().amax(-1)
        assert (err <= bound).all(), (err / bound).max().item()
    return idx, hits


@pytest.mark.parametrize("P,N,f", [(8, 50_000, 1.5), (257, 100_000, 0.7), (4096, 200_000, 1.5)])
def test_gradients_against_float64(P, N, f):
    """Non-unit quaternions, f != 1, and rows hit many times (the end of the ramp)."""
    _, hits = _grad_case(P, N, f, seed=P)
    assert hits.max() > 100


def test_gradients_through_sugar_like_getters():
    """Getters exp / normalize / sigmoid of raw leaves: the gradients reach the leaves as in torch (float64 autograd)."""
    P, N, f = 1000, 100_000, 1.5
    g0 = torch.Generator().manual_seed(5)
    raw = [torch.randn(P, 3, generator=g0), math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g0), torch.randn(P, 4, generator=g0),
           torch.randn(P, 1, generator=g0)]
    leaves = [t.to(DEV).requires_grad_(True) for t in raw]
    model = SR.RawModel(*leaves)
    mask = _mask(P)
    x, idx = _call(model, N, f, mask, True, True, seed=41)
    g = torch.randn(N, 3, generator=torch.Generator().manual_seed(6)).to(DEV)
    (x * g).sum().backward()
    assert leaves[3].grad is None  # the weights get no gradient
    _, z = SR.draws(N, DEV, 41)
    l64 = [t.detach().double().requires_grad_(True) for t in leaves[:3]]
    m64 = SR.RawModel(*l64, None)
    (SR.place_pytorch3d(m64.points, m64.scaling, m64.quaternions, idx, z.double(), f) * g.double()).sum().backward()
    # the raw leaves: d/draw_s = s * d/ds, d/draw_q = (I - n n^T) d/dq / |raw_q|
    bound, _ = _row_bound(m64.scaling.detach(), m64.quaternions.detach(), z, g, idx, f, P)
    chain = [torch.ones_like(bound), m64.scaling.detach().amax(-1), 2 / l64[2].detach().norm(dim=-1)]
    for a, b, c in zip(leaves[:3], l64, chain):
        err = (a.grad.double() - b.grad).abs().amax(-1)
        assert (err <= bound * c.clamp(min=1)).all(), (err / (bound * c.clamp(min=1))).max().item()


def test_same_seed_same_outputs_and_no_host_sync():
    P, N = 4096, 50_000
    points, scaling, quats, strengths = _scene(P)
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats)]
    model = SR.Getters(*leaves, strengths)
    mask = _mask(P)
    outs = []
    for _ in range(2):
        torch.manual_seed(3)
        torch.cuda.set_sync_debug_mode("error")
        try:
            x, idx = _sample()(model, N, 1.5, mask=mask, probabilities_proportional_to_opacity=True)
            (x * x).sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        outs.append((x.detach().clone(), idx.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("how", ["empty_mask", "zero_volume", "nan_scale"])
def test_empty_or_non_finite_total(how):
    """No row to draw: indices stay in [0, P), the samples are NaN and the gradients zero."""
    P, N = 300, 1000
    points, scaling, quats, strengths = _scene(P)
    mask = None
    if how == "empty_mask":
        mask = torch.zeros(P, dtype=torch.bool, device=DEV)
    elif how == "zero_volume":
        scaling[:, 0] = 0.0
    else:
        scaling[7, 2] = float("nan")
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats)]
    x, idx = _sample()(SR.Getters(*leaves, strengths), N, 1.5, mask=mask)
    x.sum().backward()
    assert ((idx >= 0) & (idx < P)).all()
    assert torch.isnan(x).all()
    for t in leaves:
        assert torch.equal(t.grad, torch.zeros_like(t))


def test_coarse_density_block_end_to_end():
    """Sampling through to coarse_density's loss with the library's field, estimate and normal loss, against the torch sampler
    fed the same draws (same rows and bit-identical samples), then the same library block."""
    from autovfx_b200 import sugar_field
    from autovfx_b200.knn import knn_points
    P, N = 20_000, 100_000
    points, scaling, quats, strengths = _scene(P, seed=9, unit=True)
    knn = knn_points(points[None], points[None], K=16).idx[0]
    mask = _mask(P)
    res = []
    for lib_sampler in (True, False):
        leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats, strengths)]
        model = SN.Getters(*leaves, knn)
        model.get_field_values = sugar_field.get_field_values.__get__(model)
        if lib_sampler:
            x, idx = _call(model, N, 1.5, mask, False, True, seed=51)
        else:
            u, z = SR.draws(N, DEV, 51)
            T = SR.prefix(SR.weights(model.scaling.detach(), None, mask, True), mask)
            idx, _ = SR.select_rows(T, u)
            x = SR.place_pytorch3d(model.points, model.scaling, model.quaternions, idx, z, 1.5)
        loss = SN.density_block(model, x, idx, estimate=sugar_field.projection_estimate, normal_loss=sugar_field.better_normal_loss)
        loss.backward()
        res.append((x.detach(), idx, loss.detach(), [t.grad for t in leaves]))
    (xa, ia, la, ga), (xb, ib, lb, gb) = res
    assert torch.equal(ia, ib) and torch.equal(xa.view(torch.int32), xb.view(torch.int32))
    torch.testing.assert_close(la, lb, rtol=1e-6, atol=0)
    for a, b in zip(ga, gb):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-4 * b.abs().max().item())


def test_full_size():
    """3M Gaussians, 1M samples, a mask with about 70 % of rows set: finite samples, every row in range and selected; the peak
    allocation of the call stays within the outputs, the draws and gsr_sugar_sample_bytes(P), plus 8 MiB for the allocator's
    rounding."""
    from autovfx_b200 import _lib, scene
    g = scene.config3_scene(P=3_000_000)
    points = g["means3D"].to(DEV).contiguous()
    scaling = g["scales"].to(DEV).contiguous()
    quats = torch.nn.functional.normalize(g["rotations"].to(DEV), dim=-1).contiguous()
    strengths = g["opacities"].reshape(-1, 1).to(DEV).contiguous()
    P, N = points.shape[0], 1_000_000
    mask = torch.rand(P, generator=torch.Generator().manual_seed(0)).to(DEV) < 0.7
    model = SR.Getters(points, scaling, quats, strengths)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        x, idx = _call(model, N, 1.5, mask, False, True, seed=61)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    budget = N * (12 + 8) + 8 + N * (8 + 12) + _lib.lib.gsr_sugar_sample_bytes(P) + 8 * 2 ** 20
    assert peak <= budget, (peak, budget)
    assert torch.isfinite(x).all()
    assert ((idx >= 0) & (idx < P)).all() and mask[idx].all()
