"""GPU tests of autovfx_b200.sugar_field (gsr_sugar_field / gsr_sugar_field_backward) against SuGaR's field restated in torch
(tests/sugar_field_ref.py): the forward against float64 within an error bound derived below, which torch's own float32 graph
must meet too; the gradients of the five inputs against float64 autograd; SuGaR's two trainer blocks end to end; one full-size
call."""
import math

import numpy as np
import pytest
import torch

from tests import sugar_field_ref as SF

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # float32 unit roundoff
DEV = "cuda"


def _sf():
    from autovfx_b200 import sugar_field
    return sugar_field


def _knn(points, K):
    from autovfx_b200.knn import knn_points
    return knn_points(points[None], points[None], K=K).idx[0]


def _scene(P, K, seed=0, edge_cases=False):
    """Getter outputs (float32) of a small SuGaR-like scene and its neighbour table.  With edge_cases: scales below the 1e-8
    clamp, three-way scale ties, and 16 coincident Gaussians (strength exactly 1 in float32) at the start."""
    g = torch.Generator().manual_seed(seed)
    points = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([1.0, 1.0, 0.3])
    log_s = math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g)
    dens = torch.randn(P, 1, generator=g) * 2
    quats = torch.randn(P, 4, generator=g)
    if edge_cases:
        points[:16] = points[16]
        dens[:16] = 40.0                     # sigmoid(40) == 1 in float32
        log_s[20:40] = math.log(1e-9)        # below the 1e-8 clamp
        log_s[40:80] = log_s[40:80, :1]      # three-way ties
        log_s[80:120, 1:] = log_s[80:120, :1]  # two-way ties, min on the tie
    scaling = torch.exp(log_s)
    strengths = torch.sigmoid(dens).reshape(-1)
    quats = torch.nn.functional.normalize(quats, dim=-1)
    t = [v.to(DEV).contiguous() for v in (points, scaling, quats, strengths)]
    knn = _knn(t[0], K)
    return t, knn


def _samples(points, scaling, quats, N, seed=1, edge_cases=False):
    g = torch.Generator().manual_seed(seed)
    P = points.shape[0]
    idx = torch.randint(0, P, (N,), generator=g).to(DEV)
    v = 1.5 * scaling[idx] * torch.randn(N, 3, generator=g).to(DEV)
    x = points[idx] + (SF.quaternion_to_matrix(quats[idx]) @ v[..., None])[..., 0]
    if edge_cases and N >= 64:
        x[:16] = points[idx[:16]]          # at the centres: q = 0
        x[16:24] = points[idx[16:24]] + 5000  # far: q clamped at 1e8, exp underflows
        idx[24:32] = torch.arange(8, device=DEV)  # inside the 16 coincident Gaussians of strength 1: d >= 1
        x[24:32] = points[:8]
        idx[32:40] = torch.arange(20, 28, device=DEV)  # at tiny Gaussians
        x[32:40] = points[20:28]
    return x.contiguous(), idx


def _models(t, knn):
    m32 = SF.Getters(t[0], t[1], t[2], t[3][:, None], knn)
    m64 = SF.Getters(*(v.double() for v in t[:3]), t[3][:, None].double(), knn)
    return m32, m64


def _bound(m64, x, rows, df, density_threshold=1.0, omc=1e-16):
    """Per-sample error bounds of a float32 evaluation against float64 on the same inputs.

    Per pair, with B = (sum_j 1 / clamp(s_j, 1e-8)) * |shift|_1 (>= the issue's sum_j inv_s_j sum_i |R_ij| |shift_i|, and it also
    covers the absolute rounding of R's entries): every w_j is a 3-term dot product of A (a few roundings per entry) and the shift
    (one rounding), so |dw_j| <= ~8 u inv_s_j |shift|_1 and |dq| <= dQ = 32 u B^2 + 4 u q.  exp is 1-Lipschitz in the exponent
    relative to its largest value on the interval: |de| <= e(q - dQ) min(dQ / 2, 1).  The opacity adds its own roundings
    (8 u o), the K-sum K u d.  The sdf path is bounded through the clamp (1-Lipschitz), log (1 / value), sqrt (Hoelder 1/2 at
    0) and the product with beta (mean of positive numbers, (K + 2) u relative)."""
    with torch.no_grad():
        pts, sc, q, st = m64.points, m64.scaling, m64.quaternions, m64.strengths[:, 0]
        x64 = x.double()
        shift = x64[:, None] - pts[rows]
        inv = 1.0 / sc.clamp(min=1e-8)
        B = inv[rows].sum(-1) * shift.abs().sum(-1)
        A = SF.quaternion_to_matrix(q) * inv[:, None]
        w = (A[rows].transpose(-1, -2) @ shift[..., None])[..., 0]
        qq = (w * w).sum(-1)
        qc = qq.clamp(0, 1e8)
        e = torch.exp(-0.5 * qc)
        dQ = 32 * U * B * B + 4 * U * qq
        e_hi = torch.exp(-0.5 * (qc - dQ).clamp(min=0))
        fs = df * st[rows]
        o = fs * e
        b_o = fs * (e_hi * (0.5 * dQ).clamp(max=1.0) + 8 * U * e) + 1e-38
        K = rows.shape[1]
        d = o.sum(-1)
        b_d = b_o.sum(-1) + 2 * K * U * d
        beta = sc.min(-1)[0][rows].mean(1)
        b_beta = (K + 2) * U * beta
        dh = torch.where(d >= 1, d / (d + 1e-12), d)
        ddh = b_d + 1.1e-12
        cd = dh.clamp(min=omc)
        cd_lo = torch.maximum(cd - ddh, torch.full_like(cd, omc * (1 - 2 * U)))
        m = -2 * torch.log(cd)
        dm = 2 * ddh / cd_lo + 4 * U * m.abs() + 8 * U
        sq = torch.sqrt(m)
        dsq = torch.minimum(torch.where(sq > 0, dm / (2 * sq.clamp(min=1e-300)), torch.full_like(sq, math.inf)), torch.sqrt(dm)) + 2 * U * sq
        c = float(np.sqrt(-2. * np.log(min(density_threshold, 1.))))
        dc = U * abs(c)
        b_sdf = beta * (dsq + dc) + (sq - c).abs() * b_beta + b_beta * (dsq + dc) + 2 * U * (beta * (sq - c)).abs()
    return {"density": b_d, "closest_gaussian_opacities": b_o + U * o, "beta": b_beta, "sdf": b_sdf}


FLAGS = [  # (return_sdf, return_beta, return_closest_gaussian_opacities, density_factor): the trainers' combinations
    (False, True, True, 1.0),        # coarse_density (sdf_estimation_mode 'density')
    (True, False, True, 1.0 / 16),   # coarse_sdf / refine (sdf_estimation_mode 'sdf')
    (True, False, False, 1.0 / 16),  # sdf without the better-normal loss
    (False, False, False, 1.0),      # density only
    (True, True, True, 1.0),         # everything, d >= 1 rows included
]


def _check_fields(got, want, bound, name):
    for k, b in bound.items():
        if k not in want:
            continue
        g, w = got[k].double(), want[k]
        assert g.shape == w.shape, (name, k)
        ok = (g - w).abs() <= b
        bad = (~ok).nonzero()
        assert ok.all(), "%s %s: %d rows over the bound, first %s: got %r want %r bound %r" % (
            name, k, bad.shape[0], bad[0].tolist(), g[tuple(bad[0])].item(), w[tuple(bad[0])].item(), b[tuple(bad[0])].item())


@pytest.mark.parametrize("K", [1, 4, 16, 32])
@pytest.mark.parametrize("N", [0, 1, 1000, 100_000])
def test_forward_within_the_error_bound_torch_float32_meets_too(K, N):
    sf = _sf()
    t, knn = _scene(4000 if N < 100_000 else 20_000, K, seed=K, edge_cases=True)
    m32, m64 = _models(t, knn)
    x, gidx = _samples(t[0], t[1], t[2], N, seed=N + K, edge_cases=True)
    rows = knn[gidx]
    for rs, rb, ro, df in FLAGS:
        kw = dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=df)
        got = sf.get_field_values(m32, x, gidx, **kw)
        want = SF.get_field_values(m64, x.double(), gidx, **kw)
        torch32 = SF.get_field_values(m32, x, gidx, **kw)
        assert list(got) == list(torch32)  # same keys, same order
        b = _bound(m64, x, rows, df)
        _check_fields(got, want, b, "cuda %s" % (kw,))
        _check_fields(torch32, want, b, "torch float32 %s" % (kw,))
        # explicit indices give the same values as the knn_idx[gaussian_idx] path
        again = sf.get_field_values(m32, x, closest_gaussians_idx=rows, **kw)
        for k in got:
            assert torch.equal(got[k], again[k]), k
    # compute_density, indices given and through the model's own search
    d, o = sf.compute_density(m32, x, rows, density_factor=0.5, return_closest_gaussian_opacities=True)
    dw, ow = SF.compute_density(m64, x.double(), rows, density_factor=0.5, return_closest_gaussian_opacities=True)
    b = _bound(m64, x, rows, 0.5)
    _check_fields({"density": d, "closest_gaussian_opacities": o}, {"density": dw, "closest_gaussian_opacities": ow}, b, "compute_density")
    if 0 < N <= 1000:
        d2 = sf.compute_density(m32, x)
        own = SF.get_gaussians_closest_to_samples(m32, x)
        assert torch.equal(d2, sf.compute_density(m32, x, own))


def test_edge_cases_forward_values():
    sf = _sf()
    t, knn = _scene(4000, 16, edge_cases=True)
    m32, _ = _models(t, knn)
    x, gidx = _samples(t[0], t[1], t[2], 1000, edge_cases=True)
    f = sf.get_field_values(m32, x, gidx, return_sdf=True, return_beta=True, return_closest_gaussian_opacities=True)
    # 16 coincident Gaussians of strength 1, samples on them: d = 16, normalised to exactly 1, sdf = beta * (0 - 0) = 0
    assert (f["density"][24:32] == 16).all() and (f["sdf"][24:32] == 0).all()
    # far samples: every exponential underflows, the density is 0 and clamped to 1e-16 before the log
    assert (f["density"][16:24] == 0).all()
    torch.testing.assert_close(f["sdf"][16:24], f["beta"][16:24] * math.sqrt(-2 * math.log(np.float32(1e-16))), rtol=1e-6, atol=0)
    # at a centre the own Gaussian contributes its strength
    o = f["closest_gaussian_opacities"]
    assert (o[:16, 0] == m32.strengths[knn[gidx[:16], 0], 0]).all()


def _grad_case(t, knn, N, seed, kw, weights_seed=5):
    """Gradients of a random linear functional of the requested fields with respect to x, points, scaling, quaternions and
    strengths: CUDA (float32), torch's float32 graph and float64 autograd."""
    sf = _sf()
    x, gidx = _samples(t[0], t[1], t[2], N, seed=seed)
    out = {}
    for name, dtype, fn in (("cuda", torch.float32, sf.get_field_values), ("torch32", torch.float32, SF.get_field_values),
                            ("f64", torch.float64, SF.get_field_values)):
        leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
        m = SF.Getters(*leaves[1:], knn)
        f = fn(m, leaves[0], gidx, **kw)
        loss = 0
        for i, k in enumerate(sorted(f)):
            w = torch.randn(f[k].shape, generator=torch.Generator().manual_seed(weights_seed + i)).to(DEV, dtype)
            loss = loss + (w * f[k]).sum()
        loss.backward()
        out[name] = [v.grad for v in leaves]
    return out


@pytest.mark.parametrize("K", [4, 16, 32])
@pytest.mark.parametrize("flags", FLAGS[:4], ids=["density", "sdf_opac", "sdf", "density_only"])
def test_gradients_of_the_five_inputs_against_float64(K, flags):
    rs, rb, ro, df = flags
    t, knn = _scene(3000, K, seed=7 + K)
    kw = dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=df)
    out = _grad_case(t, knn, 20_000, seed=K, kw=kw)
    names = ("x", "points", "scaling", "quaternions", "strengths")
    for i, n in enumerate(names):
        ref = out["f64"][i]
        tol = 1e-4 * ref.abs().max().item()
        for arm in ("cuda", "torch32"):
            g = out[arm][i]
            assert torch.isfinite(g).all(), (arm, n)
            err = (g.double() - ref).abs().max().item()
            assert err <= tol, "%s %s: max error %.3g > %.3g" % (arm, n, err, tol)


def test_sdf_gradient_is_non_finite_exactly_where_torch_is():
    """d >= 1 in the sdf path: d / (d + 1e-12) == 1 in float32, sqrt(-2 log 1) = 0 and sqrt's backward divides by it."""
    sf = _sf()
    t, knn = _scene(4000, 16, edge_cases=True)
    x, gidx = _samples(t[0], t[1], t[2], 2000, edge_cases=True)
    res = {}
    for name, fn in (("cuda", sf.get_field_values), ("torch32", SF.get_field_values)):
        leaves = [v.detach().clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
        m = SF.Getters(*leaves[1:], knn)
        f = fn(m, leaves[0], gidx, return_sdf=True, density_factor=1.0)
        f["sdf"].sum().backward()
        res[name] = (f["density"].detach(), [v.grad for v in leaves])
    d = res["cuda"][0]
    rows = torch.isfinite(res["cuda"][1][0]).all(1)
    rows_t = torch.isfinite(res["torch32"][1][0]).all(1)
    assert (~rows).any() and torch.equal(rows, rows_t)
    assert torch.equal(~rows, d >= 1)
    for i in range(1, 5):
        fin = torch.isfinite(res["cuda"][1][i]).reshape(res["cuda"][1][i].shape[0], -1).all(1)
        fin_t = torch.isfinite(res["torch32"][1][i]).reshape(res["torch32"][1][i].shape[0], -1).all(1)
        assert torch.equal(fin, fin_t), i


def _field_model(P, K, dtype, seed=3):
    from autovfx_b200 import scene
    g = scene.synthetic_gaussians(P, seed=seed, extent=(1, 1, 0.3), log_scale_mean=math.log(0.02), log_scale_std=0.4,
                                  opacity_mean=0.0, opacity_std=2.0)
    g = {k: v.to(DEV) for k, v in g.items()}
    knn = _knn(g["means3D"].contiguous(), K)
    return g, knn


@pytest.mark.parametrize("block", ["density", "sdf"])
def test_trainer_blocks_end_to_end(block):
    """coarse_density's and coarse_sdf's SDF blocks on a 20k-Gaussian stand-in: the method bound to the restatement (float64 and
    float32) versus the CUDA path; the loss and every raw leaf's gradient."""
    sf = _sf()
    g, knn = _field_model(20_000, 16, torch.float32)
    fn = SF.density_block if block == "density" else SF.sdf_block
    res = {}
    for name, dtype, method in (("f64", torch.float64, None), ("torch32", torch.float32, None),
                                ("cuda", torch.float32, sf.get_field_values)):
        m = SF.FieldModel(g, knn, dtype=dtype)
        if method is not None:
            m.get_field_values = method.__get__(m)
        x, gidx = SF.sample_points_in_gaussians(m, 100_000, 1.5, generator=torch.Generator().manual_seed(9))
        loss = fn(m, x, gidx)
        loss.backward()
        res[name] = (loss.item(), {k: v.grad.clone() for k, v in m.leaves.items() if v.grad is not None})
    l64, g64 = res["f64"]
    for arm in ("cuda", "torch32"):
        l, gr = res[arm]
        assert abs(l - l64) <= 1e-5 * abs(l64), (arm, l, l64)
        for k in ("_points", "all_densities", "_scales", "_quaternions"):
            ref = g64[k]
            err = (gr[k].double() - ref).abs().max().item()
            assert err <= 1e-4 * ref.abs().max().item(), "%s %s: %.3g vs max %.3g" % (arm, k, err, ref.abs().max().item())


def test_no_grad_saves_nothing_and_matches_the_graph_path():
    sf = _sf()
    t, knn = _scene(3000, 16)
    m32, _ = _models(t, knn)
    x, gidx = _samples(t[0], t[1], t[2], 5000)
    with torch.no_grad():
        a = sf.get_field_values(m32, x, gidx, return_beta=True, return_closest_gaussian_opacities=True)
    assert all(v.grad_fn is None for v in a.values())
    leaves = [v.clone().requires_grad_(True) for v in t]
    m = SF.Getters(leaves[0], leaves[1], leaves[2], leaves[3][:, None], knn)
    b = sf.get_field_values(m, x, gidx, return_beta=True, return_closest_gaussian_opacities=True)
    for k in a:
        assert torch.equal(a[k], b[k].detach()) and b[k].grad_fn is not None


def test_full_size_three_million_gaussians_one_million_samples():
    """config-3's 3M Gaussians, 1M samples, K = 16, forward and backward; forward rows and dL/dx on a stratified row sample
    against torch float32 evaluated on those rows, the per-Gaussian gradients against torch float32 on all rows."""
    sf = _sf()
    from autovfx_b200 import scene
    g = scene.config3_scene()
    t = [g["means3D"].to(DEV), g["scales"].to(DEV), torch.nn.functional.normalize(g["rotations"].to(DEV), dim=-1),
         g["opacities"].reshape(-1).to(DEV)]
    t = [v.contiguous() for v in t]
    knn = _knn(t[0], 16)
    x, gidx = _samples(t[0], t[1], t[2], 1_000_000, seed=4)
    kw = dict(return_sdf=True, return_beta=False, return_closest_gaussian_opacities=True, density_factor=1.0 / 16)
    gen = torch.Generator().manual_seed(6)
    w_sdf = torch.randn(1_000_000, generator=gen).to(DEV)
    w_d = torch.randn(1_000_000, generator=gen).to(DEV)
    grads = {}
    fields = {}
    for name, fn in (("cuda", sf.get_field_values), ("torch32", SF.get_field_values)):
        leaves = [v.detach().clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
        m = SF.Getters(*leaves[1:], knn)
        f = fn(m, leaves[0], gidx, **kw)
        ((w_sdf * f["sdf"]).sum() + (w_d * f["density"]).sum()).backward()
        grads[name] = [v.grad for v in leaves]
        fields[name] = {k: v.detach() for k, v in f.items()}
        del f, m, leaves
        torch.cuda.empty_cache()
    # stratified rows: 64 strata of 15,625 rows, 256 rows each
    rows = torch.cat([torch.randperm(15_625, generator=torch.Generator().manual_seed(s))[:256] + s * 15_625 for s in range(64)]).to(DEV)
    m64 = SF.Getters(*(v.double() for v in t[:3]), t[3][:, None].double(), knn)
    want = SF.get_field_values(m64, x[rows].double(), gidx[rows], **kw)
    b = _bound(m64, x[rows], knn[gidx[rows]], 1.0 / 16)
    _check_fields({k: v[rows] for k, v in fields["cuda"].items()}, want, b, "cuda full size")
    _check_fields({k: v[rows] for k, v in fields["torch32"].items()}, want, b, "torch32 full size")
    for i, n in enumerate(("x", "points", "scaling", "quaternions", "strengths")):
        a, r = grads["cuda"][i], grads["torch32"][i]
        if i == 0:
            a, r = a[rows], r[rows]
        assert torch.isfinite(a).all(), n
        err = (a - r).abs().max().item()
        assert err <= 2e-4 * r.abs().max().item(), "%s: %.3g vs max %.3g" % (n, err, r.abs().max().item())
