"""GPU tests of autovfx_b200.sugar_field's projection_estimate and better_normal_loss (gsr_sugar_sdf_normal and its backward)
against the trainer's code restated in torch (tests/sugar_normal_ref.py): the forward against float64 within an error bound
derived below, which torch's own float32 graph must meet too; the gradients against float64 autograd; edge cases; coarse_density's
whole regularisation block end to end; one full-size call."""
import math

import pytest
import torch

from tests import sugar_normal_ref as SN

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # float32 unit roundoff
DEV = "cuda"
DN = 32 * U     # |n_f32 - n_f64| per component: quaternion_to_matrix of a unit q, about a dozen roundings of terms <= 2
BAND = 1e-4     # |n_j . n_i| below this may take another sign under another rounding order


def _sf():
    from autovfx_b200 import sugar_field
    return sugar_field


def _knn(points, K):
    from autovfx_b200.knn import knn_points
    return knn_points(points[None], points[None], K=K).idx[0]


def _scene(P, K, seed=0, edge_cases=False):
    """Getter outputs (float32) of a SuGaR-like scene and its neighbour table.  With edge_cases: 2- and 3-way scale ties, scales
    below the 1e-6 clamp, and a block of axis-aligned Gaussians whose normals are exactly orthogonal or parallel."""
    g = torch.Generator().manual_seed(seed)
    points = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([1.0, 1.0, 0.3])
    log_s = math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g)
    quats = torch.randn(P, 4, generator=g)
    if edge_cases:
        log_s[20:40] = math.log(1e-8)          # below the 1e-6 clamp of the min scale
        log_s[40:80] = log_s[40:80, :1]        # three-way ties
        log_s[80:120, 2] = log_s[80:120, 1]    # two-way ties of the min at indices 1 and 2
        log_s[80:120, 0] = log_s[80:120, 1] + 0.5
        quats[120:120 + P // 8] = torch.tensor([1.0, 0, 0, 0])  # axis-aligned: normals are exact unit axes
        log_s[120:120 + P // 8] = math.log(0.02)
        axis = torch.randint(0, 3, (P // 8,), generator=g)
        log_s[torch.arange(120, 120 + P // 8), axis] = math.log(0.005)
        points[120:120 + P // 8] = points[120:120 + P // 8] * 0.05  # packed together, so they are each other's neighbours
    scaling = torch.exp(log_s)
    quats = torch.nn.functional.normalize(quats, dim=-1)
    t = [v.to(DEV).contiguous() for v in (points, scaling, quats)]
    K = min(K, P)
    return t, _knn(t[0], K)


def _samples(points, scaling, quats, N, K, seed=1):
    """Samples drawn like sample_points_in_gaussians, and opacities [N,K] with some exact zeros."""
    g = torch.Generator().manual_seed(seed)
    P = points.shape[0]
    idx = torch.randint(0, P, (N,), generator=g).to(DEV)
    v = 1.5 * scaling[idx] * torch.randn(N, 3, generator=g).to(DEV)
    x = points[idx] + (SN.sugar_ref.quaternion_to_matrix(quats[idx]) @ v[..., None])[..., 0]
    o = torch.rand(N, K, generator=g)
    o[o < 0.05] = 0
    return x.contiguous(), idx, o.to(DEV)


def _models(t, knn):
    strengths = torch.ones(t[0].shape[0], 1, device=DEV)
    m32 = SN.Getters(t[0], t[1], t[2], strengths, knn)
    m64 = SN.Getters(*(v.double() for v in t), strengths.double(), knn)
    return m32, m64


def _bound(m64, x, gidx, o, sign):
    """Per-sample error bounds of a float32 evaluation against float64 on the same inputs and the same sign decisions.

    Normals: DN per component.  A 3-term dot with a difference x - p (one rounding per component) and |n| <= 1: 3 u for the
    products and sums, DN + u for the normal and the difference, so |dd| <= 6 DN |x - p|_1 with room to spare; the estimate is
    that dot.  w = (o d) / c: its own 2 roundings, c's one, and o |dd| / c.  The K-sum of non-negative terms adds K u S.  w_hat
    = w / max(S, 1e-6) moves by (e_w + w_hat e_S) / max(S - e_S, 1e-6) + 2 u w_hat; T_c = sum_j w_hat_j n'_jc by
    sum_j (e_wh_j + w_hat_j (DN + 2 u)) + K u sum_j w_hat_j |n'_jc|; r_c by DN + e_T + u |r_c|; the loss by
    sum_c (2 |r_c| e_r + e_r^2) + 4 u loss.  The first-order expansion drops products of errors: the bound is doubled."""
    with torch.no_grad():
        n = SN.get_normals(m64)
        p = m64.points
        x = x.double()
        di = x - p[gidx]
        est = (di * n[gidx]).sum(-1)
        b_est = 2 * (6 * DN * di.abs().sum(-1) + 2 * U * est.abs()) + 1e-30
        idx = m64.knn_idx[gidx]
        s = sign.double()
        nj = n[idx] * s[..., None]
        dj = x[:, None] - p[idx]
        d = (dj * nj).sum(-1).abs()
        e_d = 6 * DN * dj.abs().sum(-1) * s.abs()
        c = m64.scaling.min(-1)[0][idx].clamp(min=1e-6) ** 2
        o = o.double()
        w = o * d / c
        e_w = o * e_d / c + 3 * U * w
        K = idx.shape[1]
        S = w.sum(-1, keepdim=True)
        e_S = e_w.sum(-1, keepdim=True) + K * U * S
        wh = w / S.clamp(min=1e-6)
        e_wh = (e_w + wh * e_S) / (S - e_S).clamp(min=1e-6) + 2 * U * wh
        T = (wh[..., None] * nj).sum(-2)
        e_T = (e_wh + wh * (DN + 2 * U)).sum(-1, keepdim=True) + K * U * (wh[..., None] * nj.abs()).sum(-2)
        r = n[gidx] - T
        e_r = DN + e_T + U * r.abs()
        loss = (r * r).sum(-1)
        b_loss = 2 * ((2 * r.abs() * e_r + e_r * e_r).sum(-1) + 4 * U * loss) + 1e-30
    return b_loss, b_est


def _check(got, want, bound, name, rows=None):
    g = got.double()
    ok = (g - want).abs() <= bound
    if rows is not None:
        ok = ok | ~rows
    bad = (~ok).nonzero()
    assert ok.all(), "%s: %d rows over the bound, first %d: got %r want %r bound %r" % (
        name, bad.shape[0], bad[0].item(), g[bad[0]].item(), want[bad[0]].item(), bound[bad[0]].item())


def _outside_band(m32, gidx):
    n = SN.get_normals(m32, pinned=True)
    idx = m32.knn_idx[gidx]
    return (SN.dot3(n[idx], n[gidx][:, None]).abs() > BAND).all(-1)


@pytest.mark.parametrize("K", [1, 4, 16, 32])
@pytest.mark.parametrize("N", [0, 1, 1000, 100_000])
def test_forward_within_the_error_bound_torch_float32_meets_too(K, N):
    sf = _sf()
    t, knn = _scene(4000 if N < 100_000 else 20_000, K, seed=K, edge_cases=True)
    m32, m64 = _models(t, knn)
    x, gidx, o = _samples(*t, N, K, seed=N + K)
    sign = SN.pinned_signs(m32, gidx)
    loss = sf.better_normal_loss(m32, x, gidx, o)
    est = sf.projection_estimate(m32, x, gidx)
    assert loss.shape == (N,) and est.shape == (N,) and loss.dtype == est.dtype == torch.float32
    if N == 0:  # SuGaR's .view(len(sdf_samples), -1) cannot take 0 samples (the trainer skips the block then)
        return
    want_loss = SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign)
    want_est = SN.projection_estimate(m64, x.double(), gidx)
    b_loss, b_est = _bound(m64, x, gidx, o, sign)
    _check(loss, want_loss, b_loss, "cuda loss K=%d N=%d" % (K, N))
    _check(est, want_est, b_est, "cuda estimate K=%d N=%d" % (K, N))
    # torch's own float32 graph meets the same bound wherever its sign decisions cannot differ from the pinned ones
    rows = _outside_band(m32, gidx)
    _check(SN.better_normal_loss(m32, x, gidx, o), want_loss, b_loss, "torch float32 loss", rows)
    _check(SN.projection_estimate(m32, x, gidx), want_est, b_est, "torch float32 estimate")


def test_the_bound_sees_a_wrong_sign():
    """A sign decision other than the pinned one moves the loss far outside the bound (so the bound checks the decisions)."""
    t, knn = _scene(4000, 16, seed=3)
    m32, m64 = _models(t, knn)
    x, gidx, o = _samples(*t, 2000, 16, seed=3)
    sign = SN.pinned_signs(m32, gidx)
    flipped = sign.clone()
    flipped[:, 1] = -flipped[:, 1]
    want = SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign)
    moved = SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=flipped)
    b_loss, _ = _bound(m64, x, gidx, o, sign)
    assert ((moved - want).abs() > b_loss).float().mean() > 0.5


def test_orthogonal_normals_drop_the_neighbour():
    """Axis-aligned Gaussians: normals are exact unit axes, sign(n_j . n_i) = 0 for a perpendicular neighbour."""
    sf = _sf()
    P = 512
    g = torch.Generator().manual_seed(5)
    points = (torch.rand(P, 3, generator=g) * 0.2).to(DEV)
    scaling = torch.full((P, 3), 0.02)
    scaling[torch.arange(P), torch.randint(0, 3, (P,), generator=g)] = 0.005
    quats = torch.zeros(P, 4)
    quats[:, 0] = 1
    t = [points, scaling.to(DEV), quats.to(DEV)]
    knn = _knn(points, 8)
    m32, m64 = _models(t, knn)
    x, gidx, o = _samples(*t, 5000, 8, seed=5)
    sign = SN.pinned_signs(m32, gidx)
    assert (sign == 0).float().mean() > 0.3
    loss = sf.better_normal_loss(m32, x, gidx, o)
    want = SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign)
    b_loss, _ = _bound(m64, x, gidx, o, sign)
    _check(loss, want, b_loss, "axis-aligned")


def test_all_zero_opacities():
    sf = _sf()
    t, knn = _scene(2000, 16, seed=2)
    m32, _ = _models(t, knn)
    x, gidx, o = _samples(*t, 3000, 16, seed=2)
    loss = sf.better_normal_loss(m32, x, gidx, torch.zeros_like(o))
    n = SN.get_normals(m32, pinned=True)[gidx]
    assert torch.equal(loss, SN.dot3(n, n))  # every weight 0: r = n_i


def test_scale_ties_and_tiny_scales_give_the_lowest_index_axis():
    sf = _sf()
    t, knn = _scene(4000, 1, seed=4, edge_cases=True)
    m32, _ = _models(t, knn)
    gidx = torch.arange(20, 120, device=DEV)  # tiny scales, 3-way and 2-way ties
    x = t[0][gidx] + 0.01
    n = SN.get_normals(m32, pinned=True)[gidx]
    want = SN.dot3(x - t[0][gidx], n)
    assert torch.equal(sf.projection_estimate(m32, x, gidx), want)
    k = t[1][gidx].min(-1)[1]
    assert (k[20:60] == 0).all() and (k[60:100] == 1).all()


def test_out_of_range_indices_give_nan_and_read_nothing():
    sf = _sf()
    t, knn = _scene(1000, 8, seed=6)
    m32, _ = _models(t, knn)
    x, gidx, o = _samples(*t, 200, 8, seed=6)
    gidx = gidx.clone()
    gidx[0], gidx[1], gidx[2] = -1, 1000, 1 << 40
    bad_row = int(gidx[10])
    knn = knn.clone()
    knn[bad_row, 3] = 5000
    m32.knn_idx = knn
    rows_bad = (gidx < 0) | (gidx >= 1000) | (gidx == bad_row)
    loss = sf.better_normal_loss(m32, x, gidx, o)
    est = sf.projection_estimate(m32, x, gidx)
    assert torch.isnan(loss[rows_bad]).all() and torch.isfinite(loss[~rows_bad]).all()
    assert torch.isnan(est[:3]).all() and torch.isfinite(est[3:]).all()
    # the backward: bad samples add nothing and get a NaN dL/dx; everything else stays finite
    xl = x.clone().requires_grad_(True)
    q = t[2].clone().requires_grad_(True)
    p = t[0].clone().requires_grad_(True)
    m = SN.Getters(p, t[1], q, m32.strengths, knn)
    (sf.better_normal_loss(m, xl, gidx, o).nan_to_num().sum() + sf.projection_estimate(m, xl, gidx).nan_to_num().sum()).backward()
    assert torch.isfinite(q.grad).all() and torch.isfinite(p.grad).all()
    assert torch.isnan(xl.grad[:3]).all() and torch.isfinite(xl.grad[3:]).all()
    torch.cuda.synchronize()


def test_single_gaussian():
    sf = _sf()
    t, knn = _scene(1, 1, seed=7)
    m32, m64 = _models(t, knn)
    x, gidx, o = _samples(*t, 50, 1, seed=7)
    sign = SN.pinned_signs(m32, gidx)
    assert (sign == 1).all()
    b_loss, b_est = _bound(m64, x, gidx, o, sign)
    _check(sf.better_normal_loss(m32, x, gidx, o), SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign), b_loss, "P=1")
    _check(sf.projection_estimate(m32, x, gidx), SN.projection_estimate(m64, x.double(), gidx), b_est, "P=1 estimate")


def test_no_grad_equals_the_graph_path_and_calls_repeat_bitwise():
    sf = _sf()
    t, knn = _scene(3000, 16, seed=8)
    m32, _ = _models(t, knn)
    x, gidx, o = _samples(*t, 5000, 16, seed=8)
    with torch.no_grad():
        a = (sf.better_normal_loss(m32, x, gidx, o), sf.projection_estimate(m32, x, gidx))
    assert all(v.grad_fn is None for v in a)
    leaves = [v.clone().requires_grad_(True) for v in (x, t[0], t[2])]
    m = SN.Getters(leaves[1], t[1], leaves[2], m32.strengths, knn)
    b = (sf.better_normal_loss(m, leaves[0], gidx, o), sf.projection_estimate(m, leaves[0], gidx))
    c = (sf.better_normal_loss(m, leaves[0], gidx, o), sf.projection_estimate(m, leaves[0], gidx))
    for u, v, w in zip(a, b, c):
        assert v.grad_fn is not None and torch.equal(u, v.detach()) and torch.equal(v, w)


def _grads(t, knn, N, K, seed):
    """dL/dx, dL/dpoints, dL/dquaternions of sum(g_l loss) + sum(g_e est): CUDA (float32) and float64 autograd of the restatement
    with the pinned sign decisions."""
    sf = _sf()
    x, gidx, o = _samples(*t, N, K, seed=seed)
    m32, _ = _models(t, knn)
    sign = SN.pinned_signs(m32, gidx)
    gen = torch.Generator().manual_seed(seed + 1)
    gl = torch.randn(N, generator=gen).to(DEV)
    ge = torch.randn(N, generator=gen).to(DEV)
    out = {}
    for name, dtype in (("cuda", torch.float32), ("f64", torch.float64)):
        leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in (x, t[0], t[2])]
        m = SN.Getters(leaves[1], t[1].to(dtype), leaves[2], torch.ones(t[0].shape[0], 1, device=DEV, dtype=dtype), knn)
        if name == "cuda":
            loss, est = sf.better_normal_loss(m, leaves[0], gidx, o), sf.projection_estimate(m, leaves[0], gidx)
        else:
            loss = SN.better_normal_loss(m, leaves[0], gidx, o.double(), sign=sign)
            est = SN.projection_estimate(m, leaves[0], gidx)
        ((gl.to(dtype) * loss).sum() + (ge.to(dtype) * est).sum()).backward()
        out[name] = [v.grad for v in leaves]
    return out


def _check_rows(g, ref, name, rtol=1e-3, atol_frac=2e-4):
    """Per row: max |g - ref| <= rtol * max |ref_row| + atol_frac * max |ref|."""
    g, ref = g.double().reshape(g.shape[0], -1), ref.reshape(ref.shape[0], -1)
    assert torch.isfinite(g).all(), name
    err = (g - ref).abs().max(-1)[0]
    tol = rtol * ref.abs().max(-1)[0] + atol_frac * ref.abs().max()
    bad = (err > tol).nonzero()
    assert bad.numel() == 0, "%s: %d rows over, first %d: err %.3g tol %.3g" % (name, bad.shape[0], bad[0].item(), err[bad[0]].item(),
                                                                              tol[bad[0]].item())


@pytest.mark.parametrize("K", [4, 16, 32])
def test_gradients_against_float64(K):
    t, knn = _scene(3000, K, seed=9 + K, edge_cases=True)
    out = _grads(t, knn, 20_000, K, seed=K)
    for i, n in enumerate(("x", "points", "quaternions")):
        _check_rows(out["cuda"][i], out["f64"][i], "%s K=%d" % (n, K))


def test_loss_reaches_only_the_quaternions():
    sf = _sf()
    t, knn = _scene(2000, 16, seed=10)
    x, gidx, o = _samples(*t, 4000, 16, seed=10)
    leaves = [v.clone().requires_grad_(True) for v in (x, t[0], t[1], t[2])]
    oo = o.clone().requires_grad_(True)
    m = SN.Getters(leaves[1], leaves[2], leaves[3], torch.ones(2000, 1, device=DEV), knn)
    sf.better_normal_loss(m, leaves[0], gidx, oo).sum().backward()
    assert leaves[0].grad is None and leaves[1].grad is None and leaves[2].grad is None and oo.grad is None
    assert leaves[3].grad is not None and leaves[3].grad.abs().sum() > 0


def test_coarse_density_block_end_to_end():
    """coarse_density's regularisation block on a 20k-Gaussian stand-in, 100k samples: the field, the estimate and the normal
    term all on the library against the block restated in float64; the loss and every raw leaf's gradient."""
    sf = _sf()
    from autovfx_b200 import scene
    g = scene.synthetic_gaussians(20_000, seed=3, extent=(1, 1, 0.3), log_scale_mean=math.log(0.02), log_scale_std=0.4,
                                  opacity_mean=0.0, opacity_std=2.0)
    g = {k: v.to(DEV) for k, v in g.items()}
    knn = _knn(g["means3D"].contiguous(), 16)
    m32 = SN.FieldModel(g, knn, dtype=torch.float32, grad=False)
    x32, gidx = SN.sample_points_in_gaussians(m32, 100_000, 1.5, generator=torch.Generator().manual_seed(9))
    sign = SN.pinned_signs(m32, gidx)
    res = {}
    for name, dtype in (("f64", torch.float64), ("cuda", torch.float32)):
        m = SN.FieldModel(g, knn, dtype=dtype)
        x, gi = SN.sample_points_in_gaussians(m, 100_000, 1.5, generator=torch.Generator().manual_seed(9))
        assert torch.equal(gi, gidx)
        if name == "cuda":
            m.get_field_values = sf.get_field_values.__get__(m)
            loss = SN.density_block(m, x, gi, estimate=sf.projection_estimate, normal_loss=sf.better_normal_loss)
        else:
            loss = SN.density_block(m, x, gi, sign=sign)
        loss.backward()
        res[name] = (loss.item(), {k: v.grad.clone() for k, v in m.leaves.items() if v.grad is not None})
    l64, g64 = res["f64"]
    l, gr = res["cuda"]
    assert abs(l - l64) <= 1e-5 * abs(l64), (l, l64)
    for k in ("_points", "all_densities", "_scales", "_quaternions"):
        ref = g64[k]
        err = (gr[k].double() - ref).abs().max().item()
        assert err <= 1e-4 * ref.abs().max().item(), "%s: %.3g vs max %.3g" % (k, err, ref.abs().max().item())


def test_full_size_three_million_gaussians_one_million_samples():
    """config-3's 3M Gaussians, knn_idx from knn_points(K = 16), 1M samples drawn as tools/bench_sugar_field.py draws them, the
    opacities from the library's field: forward rows on a stratified sample and the gradients of a sampled set of Gaussians
    against float64, nothing NaN."""
    sf = _sf()
    from autovfx_b200 import scene
    g = scene.config3_scene()
    t = [g["means3D"].to(DEV), g["scales"].to(DEV), torch.nn.functional.normalize(g["rotations"].to(DEV), dim=-1)]
    t = [v.contiguous() for v in t]
    strengths = g["opacities"].reshape(-1, 1).to(DEV).contiguous()
    knn = _knn(t[0], 16)
    N = 1_000_000
    gen = torch.Generator().manual_seed(0)
    gidx = torch.randint(0, t[0].shape[0], (N,), generator=gen).to(DEV)
    noise = torch.randn(N, 3, generator=gen).to(DEV)
    x = t[0][gidx] + (SN.sugar_ref.quaternion_to_matrix(t[2][gidx]) @ (1.5 * t[1][gidx] * noise)[..., None])[..., 0]
    m32 = SN.Getters(t[0], t[1], t[2], strengths, knn)
    with torch.no_grad():
        o = sf.get_field_values(m32, x, gidx, return_sdf=False, return_closest_gaussian_opacities=True)["closest_gaussian_opacities"]
    sign = SN.pinned_signs(m32, gidx)
    gen = torch.Generator().manual_seed(1)
    gl = torch.randn(N, generator=gen).to(DEV)
    ge = torch.randn(N, generator=gen).to(DEV)
    grads, outs = {}, {}
    for name, dtype in (("cuda", torch.float32), ("f64", torch.float64)):
        leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in (x, t[0], t[2])]
        m = SN.Getters(leaves[1], t[1].to(dtype), leaves[2], strengths.to(dtype), knn)
        if name == "cuda":
            loss, est = sf.better_normal_loss(m, leaves[0], gidx, o), sf.projection_estimate(m, leaves[0], gidx)
        else:
            loss = SN.better_normal_loss(m, leaves[0], gidx, o.double(), sign=sign)
            est = SN.projection_estimate(m, leaves[0], gidx)
        ((gl.to(dtype) * loss).sum() + (ge.to(dtype) * est).sum()).backward()
        grads[name] = [v.grad for v in leaves]
        outs[name] = (loss.detach(), est.detach())
        del loss, est, m, leaves
        torch.cuda.empty_cache()
    assert not torch.isnan(outs["cuda"][0]).any() and not torch.isnan(outs["cuda"][1]).any()
    for gcu in grads["cuda"]:
        assert not torch.isnan(gcu).any()
    # stratified rows: 64 strata of 15,625 rows, 1,024 rows each
    rows = torch.cat([torch.randperm(15_625, generator=torch.Generator().manual_seed(s))[:1024] + s * 15_625 for s in range(64)]).to(DEV)
    m64 = SN.Getters(*(v.double() for v in t), strengths.double(), knn)
    b_loss, b_est = _bound(m64, x[rows], gidx[rows], o[rows], sign[rows])
    _check(outs["cuda"][0][rows], outs["f64"][0][rows], b_loss, "full-size loss")
    _check(outs["cuda"][1][rows], outs["f64"][1][rows], b_est, "full-size estimate")
    _check_rows(grads["cuda"][0][rows], grads["f64"][0][rows], "full-size x")
    gs = torch.randperm(t[0].shape[0], generator=torch.Generator().manual_seed(2))[:65_536].to(DEV)
    _check_rows(grads["cuda"][1][gs], grads["f64"][1][gs], "full-size points")
    _check_rows(grads["cuda"][2][gs], grads["f64"][2][gs], "full-size quaternions")
