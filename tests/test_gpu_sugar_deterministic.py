"""SuGaR's regularisation backwards under torch.use_deterministic_algorithms(True): gsr_sugar_field_backward_det,
gsr_sugar_sdf_normal_backward_det and gsr_sugar_sample_backward_det.  Repeated backwards are bit-identical; the documented order
(ascending partial id per Gaussian, from +0.0) is pinned bit for bit by masking the output gradient to one sample, or one pair, at a
time and summing on the host; the values meet the default path's fp64 bounds; the edge rules hold; and a seeded coarse_density step
loop with the library's render, sampler, field, normal loss, densifier and Adam repeats bit for bit across processes."""
from __future__ import annotations

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import sugar_field_ref as SF  # noqa: E402
from tests import sugar_normal_ref as SN  # noqa: E402
from tests import sugar_sample_ref as SR  # noqa: E402
from tests import test_gpu_sugar_field as TF  # noqa: E402
from tests import test_gpu_sugar_normal as TN  # noqa: E402
from tests import test_gpu_sugar_sample as TS  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture
def deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was)


def _sf():
    from autovfx_b200 import sugar_field
    return sugar_field


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _assert_bits(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert (a is None) == (b is None), (what, i)
        if a is not None:
            assert torch.equal(_bits(a), _bits(b)), (what, i)


# ---- gradients of the three families ------------------------------------------------------------------------------------------------
def _field_grads(t, knn, x, gidx, kw, weights_seed=5, rows=None, grad_outputs=None):
    """dL/d(x, points, scaling, quaternions, strengths) of a random linear functional of the requested fields (or of the given
    per-output gradients)."""
    sf = _sf()
    leaves = [v.detach().clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
    m = SF.Getters(*leaves[1:], knn)
    f = sf.get_field_values(m, leaves[0], None if rows is not None else gidx, closest_gaussians_idx=rows, **kw)
    keys = sorted(f)
    if grad_outputs is None:
        grad_outputs = {k: torch.randn(f[k].shape, generator=torch.Generator().manual_seed(weights_seed + i)).to(DEV)
                        for i, k in enumerate(keys)}
    keys = [k for k in keys if k in grad_outputs]
    return list(torch.autograd.grad([f[k] for k in keys], leaves, [grad_outputs[k] for k in keys], allow_unused=True))


def _normal_grads(t, knn, x, gidx, o, loss, est, gl=None, ge=None, seed=3):
    """dL/d(x, points, quaternions) of sum(gl * loss) + sum(ge * estimate) (either term optional)."""
    sf = _sf()
    gen = torch.Generator().manual_seed(seed)
    N = x.shape[0]
    gl = torch.randn(N, generator=gen).to(DEV) if gl is None else gl
    ge = torch.randn(N, generator=gen).to(DEV) if ge is None else ge
    leaves = [v.detach().clone().requires_grad_(True) for v in (x, t[0], t[2])]
    m = SN.Getters(leaves[1], t[1], leaves[2], torch.ones(t[0].shape[0], 1, device=DEV), knn)
    outs, gos = [], []
    if loss:
        outs.append(sf.better_normal_loss(m, leaves[0], gidx, o))
        gos.append(gl)
    if est:
        outs.append(sf.projection_estimate(m, leaves[0], gidx))
        gos.append(ge)
    return list(torch.autograd.grad(outs, leaves, gos, allow_unused=True))


def _sample_case(P, N, seed=5, opacity=True, volume=True):
    points, scaling, quats, strengths = TS._scene(P, seed=seed, zero_volume=False)
    mask = TS._mask(P, seed=seed + 1)
    leaves = [v.clone().requires_grad_(True) for v in (points, scaling, quats)]
    model = SR.Getters(*leaves, strengths)
    x, idx = TS._call(model, N, 1.5, mask, opacity, volume, seed=seed + 2)
    return leaves, x, idx


def _sample_grads(leaves, x, g):
    return list(torch.autograd.grad([x], leaves, [g], retain_graph=True))


# ---- 1. repeatability ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 3, 16, 32])
def test_field_backwards_repeat_bitwise(deterministic, K):
    t, knn = TF._scene(3000, K, seed=20 + K, edge_cases=True)
    x, gidx = TF._samples(t[0], t[1], t[2], 20_000, seed=K, edge_cases=True)
    for rs, rb, ro, df in TF.FLAGS:
        kw = dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=df)
        want = _field_grads(t, knn, x, gidx, kw)
        for i in range(4):
            _assert_bits(_field_grads(t, knn, x, gidx, kw), want, (K, kw, i))


@pytest.mark.parametrize("terms", [(True, False), (False, True), (True, True)], ids=["loss", "estimate", "both"])
def test_normal_backwards_repeat_bitwise(deterministic, terms):
    t, knn = TN._scene(3000, 16, seed=4, edge_cases=True)
    x, gidx, o = TN._samples(*t, 20_000, 16, seed=4)
    want = _normal_grads(t, knn, x, gidx, o, *terms)
    for i in range(4):
        _assert_bits(_normal_grads(t, knn, x, gidx, o, *terms), want, (terms, i))


def test_sample_backwards_repeat_bitwise(deterministic):
    leaves, x, idx = _sample_case(4096, 200_000)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    want = _sample_grads(leaves, x, g)
    for i in range(4):
        _assert_bits(_sample_grads(leaves, x, g), want, i)


def test_field_bitwise_next_to_a_concurrent_stream(deterministic):
    t, knn = TF._scene(3000, 16, seed=2)
    x, gidx = TF._samples(t[0], t[1], t[2], 20_000, seed=2)
    kw = dict(return_sdf=False, return_beta=True, return_closest_gaussian_opacities=True, density_factor=1.0)
    want = _field_grads(t, knn, x, gidx, kw)
    tb, knnb = TF._scene(200_000, 16, seed=3)
    xb, gb = TF._samples(tb[0], tb[1], tb[2], 1_000_000, seed=3)
    side = torch.cuda.Stream()
    for i in range(3):
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            _field_grads(tb, knnb, xb, gb, kw)
        got = _field_grads(t, knn, x, gidx, kw)
        torch.cuda.synchronize()
        _assert_bits(got, want, i)


# ---- 2. the documented order, bit for bit ------------------------------------------------------------------------------------------
def _host_sum(parts):
    """Sequential float32 sum from +0.0 in the given order."""
    acc = np.zeros_like(parts[0])
    for p in parts:
        acc = (acc + p).astype(np.float32)
    return acc


def _small_field_scene(N=300, K=16, P=48):
    t, knn = TF._scene(P, K, seed=31)
    x, gidx = TF._samples(t[0], t[1], t[2], N, seed=32)
    return t, knn, x, gidx


def test_field_order_per_sample(deterministic):
    """Ascending n: one backward per sample (dL/ddensity and dL/dbeta masked to it), summed on the host in ascending n, equals
    the full backward for dL/dpoints and dL/dstrengths (density_factor = 1), which are the summed records before any chain."""
    t, knn, x, gidx = _small_field_scene()
    N = x.shape[0]
    kw = dict(return_sdf=False, return_beta=True, return_closest_gaussian_opacities=False, density_factor=1.0)
    gen = torch.Generator().manual_seed(7)
    gd, gb = torch.randn(N, generator=gen).to(DEV), torch.randn(N, generator=gen).to(DEV)
    full = _field_grads(t, knn, x, gidx, kw, grad_outputs={"density": gd, "beta": gb})
    hits = torch.bincount(knn[gidx].reshape(-1), minlength=t[0].shape[0])
    assert hits.double().mean() >= 24  # Gaussians collect dozens of partials
    parts = {1: [], 4: []}
    for n in range(N):
        m = torch.zeros(N, device=DEV)
        m[n] = 1
        g = _field_grads(t, knn, x, gidx, kw, grad_outputs={"density": gd * m, "beta": gb * m})
        for i in parts:
            parts[i].append(g[i].detach().cpu().numpy())
    for i in parts:
        want = _host_sum(parts[i])
        got = full[i].detach().cpu().numpy()
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), i


def test_field_order_within_a_sample(deterministic):
    """Ascending k within a sample: rows with repeated Gaussians, dL/dopacities masked to one (n, k) at a time."""
    t, knn, x, gidx = _small_field_scene(N=24, K=8)
    rows = knn[gidx].clone()
    rows[:, 4:] = rows[:, :4]  # every Gaussian of a row twice
    rows[::3, 1:] = rows[::3, :1]  # and a third of the rows all one Gaussian
    N, K = rows.shape
    kw = dict(return_sdf=False, return_beta=False, return_closest_gaussian_opacities=True, density_factor=1.0)
    go = torch.randn(N, K, generator=torch.Generator().manual_seed(8)).to(DEV)
    full = _field_grads(t, knn, x, gidx, kw, rows=rows, grad_outputs={"closest_gaussian_opacities": go})
    parts = {1: [], 4: []}
    for n in range(N):
        for k in range(K):
            m = torch.zeros(N, K, device=DEV)
            m[n, k] = 1
            g = _field_grads(t, knn, x, gidx, kw, rows=rows, grad_outputs={"closest_gaussian_opacities": go * m})
            for i in parts:
                parts[i].append(g[i].detach().cpu().numpy())
    for i in parts:
        assert np.array_equal(full[i].detach().cpu().numpy().view(np.int32), _host_sum(parts[i]).view(np.int32)), i


def test_normal_order_per_sample(deterministic):
    """The centre gradient sums own terms only, in ascending n: dL/dloss and dL/destimate masked to one sample at a time."""
    t, knn = TN._scene(48, 16, seed=33)
    x, gidx, o = TN._samples(*t, 300, 16, seed=34)
    N = x.shape[0]
    gen = torch.Generator().manual_seed(9)
    gl, ge = torch.randn(N, generator=gen).to(DEV), torch.randn(N, generator=gen).to(DEV)
    full = _normal_grads(t, knn, x, gidx, o, True, True, gl, ge)
    assert torch.bincount(gidx, minlength=48).max() >= 10
    parts = []
    for n in range(N):
        m = torch.zeros(N, device=DEV)
        m[n] = 1
        parts.append(_normal_grads(t, knn, x, gidx, o, True, True, gl * m, ge * m)[1].detach().cpu().numpy())
    assert np.array_equal(full[1].detach().cpu().numpy().view(np.int32), _host_sum(parts).view(np.int32))


def test_sample_order_per_sample(deterministic):
    leaves, x, idx = _sample_case(16, 400)
    N = x.shape[0]
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    full = _sample_grads(leaves, x, g)
    assert torch.bincount(idx, minlength=16).max() >= 24
    parts = [[] for _ in full]
    for n in range(N):
        m = torch.zeros(N, 1, device=DEV)
        m[n] = 1
        for i, v in enumerate(_sample_grads(leaves, x, g * m)):
            parts[i].append(v.detach().cpu().numpy())
    for i in range(3):
        assert np.array_equal(full[i].detach().cpu().numpy().view(np.int32), _host_sum(parts[i]).view(np.int32)), i


# ---- 3. accuracy --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [4, 16, 32])
def test_field_accuracy_against_float64_and_the_default_path(K):
    rs, rb, ro, df = TF.FLAGS[0]
    kw = dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=df)
    t, knn = TF._scene(3000, K, seed=7 + K)
    default = TF._grad_case(t, knn, 20_000, seed=K, kw=kw)  # the default path and fp64 autograd, flag off
    x, gidx = TF._samples(t[0], t[1], t[2], 20_000, seed=K)
    torch.use_deterministic_algorithms(True)
    try:
        det = _field_grads(t, knn, x, gidx, kw)  # the same functional
    finally:
        torch.use_deterministic_algorithms(False)
    for i in range(5):
        ref = default["f64"][i]
        tol = 1e-4 * ref.abs().max().item()
        assert torch.isfinite(det[i]).all()
        assert (det[i].double() - ref).abs().max().item() <= tol, i
        assert (det[i].double() - default["cuda"][i].double()).abs().max().item() <= tol, i


def test_normal_accuracy_against_float64_and_the_default_path():
    t, knn = TN._scene(3000, 16, seed=25, edge_cases=True)
    N, seed = 20_000, 16
    default = TN._grads(t, knn, N, 16, seed=seed)  # the default path and fp64 autograd, flag off
    x, gidx, o = TN._samples(*t, N, 16, seed=seed)
    gen = torch.Generator().manual_seed(seed + 1)
    gl, ge = torch.randn(N, generator=gen).to(DEV), torch.randn(N, generator=gen).to(DEV)
    torch.use_deterministic_algorithms(True)
    try:
        det = _normal_grads(t, knn, x, gidx, o, True, True, gl, ge)
    finally:
        torch.use_deterministic_algorithms(False)
    for i, n in enumerate(("x", "points", "quaternions")):
        TN._check_rows(det[i], default["f64"][i], n)
        TN._check_rows(det[i], default["cuda"][i].double(), n + " vs default")


@pytest.mark.parametrize("P,N,f", [(8, 50_000, 1.5), (4096, 200_000, 0.7)])
def test_sample_accuracy_against_float64_and_the_default_path(P, N, f):
    """test_gpu_sugar_sample's per-row fp64 bound, for the flag-on gradients and for their distance to the default path's."""
    points, scaling, quats, strengths = TS._scene(P, seed=P, zero_volume=False)
    mask = TS._mask(P, seed=P + 1)
    g = torch.randn(N, 3, generator=torch.Generator().manual_seed(P + 2)).to(DEV)
    grads = {}
    for det in (False, True):
        leaves = [v.clone().requires_grad_(True) for v in (points, scaling, quats)]
        x, idx = TS._call(SR.Getters(*leaves, strengths), N, f, mask, False, True, seed=31)
        torch.use_deterministic_algorithms(det)
        try:
            (x * g).sum().backward()
        finally:
            torch.use_deterministic_algorithms(False)
        grads[det] = [v.grad for v in leaves]
    _, z = SR.draws(N, DEV, 31)
    l64 = [v.detach().double().requires_grad_(True) for v in (points, scaling, quats)]
    (SR.place_pytorch3d(*l64, idx, z.double(), f) * g.double()).sum().backward()
    bound, hits = TS._row_bound(l64[1].detach(), l64[2].detach(), z, g, idx, f, P)
    assert hits.max() > 100
    for d, a, b in zip(grads[True], grads[False], l64):
        assert ((d.double() - b.grad).abs().amax(-1) <= bound).all()
        assert ((d.double() - a.double()).abs().amax(-1) <= 2 * bound).all()


# ---- 4. edges under the flag --------------------------------------------------------------------------------------------------------
def test_out_of_range_indices_add_nothing(deterministic):
    sf = _sf()
    t, knn = TN._scene(1000, 8, seed=6)
    x, gidx, o = TN._samples(*t, 200, 8, seed=6)
    gidx = gidx.clone()
    gidx[0], gidx[1] = -1, 1000
    knn = knn.clone()
    knn[int(gidx[10]), 3] = 5000
    xl = x.clone().requires_grad_(True)
    q, p = t[2].clone().requires_grad_(True), t[0].clone().requires_grad_(True)
    m = SN.Getters(p, t[1], q, torch.ones(1000, 1, device=DEV), knn)
    (sf.better_normal_loss(m, xl, gidx, o).nan_to_num().sum() + sf.projection_estimate(m, xl, gidx).nan_to_num().sum()).backward()
    assert torch.isfinite(q.grad).all() and torch.isfinite(p.grad).all()
    assert torch.isnan(xl.grad[:2]).all() and torch.isfinite(xl.grad[2:10]).all()
    # the field: a row with a Gaussian index outside the model
    t, knn = TF._scene(1000, 8, seed=6)
    x, gidx = TF._samples(t[0], t[1], t[2], 200, seed=6)
    rows = knn[gidx].clone()
    rows[5, 2] = 1000
    kw = dict(return_sdf=False, return_beta=True, return_closest_gaussian_opacities=True, density_factor=1.0)
    go = {"density": torch.ones(200, device=DEV), "beta": torch.ones(200, device=DEV)}
    g = _field_grads(t, knn, x, gidx, kw, rows=rows, grad_outputs=go)
    assert torch.isnan(g[0][5]).all() and torch.isfinite(g[0][:5]).all() and torch.isfinite(g[0][6:]).all()
    assert all(torch.isfinite(v).all() for v in g[1:])
    # the same backward with sample 5 dropped gives the same Gaussian gradients: it added nothing
    keep = torch.arange(200, device=DEV) != 5
    go2 = {k: v * keep for k, v in go.items()}
    rows2 = rows.clone()
    rows2[5] = rows2[4]
    g2 = _field_grads(t, knn, x, gidx, kw, rows=rows2, grad_outputs=go2)
    for a, b in zip(g[1:], g2[1:]):
        assert torch.equal(a, b)


def _lib():
    from autovfx_b200 import _lib
    return _lib


def _raw_field(t, knn, x, gidx, N, nan_fill=True, nbytes_delta=0):
    """gsr_sugar_field_backward_det called directly, outputs and scratch pre-filled with NaN."""
    L = _lib()
    P, K = t[0].shape[0], knn.shape[1]
    nan = float("nan")
    outs = [torch.full((N, 3), nan, device=DEV)] + [torch.full(s, nan, device=DEV) for s in ((P, 3), (P, 3), (P, 4), (P,))]
    nbytes = L.lib.gsr_sugar_field_backward_det_bytes(N, K, P)
    scratch = torch.full((nbytes + 256,), 255 if nan_fill else 0, dtype=torch.uint8, device=DEV)
    gd = torch.randn(max(N, 1), generator=torch.Generator().manual_seed(3)).to(DEV)
    rc = L.lib.gsr_sugar_field_backward_det(N, K, P, P, x.data_ptr(), knn.data_ptr(), gidx.data_ptr(), t[0].data_ptr(), t[1].data_ptr(),
                                            t[2].data_ptr(), t[3].data_ptr(), 1.0, 1e-16, 0.0, gd.data_ptr(), None, None, None,
                                            outs[0].data_ptr(), *[o.data_ptr() for o in outs[1:]], scratch.data_ptr(),
                                            nbytes + nbytes_delta, L.stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    return rc, outs


def test_unreached_gaussians_get_zero_and_nothing_unwritten_is_read(deterministic):
    t, knn = TF._scene(2000, 16, seed=12)
    x, gidx = TF._samples(t[0], t[1], t[2], 40, seed=12)  # 40 samples reach a small part of 2000 Gaussians
    gidx = gidx.contiguous()
    rc, outs = _raw_field(t, knn, x, gidx, 40)
    assert rc == 0
    reached = torch.zeros(2000, dtype=torch.bool, device=DEV)
    reached[knn[gidx].reshape(-1)] = True
    assert (~reached).sum() > 1000  # 40 * 16 pairs at most reach 640
    for o in outs:
        assert torch.isfinite(o).all()  # every row written, no NaN scratch byte read
    assert torch.equal(_bits(outs[1][~reached]), torch.zeros_like(_bits(outs[1][~reached])))  # +0.0 exactly
    assert torch.equal(_bits(outs[4][~reached]), torch.zeros_like(_bits(outs[4][~reached])))
    for o in outs[2:4]:
        assert (o[~reached] == 0).all()
    # the same call on a zeroed scratch gives the same bits
    rc, outs0 = _raw_field(t, knn, x, gidx, 40, nan_fill=False)
    _assert_bits(outs0, outs, "scratch contents")
    # one byte short: GSR_ERR_WORKSPACE and nothing enqueued (the NaN-filled outputs stay NaN)
    rc, outs1 = _raw_field(t, knn, x, gidx, 40, nbytes_delta=-1)
    assert rc == -2 and all(torch.isnan(o).all() for o in outs1)


def test_normal_and_sample_short_scratch_enqueue_nothing(deterministic):
    L = _lib()
    t, knn = TN._scene(500, 8, seed=13)
    x, gidx, o = TN._samples(*t, 100, 8, seed=13)
    P = 500
    g = torch.ones(100, device=DEV)
    outs = [torch.full(s, float("nan"), device=DEV) for s in ((100, 3), (P, 3), (P, 4))]
    need = L.lib.gsr_sugar_sdf_normal_backward_det_bytes(100, 8, P, 1)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    rc = L.lib.gsr_sugar_sdf_normal_backward_det(100, 8, P, x.data_ptr(), gidx.data_ptr(), knn.data_ptr(), t[0].data_ptr(), t[1].data_ptr(),
                                                 t[2].data_ptr(), o.data_ptr(), g.data_ptr(), None, *[v.data_ptr() for v in outs],
                                                 scratch.data_ptr(), need - 1, L.stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    assert rc == -2 and all(torch.isnan(v).all() for v in outs)
    idx = torch.randint(0, P, (100,), device=DEV)
    total = torch.ones(1, dtype=torch.float64, device=DEV)
    z = torch.randn(100, 3, device=DEV)
    need = L.lib.gsr_sugar_sample_backward_det_bytes(100, P)
    souts = [torch.full(s, float("nan"), device=DEV) for s in ((P, 3), (P, 3), (P, 4))]
    rc = L.lib.gsr_sugar_sample_backward_det(100, P, 1.5, idx.data_ptr(), z.data_ptr(), t[1].data_ptr(), t[2].data_ptr(), total.data_ptr(),
                                             x.data_ptr(), *[v.data_ptr() for v in souts],
                                             torch.empty(need, dtype=torch.uint8, device=DEV).data_ptr(), need - 1,
                                             L.stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    assert rc == -2 and all(torch.isnan(v).all() for v in souts)


def test_empty_inputs(deterministic):
    sf = _sf()
    t, knn = TF._scene(500, 8, seed=14)
    leaves = [v.clone().requires_grad_(True) for v in (t[0], t[1], t[2], t[3][:, None])]
    m = SF.Getters(*leaves, knn)
    x = torch.zeros(0, 3, device=DEV, requires_grad=True)
    f = sf.get_field_values(m, x, torch.zeros(0, dtype=torch.int64, device=DEV), return_sdf=False, return_beta=True)
    (f["density"].sum() + f["beta"].sum()).backward()
    for v in leaves:
        assert v.grad is None or (v.grad == 0).all()


@pytest.mark.parametrize("how", ["empty_mask", "zero_volume", "nan_scale"])
def test_zero_or_non_finite_total_gives_zero_gradients(deterministic, how):
    TS.test_empty_or_non_finite_total(how)


def test_sample_rows_never_drawn_get_zero(deterministic):
    leaves, x, idx = _sample_case(4096, 1000)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    grads = _sample_grads(leaves, x, g)
    drawn = torch.zeros(4096, dtype=torch.bool, device=DEV)
    drawn[idx] = True
    for v in grads:
        assert torch.equal(_bits(v[~drawn]), torch.zeros_like(_bits(v[~drawn])))


# ---- 5. a whole seeded coarse_density loop -------------------------------------------------------------------------------------------
def _coarse_loop(dev, steps=20):
    """coarse_density's iteration on a small seeded SuGaR stand-in: render_sugar_raw, the photometric loss and the entropy term,
    the SDF-regularisation block on samples drawn in the visible Gaussians (the library's sampler, field, projection estimate and
    better-normal loss), backward, the densification statistics, one densify-and-prune followed by a new knn_idx, the library's
    Adam."""
    import types
    from autovfx_b200 import densify, losses, sugar_field
    from autovfx_b200.knn import knn_points
    from autovfx_b200.optim import use_cuda_adam
    from autovfx_b200.renderer import render_sugar_raw
    from tests import test_gpu_sugar_render as TR
    model = TR._scene(dev, M=16, P=3000)
    model.beta_mode = "average"
    model.get_field_values = sugar_field.get_field_values.__get__(model)
    names = (("points", "_points"), ("all_densities", "all_densities"), ("scales", "_scales"), ("quaternions", "_quaternions"),
             ("sh_coordinates_dc", "_sh_coordinates_dc"), ("sh_coordinates_rest", "_sh_coordinates_rest"))
    lrs = {"points": 1.6e-4, "all_densities": 0.05, "scales": 5e-3, "quaternions": 1e-3, "sh_coordinates_dc": 2.5e-3,
           "sh_coordinates_rest": 1.25e-4}
    for _, a in names:
        setattr(model, a, torch.nn.Parameter(getattr(model, a).detach().clone()))
    opt = use_cuda_adam(torch.optim.Adam([{"params": [getattr(model, a)], "lr": lrs[n], "name": n} for n, a in names], lr=0.0, eps=1e-15))
    P = model.n_points
    dens = types.SimpleNamespace(model=model, optimizer=opt, points_gradient_accum=torch.zeros(P, 1, device=dev),
                                 denom=torch.zeros(P, 1, device=dev), max_radii2D=torch.zeros(P, device=dev), max_grad=2e-7,
                                 min_opacity=0.005, scene_extent=1.0, percent_dense=0.01, params_to_densify=[n for n, _ in names])
    model.knn_idx = knn_points(model.points[None], model.points[None], K=16).idx[0]
    gen = torch.Generator().manual_seed(5)
    gts = [torch.rand(TR.H, TR.W, 3, generator=gen).to(dev) for _ in range(4)]
    sizes = [P]
    for it in range(steps):
        out = render_sugar_raw(model, camera_indices=it % 4, bg_color=torch.zeros(3, device=dev), sh_deg=3, return_2d_radii=True)
        img = out["image"][..., :3]  # the RGB channels, as coarse_density's pred_rgb
        loss = losses.photometric_loss(img.permute(2, 0, 1), gts[it % 4].permute(2, 0, 1), 0.2)
        op = model.strengths
        loss = loss + 0.1 * (-op * torch.log(op + 1e-10) - (1 - op) * torch.log(1 - op + 1e-10)).mean()
        radii = out["radii"]
        x, gidx = sugar_field.sample_points_in_gaussians(model, 20_000, 1.5, mask=radii > 0)
        loss = loss + SN.density_block(model, x, gidx, estimate=sugar_field.projection_estimate,
                                       normal_loss=sugar_field.better_normal_loss)
        loss.backward()
        with torch.no_grad():
            densify.update_densification_stats(dens, out["viewspace_points"], radii, radii > 0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        if it == steps // 2:
            with torch.no_grad():
                densify.sugar_densify_and_prune(dens, max_screen_size=None)
                model.knn_idx = knn_points(model.points[None], model.points[None], K=16).idx[0]
            sizes.append(model.n_points)
    res = {"sizes": np.asarray(sizes)}
    for n, a in names:
        p = getattr(model, a)
        res[n] = p.detach().cpu().numpy()
        st = opt.state[p]
        res[n + "/exp_avg"], res[n + "/exp_avg_sq"] = st["exp_avg"].cpu().numpy(), st["exp_avg_sq"].cpu().numpy()
    return res


def test_coarse_density_loop_is_bit_identical(tmp_path):
    outs = []
    for i in range(2):
        path = tmp_path / ("coarse%d.npz" % i)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--coarse-worker", str(path)]
        res = subprocess.run(cmd, env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"), cwd=ROOT, capture_output=True, text=True,
                             timeout=900)
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        outs.append(dict(np.load(path)))
    a, b = outs
    assert a["sizes"][1] != a["sizes"][0], a["sizes"]  # the densification changed the Gaussian count
    assert sorted(a) == sorted(b)
    for k in a:
        va, vb = a[k], b[k]
        assert va.shape == vb.shape, k
        assert np.array_equal(va.view(np.int32) if va.dtype == np.float32 else va, vb.view(np.int32) if vb.dtype == np.float32 else vb), k


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--coarse-worker":
    torch.use_deterministic_algorithms(True)
    torch.manual_seed(0)
    np.savez(sys.argv[2], **_coarse_loop(torch.device("cuda:0")))
