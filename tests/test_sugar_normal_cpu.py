"""CPU tests of the better-normal loss and projection estimate restatement (tests/sugar_normal_ref.py) and of the host side of
autovfx_b200.sugar_field's projection_estimate / better_normal_loss: the restatement's quirks in float64, the closed-form
gradients the kernels implement against float64 autograd, the wrapper's argument errors (raised before any device is touched)
and the C-ABI validation."""
import os
import re

import pytest
import torch

from tests import sugar_normal_ref as SN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _getters(P=12, K=4, dtype=F64, seed=0):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(P, 3, generator=g, dtype=dtype)
    sc = torch.rand(P, 3, generator=g, dtype=dtype) * 0.5 + 0.1
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g, dtype=dtype), dim=-1)
    st = torch.rand(P, 1, generator=g, dtype=dtype)
    knn = torch.stack([torch.roll(torch.arange(P), -s) for s in range(K)], 1)
    return SN.Getters(pts, sc, q, st, knn)


def _axis_model(scales, points=None):
    """Identity rotations: Gaussian g's normal is the unit axis of its smallest scale."""
    P = len(scales)
    q = torch.zeros(P, 4, dtype=F64)
    q[:, 0] = 1
    pts = torch.zeros(P, 3, dtype=F64) if points is None else torch.tensor(points, dtype=F64)
    return SN.Getters(pts, torch.tensor(scales, dtype=F64), q, torch.ones(P, 1, dtype=F64), None)


def test_sign_zero_drops_a_neighbour():
    m = _axis_model([[1.0, 1.0, 0.1], [0.1, 1.0, 1.0]], points=[[0, 0, 0], [1, 0, 0]])
    m.knn_idx = torch.tensor([[0, 1], [1, 0]])
    x = torch.tensor([[0.3, 0.2, 0.5]], dtype=F64)
    gidx = torch.tensor([0])
    assert SN.pinned_signs(m, gidx).tolist() == [[1.0, 0.0]]
    o = torch.tensor([[0.5, 0.9]], dtype=F64)
    # the orthogonal neighbour gets weight 0, so w_hat of the own Gaussian is 1 and r = n_0 - n_0 = 0
    assert SN.better_normal_loss(m, x, gidx, o).item() == 0.0
    # with the neighbour kept (sigma forced to 1) the loss is not 0
    assert SN.better_normal_loss(m, x, gidx, o, sign=torch.ones(1, 2, dtype=F64)).item() > 0


def test_weight_sum_below_the_clamp():
    m = _axis_model([[1.0, 1.0, 0.1]])
    m.knn_idx = torch.tensor([[0]])
    x = torch.tensor([[0.0, 0.0, 0.5]], dtype=F64)
    o = torch.tensor([[1e-10]], dtype=F64)
    w = 1e-10 * 0.5 / 0.1 ** 2  # 5e-9 < 1e-6: w_hat = w / 1e-6
    torch.testing.assert_close(SN.better_normal_loss(m, x, torch.tensor([0]), o), torch.tensor([(1 - w / 1e-6) ** 2], dtype=F64))
    # all-zero opacities: every weight is 0 and the loss is |n_i|^2 = 1
    assert SN.better_normal_loss(m, x, torch.tensor([0]), torch.zeros(1, 1, dtype=F64)).item() == 1.0


def test_min_scale_below_the_clamp():
    # the own Gaussian (min scale 1e-9, clamped to 1e-6) and a tilted neighbour (min scale 1e-3): w = o d / clamp(s, 1e-6)^2
    m = _axis_model([[1.0, 1.0, 1e-9], [1.0, 1.0, 1e-3]], points=[[0, 0, 0], [0, 0, -1]])
    m.knn_idx = torch.tensor([[0, 1], [1, 0]])
    m.quaternions = torch.tensor([[1.0, 0, 0, 0], [0.9, 0.1, 0, 0]], dtype=F64)
    x = torch.tensor([[0.0, 0.0, 1.0]], dtype=F64)
    o = torch.ones(1, 2, dtype=F64)
    n1 = SN.get_normals(m)[1]
    d0, d1 = 1.0, abs(float((x[0] - m.points[1]) @ n1))
    w0, w1 = d0 / 1e-12, d1 / 1e-6
    r = m.quaternions.new_tensor([0, 0, 1.0]) - (w0 * m.quaternions.new_tensor([0, 0, 1.0]) + w1 * n1) / (w0 + w1)
    torch.testing.assert_close(SN.better_normal_loss(m, x, torch.tensor([0]), o), (r * r).sum()[None], rtol=1e-12, atol=0)


def test_scale_ties_pick_the_lowest_index():
    g = torch.Generator().manual_seed(3)
    q = torch.nn.functional.normalize(torch.randn(4, 4, generator=g, dtype=F64), dim=-1)
    s = torch.tensor([[0.2, 0.2, 0.5], [0.5, 0.2, 0.2], [0.3, 0.3, 0.3], [0.4, 0.5, 0.4]], dtype=F64)
    m = SN.Getters(torch.zeros(4, 3, dtype=F64), s, q, torch.ones(4, 1, dtype=F64), None)
    R = SN.sugar_ref.quaternion_to_matrix(q)
    want = torch.stack([R[0, :, 0], R[1, :, 1], R[2, :, 0], R[3, :, 0]])
    assert torch.equal(SN.get_normals(m), want)
    torch.testing.assert_close(SN.get_normals(m, pinned=True), want, rtol=0, atol=1e-15)


def _closed_form(m, x, gidx, o, sign):
    """The kernels' formulas: dL/dn [P,3] of sum(g_l * loss) + sum(g_e * est), and dL/dx, dL/dp of the estimate."""
    P = m.points.shape[0]
    n = SN.get_normals(m).detach()
    p = m.points.detach()
    idx = m.knn_idx[gidx]
    ni, nj = n[gidx], n[idx] * sign[..., None]
    d = ((x[:, None] - p[idx]) * nj).sum(-1).abs()
    c = m.scaling.detach().min(-1)[0][idx].clamp(min=1e-6) ** 2
    w = o * d / c
    wh = w / w.sum(-1, keepdim=True).clamp(min=1e-6)
    r = ni - (wh[..., None] * nj).sum(-2)
    gen = torch.Generator().manual_seed(11)
    gl = torch.randn(x.shape[0], generator=gen, dtype=F64)
    ge = torch.randn(x.shape[0], generator=gen, dtype=F64)
    dn = torch.zeros(P, 3, dtype=F64)
    dn.index_add_(0, gidx, 2 * gl[:, None] * r)
    dn.index_add_(0, idx.reshape(-1), (-2 * gl[:, None, None] * wh[..., None] * sign[..., None] * r[:, None]).reshape(-1, 3))
    dn.index_add_(0, gidx, ge[:, None] * (x - p[gidx]))
    dx = ge[:, None] * ni
    dp = torch.zeros(P, 3, dtype=F64).index_add_(0, gidx, -ge[:, None] * ni)
    return gl, ge, dn, dx, dp


def test_closed_form_gradients_against_float64_autograd():
    m = _getters(P=40, K=6)
    g = torch.Generator().manual_seed(2)
    gidx = torch.randint(0, 40, (300,), generator=g)
    x = (m.points[gidx] + 0.1 * torch.randn(300, 3, generator=g, dtype=F64)).requires_grad_(True)
    o = torch.rand(300, 6, generator=g, dtype=F64)
    for t in (m.points, m.quaternions):
        t.requires_grad_(True)
    sign = SN.pinned_signs(m, gidx)
    gl, ge, dn, dx, dp = _closed_form(m, x.detach(), gidx, o, sign)
    loss = (gl * SN.better_normal_loss(m, x, gidx, o, sign=sign)).sum() + (ge * SN.projection_estimate(m, x, gidx)).sum()
    ax, ap, aq = torch.autograd.grad(loss, (x, m.points, m.quaternions))
    # dL/dq from dL/dn through get_normals' own graph
    want_q = torch.autograd.grad(SN.get_normals(m), m.quaternions, dn)[0]
    torch.testing.assert_close(ax, dx, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ap, dp, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(aq, want_q, rtol=1e-10, atol=1e-12)
    # the loss alone reaches neither x nor the points
    lx, lp = torch.autograd.grad(SN.better_normal_loss(m, x, gidx, o, sign=sign).sum(), (x, m.points), allow_unused=True)
    assert (lx is None or (lx == 0).all()) and (lp is None or (lp == 0).all())


# ------------------------------------------------------------------------------------------------ the wrapper's errors
def _cpu_model(P=8, K=4):
    return _getters(P=P, K=K, dtype=torch.float32)


@pytest.mark.parametrize("kwargs, match", [
    (dict(sdf_samples=torch.zeros(3, 3, dtype=F64)), "sdf_samples must be torch.float32"),
    (dict(sdf_samples=torch.zeros(3, 4)), "sdf_samples must have shape"),
    (dict(sdf_gaussian_idx=torch.arange(3, dtype=torch.int32)), "sdf_gaussian_idx must be torch.int64"),
    (dict(sdf_gaussian_idx=torch.arange(4)), "sdf_gaussian_idx must have shape"),
    (dict(closest_gaussian_opacities=torch.zeros(3, 5)), "closest_gaussian_opacities must have shape \\[3, 4\\]"),
    (dict(closest_gaussian_opacities=torch.zeros(3, 4, dtype=F64)), "closest_gaussian_opacities must be torch.float32"),
    (dict(closest_gaussian_opacities=None), "closest_gaussian_opacities must be a torch.Tensor"),
])
def test_better_normal_loss_argument_errors(kwargs, match):
    from autovfx_b200.sugar_field import better_normal_loss
    m = _cpu_model()
    args = dict(sdf_samples=torch.zeros(3, 3), sdf_gaussian_idx=torch.arange(3), closest_gaussian_opacities=torch.zeros(3, 4))
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        better_normal_loss(m, **args)


def test_model_errors():
    from autovfx_b200.sugar_field import better_normal_loss, projection_estimate
    x, gidx, o = torch.zeros(3, 3), torch.arange(3), torch.zeros(3, 4)
    m = _cpu_model()
    m.knn_idx = m.knn_idx.to(torch.int32)
    with pytest.raises(ValueError, match="self.knn_idx must be torch.int64"):
        better_normal_loss(m, x, gidx, o)
    m = _cpu_model()
    m.knn_idx = m.knn_idx[:5]
    with pytest.raises(ValueError, match="self.knn_idx must have shape \\[8, \\*\\]"):
        better_normal_loss(m, x, gidx, o)
    m = _getters(P=8, K=33, dtype=torch.float32)
    with pytest.raises(ValueError, match="K = 33"):
        better_normal_loss(m, x, gidx, torch.zeros(3, 33))
    m = _cpu_model()
    m.quaternions = torch.ones(8, 3)
    with pytest.raises(ValueError, match="self.quaternions"):
        projection_estimate(m, x, gidx)
    m = _cpu_model()
    m.binded_to_surface_mesh = True
    for fn, args in ((projection_estimate, (x, gidx)), (better_normal_loss, (x, gidx, o))):
        with pytest.raises(ValueError, match="surface mesh"):
            fn(m, *args)


def test_cpu_tensors_raise_runtime_error():
    from autovfx_b200.sugar_field import better_normal_loss, projection_estimate
    m = _cpu_model()
    with pytest.raises(RuntimeError, match="no CPU path"):
        projection_estimate(m, torch.zeros(3, 3), torch.arange(3))
    with pytest.raises(RuntimeError, match="no CPU path"):
        better_normal_loss(m, torch.zeros(3, 3), torch.arange(3), torch.zeros(3, 4))


# ------------------------------------------------------------------------------------------------ exports and the C ABI
def test_sdf_normal_exports():
    from autovfx_b200 import _lib, sugar_field
    names = {"gsr_sugar_sdf_normal_bytes", "gsr_sugar_sdf_normal", "gsr_sugar_sdf_normal_backward"}
    assert names <= set(_lib.EXPORTS) and _lib.ABI_VERSION == 4
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsr_b200.h")).read(), flags=re.S)
    for n in names:
        assert re.search(r"\b%s\(" % n, hdr)
    L = _lib.lib
    assert L.gsr_abi_version() == 4
    assert len(L.gsr_sugar_sdf_normal.argtypes) == 15 and len(L.gsr_sugar_sdf_normal_backward.argtypes) == 18
    assert L.gsr_sugar_sdf_normal_bytes(1000) == 32 * 1000 and L.gsr_sugar_sdf_normal_bytes(0) == 0
    assert L.gsr_sugar_sdf_normal_bytes(-3) == 0
    assert set(sugar_field.__all__) >= {"projection_estimate", "better_normal_loss"}


def _fwd(L, N=10, K=16, P=100, x=256, gidx=256, knn=256, pts=256, sc=256, q=256, o=256, loss=256, est=None, ws=256, nbytes=1 << 30):
    return L.gsr_sugar_sdf_normal(N, K, P, x, gidx, knn, pts, sc, q, o, loss, est, ws, nbytes, None)


def test_c_abi_rejects_bad_arguments_before_any_launch():
    from autovfx_b200 import _lib
    L = _lib.lib
    # every call below fails validation (or is a no-op) before anything is launched or dereferenced
    for kw, msg in [(dict(N=-1), b"negative"), (dict(P=-2), b"negative"), (dict(K=0), b"K = 0"), (dict(K=33), b"K = 33"),
                    (dict(x=None), b"without its inputs"), (dict(gidx=None), b"without its inputs"),
                    (dict(q=None, loss=None, est=256), b"without its inputs"), (dict(knn=None), b"needs knn_idx"),
                    (dict(o=None), b"needs knn_idx")]:
        assert _fwd(L, **kw) == -1, kw
        assert msg in L.gsr_last_error(), (kw, L.gsr_last_error())
    assert _fwd(L, ws=None) == -2 and b"workspace" in L.gsr_last_error()
    assert _fwd(L, ws=264) == -2 and b"aligned" in L.gsr_last_error()
    assert _fwd(L, nbytes=32 * 100 - 1) == -2
    assert _fwd(L, N=0, x=None, gidx=None, knn=None, pts=None, sc=None, q=None, o=None, ws=None) == 0  # N = 0 is a no-op
    # the estimate alone needs neither knn_idx nor the opacities; no output at all is a no-op
    assert _fwd(L, knn=None, o=None, loss=None, est=256, ws=None) == -2
    assert _fwd(L, loss=None, est=None) == 0

    def bw(N=10, gl=256, ge=None, dp=256, dq=256, nbytes=1 << 30, knn=256):
        return L.gsr_sugar_sdf_normal_backward(N, 16, 100, 256, 256, knn, 256, 256, 256, 256, gl, ge, None, dp, dq, 256, nbytes, None)
    assert bw(dp=None) == -1 and b"required" in L.gsr_last_error()
    assert bw(dq=None) == -1 and b"required" in L.gsr_last_error()
    assert bw(nbytes=32 * 100) == -2 and b"workspace" in L.gsr_last_error()  # the backward needs twice the forward's bytes
    assert bw(knn=None) == -1 and b"needs knn_idx" in L.gsr_last_error()
    assert bw(N=-1) == -1
