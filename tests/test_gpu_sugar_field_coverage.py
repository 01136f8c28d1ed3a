"""GPU tests of gsr_sugar_field and gsr_sugar_sdf_normal (forward and backward) where the kernels' structure can go wrong and
the older tests do not look: every segment width W = pow2 >= K with idle lanes inside the segment, the last warp and block
partial, the field's chain-rule branches (the 1 / clamp(s, 1e-8) mask, the lowest index of a min-scale tie, coincident
Gaussians, samples at centres and far away, beta and sdf together), non-unit quaternions, the C-ABI combinations the Python
wrapper never issues, heavily shared Gaussians, and out-of-range indices.

Forward values are held to the per-sample float64 bounds derived in test_gpu_sugar_field.py and test_gpu_sugar_normal.py
(torch's float32 graph must meet them too).  Gradients are held per Gaussian by ``_grad_rule``; combinations that must not
change a number are compared bitwise on scenes where every Gaussian is in at most one pair, so that no atomic order differs."""
import functools
import math

import numpy as np
import pytest
import torch

from tests import helpers as Hh
from tests import sugar_field_ref as SF
from tests import sugar_normal_ref as SN
from tests.test_gpu_sugar_field import FLAGS, _bound as _field_bound, _check_fields, _samples as _field_samples, _scene as _field_scene
from tests.test_gpu_sugar_normal import _bound as _normal_bound, _check, _outside_band, _samples as _normal_samples
from tests.test_gpu_sugar_normal import _scene as _normal_scene

pytestmark = pytest.mark.gpu

DEV = "cuda"
UNSET = 7.0  # what an output holds before a call: a number, so that an unwritten value is never taken for a NaN
# Gradient rule: per-row relative errors against float64 (Hh.row_errors), CUDA <= GRAD_FACTOR[q] * torch float32 + GRAD_FLOOR
# at the 50th, 99th and 100th percentiles.  Both arms round the same operations in float32 in different orders (K-sums, atomics).
# Over the 350 gradient tensors of this file on an H100 the largest ratio was 1.55 at q50 and q99, hence 3 there; at q100 it is
# one row, the worst-conditioned (cancellation), whose error is the condition number times an order-dependent rounding: ratios
# reached 5.3, hence 10.  A misplaced or missing term costs a relative error of order 1 in its rows.
GRAD_FACTOR, GRAD_FLOOR = {0.5: 3.0, 0.99: 3.0, 1.0: 10.0}, 2e-6
FIELD_NAMES = ("x", "points", "scaling", "quaternions", "strengths")
NORMAL_NAMES = ("x", "points", "quaternions")
UNUSED = 64  # the last UNUSED Gaussians of a gradient scene are in no row


def _sf():
    from autovfx_b200 import sugar_field
    return sugar_field


def _L():
    from autovfx_b200 import _lib
    return _lib.lib, _lib.stream_ptr(torch.device(DEV)), _lib.check


def _p(t):
    return None if t is None else t.data_ptr()


def _grad_rule(name, g, g32, g64, factor=GRAD_FACTOR, floor=GRAD_FLOOR):
    """g (the kernel's), g32 (torch's float32 graph) against g64, per row; see GRAD_FACTOR."""
    assert torch.isfinite(g).all(), "%s: not finite" % name
    if float(g64.abs().max()) == 0.0:
        assert float(g.abs().max()) == 0.0, name
        return
    e, e32 = Hh.row_errors(g, g64), Hh.row_errors(g32, g64)
    for q, f in factor.items():
        got, base = float(np.quantile(e, q)), float(np.quantile(e32, q))
        assert got <= f * base + floor, "%s: q%g per-row error %.3g, torch float32 %.3g" % (name, 100 * q, got, base)


def _denormalise(q, seed):
    """Quaternions scaled to norms in [0.3, 3] (quaternion_to_matrix divides by |q|^2, so R is unchanged)."""
    g = torch.Generator().manual_seed(seed)
    s = 0.3 * 10.0 ** torch.rand(q.shape[0], 1, generator=g)
    return (q * s.to(q.device)).contiguous()


# ------------------------------------------------------------------------------------------------ scenes
@functools.lru_cache(maxsize=None)
def _fscene(P, K, seed, unit=True):
    """The field's edge-case scene (test_gpu_sugar_field._scene) plus two-way min-scale ties at indices 1 and 2 (120:160) and
    the last UNUSED Gaussians taken out of the neighbour table."""
    t, knn = _field_scene(P, K, seed=seed, edge_cases=True)
    t = [v.clone() for v in t]
    t[1][120:160, 2] = t[1][120:160, 1]
    t[1][120:160, 0] = t[1][120:160, 1] * 1.5
    if not unit:
        t[2] = _denormalise(t[2], seed)
    knn = torch.where(knn >= P - UNUSED, knn - UNUSED, knn) if P > 2 * UNUSED else knn
    return t, knn.contiguous()


@functools.lru_cache(maxsize=None)
def _nscene(P, K, seed, unit=True):
    t, knn = _normal_scene(P, K, seed=seed, edge_cases=True)
    t = [v.clone() for v in t]
    if not unit:
        t[2] = _denormalise(t[2], seed)
    return t, knn


def _unique_scene(N, K, seed, extra_rows=5):
    """Every Gaussian in at most one (sample, neighbour) pair, so that per-Gaussian gradients are one term each and bitwise
    reproducible.  rows [R,K] (R = N + extra_rows) is a permutation of the P = R K Gaussians, row_idx [N] a permutation of rows;
    the Gaussians of a sample's row lie around it."""
    g = torch.Generator().manual_seed(seed)
    R = N + extra_rows
    P = R * K
    rows = torch.randperm(P, generator=g).reshape(R, K)
    row_idx = torch.randperm(R, generator=g)[:N]
    x = torch.rand(N, 3, generator=g) * 4 - 2
    anchor = torch.rand(R, 3, generator=g) * 4 - 2
    anchor[row_idx] = x
    points = torch.empty(P, 3)
    points[rows.reshape(-1)] = anchor.repeat_interleave(K, 0) + 0.03 * torch.randn(P, 3, generator=g)
    scaling = torch.exp(math.log(0.02) + 0.5 * torch.randn(P, 3, generator=g))
    quats = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    strengths = torch.sigmoid(2 * torch.randn(P, generator=g))
    t = [v.to(DEV).contiguous() for v in (points, scaling, quats, strengths)]
    return t, x.to(DEV).contiguous(), rows.to(DEV).contiguous(), row_idx.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------ direct C-ABI calls
def _field_fwd(t, x, rows, row_idx, df, outs, omc=1e-16, offset=0.0):
    """gsr_sugar_field with the outputs named in outs ('density', 'opac', 'beta', 'sdf'); the others are NULL."""
    L, st, check = _L()
    N, K = x.shape[0], rows.shape[1]
    P, R = t[0].shape[0], rows.shape[0]
    res = {k: torch.full((N, K) if k == "opac" else (N,), UNSET, device=DEV) for k in outs}
    nbytes = L.gsr_sugar_field_bytes(P)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=DEV)
    check(L.gsr_sugar_field(N, K, P, R, x.data_ptr(), rows.data_ptr(), _p(row_idx), *[v.data_ptr() for v in t], df, omc, offset,
                            *[_p(res.get(k)) for k in ("density", "opac", "beta", "sdf")], ws.data_ptr(), nbytes, st), "gsr_sugar_field")
    torch.cuda.synchronize()
    return res


def _field_bwd(t, x, rows, row_idx, df, grads, want_dx=True, omc=1e-16, offset=0.0):
    """gsr_sugar_field_backward with the output gradients in grads (keys as in _field_fwd, missing = NULL) -> [dx or None,
    d_points, d_scaling, d_quaternions, d_strengths]."""
    L, st, check = _L()
    N, K = x.shape[0], rows.shape[1]
    P, R = t[0].shape[0], rows.shape[0]
    dx = torch.full_like(x, UNSET) if want_dx else None
    d = [torch.full_like(v, UNSET) for v in t]
    nbytes = 2 * L.gsr_sugar_field_bytes(P)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=DEV)
    check(L.gsr_sugar_field_backward(N, K, P, R, x.data_ptr(), rows.data_ptr(), _p(row_idx), *[v.data_ptr() for v in t], df, omc,
                                     offset, *[_p(grads.get(k)) for k in ("density", "opac", "beta", "sdf")], _p(dx),
                                     *[v.data_ptr() for v in d], ws.data_ptr(), nbytes, st), "gsr_sugar_field_backward")
    torch.cuda.synchronize()
    return [dx] + d


def _normal_fwd(t, x, gidx, knn, o, want_loss, want_est):
    L, st, check = _L()
    N, P = x.shape[0], t[0].shape[0]
    K = knn.shape[1] if knn is not None else 1
    loss = torch.full((N,), UNSET, device=DEV) if want_loss else None
    est = torch.full((N,), UNSET, device=DEV) if want_est else None
    nbytes = L.gsr_sugar_sdf_normal_bytes(P)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=DEV)
    check(L.gsr_sugar_sdf_normal(N, K, P, x.data_ptr(), gidx.data_ptr(), _p(knn), t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(),
                                 _p(o), _p(loss), _p(est), ws.data_ptr(), nbytes, st), "gsr_sugar_sdf_normal")
    torch.cuda.synchronize()
    return loss, est


def _normal_bwd(t, x, gidx, knn, o, gl, ge):
    L, st, check = _L()
    N, P = x.shape[0], t[0].shape[0]
    K = knn.shape[1] if knn is not None else 1
    dx, dp, dq = torch.full_like(x, UNSET), torch.full_like(t[0], UNSET), torch.full_like(t[2], UNSET)
    nbytes = 2 * L.gsr_sugar_sdf_normal_bytes(P)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=DEV)
    check(L.gsr_sugar_sdf_normal_backward(N, K, P, x.data_ptr(), gidx.data_ptr(), _p(knn), t[0].data_ptr(), t[1].data_ptr(),
                                          t[2].data_ptr(), _p(o), _p(gl), _p(ge), dx.data_ptr(), dp.data_ptr(), dq.data_ptr(),
                                          ws.data_ptr(), nbytes, st), "gsr_sugar_sdf_normal_backward")
    torch.cuda.synchronize()
    return dx, dp, dq


# ------------------------------------------------------------------------------------------------ 1. forward at every width
WIDTH_K = [1, 2, 3, 5, 7, 8, 9, 13, 15, 16, 17, 24, 31, 32]
WIDTH_N = [1, 3, 257, 10_007]


@pytest.mark.parametrize("K", WIDTH_K)
def test_field_forward_at_every_width(K):
    """Every FLAGS combination and compute_density, N such that the last warp and block are partial at every W."""
    sf = _sf()
    t, knn = _fscene(4000, K, seed=K)
    m32, m64 = SF.Getters(t[0], t[1], t[2], t[3][:, None], knn), SF.Getters(*(v.double() for v in t[:3]), t[3][:, None].double(), knn)
    for N in WIDTH_N:
        x, gidx = _field_samples(t[0], t[1], t[2], N, seed=N + 100 * K, edge_cases=True)
        rows = knn[gidx]
        for rs, rb, ro, df in FLAGS:
            kw = dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=df)
            got = sf.get_field_values(m32, x, gidx, **kw)
            want = SF.get_field_values(m64, x.double(), gidx, **kw)
            b = _field_bound(m64, x, rows, df)
            _check_fields(got, want, b, "cuda K=%d N=%d %s" % (K, N, kw))
            _check_fields(SF.get_field_values(m32, x, gidx, **kw), want, b, "torch float32 K=%d N=%d %s" % (K, N, kw))
        d, o = sf.compute_density(m32, x, rows, density_factor=0.5, return_closest_gaussian_opacities=True)
        dw, ow = SF.compute_density(m64, x.double(), rows, density_factor=0.5, return_closest_gaussian_opacities=True)
        _check_fields({"density": d, "closest_gaussian_opacities": o}, {"density": dw, "closest_gaussian_opacities": ow},
                      _field_bound(m64, x, rows, 0.5), "compute_density K=%d N=%d" % (K, N))


@pytest.mark.parametrize("K", WIDTH_K)
def test_normal_forward_at_every_width(K):
    """The loss and the estimate through the wrapper, and the estimate alone through the C ABI with knn_idx [P,K] given, which
    runs at W = 1 whatever K: bitwise the wrapper's estimate."""
    sf = _sf()
    t, knn = _nscene(4000, K, seed=K)
    m32 = SN.Getters(t[0], t[1], t[2], torch.ones(4000, 1, device=DEV), knn)
    m64 = SN.Getters(*(v.double() for v in t), torch.ones(4000, 1, device=DEV, dtype=torch.float64), knn)
    for N in WIDTH_N:
        x, gidx, o = _normal_samples(*t, N, K, seed=N + 100 * K)
        sign = SN.pinned_signs(m32, gidx)
        loss, est = sf.better_normal_loss(m32, x, gidx, o), sf.projection_estimate(m32, x, gidx)
        want_loss = SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign)
        want_est = SN.projection_estimate(m64, x.double(), gidx)
        b_loss, b_est = _normal_bound(m64, x, gidx, o, sign)
        _check(loss, want_loss, b_loss, "cuda loss K=%d N=%d" % (K, N))
        _check(est, want_est, b_est, "cuda estimate K=%d N=%d" % (K, N))
        _check(SN.better_normal_loss(m32, x, gidx, o), want_loss, b_loss, "torch float32 loss K=%d N=%d" % (K, N),
               _outside_band(m32, gidx))
        _check(SN.projection_estimate(m32, x, gidx), want_est, b_est, "torch float32 estimate K=%d N=%d" % (K, N))
        _, est_k = _normal_fwd(t, x, gidx, knn, o, False, True)
        assert torch.equal(est_k, est), (K, N)


# ------------------------------------------------------------------------------------------------ 2, 3. gradients per Gaussian
GRAD_K = [1, 2, 3, 5, 8, 9, 16, 17, 31, 32]
GRAD_FLAGS = {"density": FLAGS[0], "sdf_opac": FLAGS[1], "sdf": FLAGS[2], "density_only": FLAGS[3], "beta_sdf": (True, True, False, None)}


def _field_grads(t, knn, N, seed, kw, rows=None):
    """Gradients of a random linear functional of the requested fields with respect to x, points, scaling, quaternions and
    strengths on the field's edge-case samples: CUDA, torch float32 and float64.  rows: explicit closest_gaussians_idx [N,K]
    (the row_idx == NULL path) instead of knn_idx[gidx]."""
    sf = _sf()
    x, gidx = _field_samples(t[0], t[1], t[2], N, seed=seed, edge_cases=True)
    out = {}
    for name, dtype, fn in (("cuda", torch.float32, sf.get_field_values), ("torch32", torch.float32, SF.get_field_values),
                            ("f64", torch.float64, SF.get_field_values)):
        leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
        m = SF.Getters(*leaves[1:], knn)
        f = fn(m, leaves[0], gidx, **kw) if rows is None else fn(m, leaves[0], closest_gaussians_idx=rows, **kw)
        loss = 0
        for i, k in enumerate(sorted(f)):
            w = torch.randn(f[k].shape, generator=torch.Generator().manual_seed(seed + 31 * i)).to(DEV, dtype)
            loss = loss + (w * f[k]).sum()
        loss.backward()
        out[name] = [v.grad for v in leaves]
    return out


def _field_grad_kw(flags, K):
    rs, rb, ro, df = flags
    # with the sdf, d < 1 everywhere (density_factor * sum of K strengths <= 0.9), so that every gradient is finite
    return dict(return_sdf=rs, return_beta=rb, return_closest_gaussian_opacities=ro, density_factor=0.9 / K if rs else df)


def _check_field_grads(out, tag, referenced=None, scaling=None, beta=False):
    for i, n in enumerate(FIELD_NAMES):
        _grad_rule("%s %s" % (tag, n), out["cuda"][i], out["torch32"][i], out["f64"][i])
    if referenced is not None:  # a Gaussian no sample references gets exactly 0
        for i in range(1, 5):
            assert torch.count_nonzero(out["cuda"][i][~referenced]) == 0, (tag, FIELD_NAMES[i])
    if scaling is not None:  # a scale below the clamp that is not the (lowest-index) min gets exactly 0
        ds = out["cuda"][2]
        below = scaling < 1e-8
        below[torch.arange(scaling.shape[0], device=DEV), scaling.min(-1)[1]] = False
        assert below.any()
        assert torch.count_nonzero(ds[below]) == 0, tag
        if beta:  # ... and the min of a sub-clamp Gaussian gets beta's gradient alone, which is not 0 where it is referenced
            km = scaling.min(-1)[1]
            tiny = (scaling < 1e-8).all(-1) & referenced
            assert torch.count_nonzero(ds[tiny, km[tiny]]) > 0, tag


@pytest.mark.parametrize("K", GRAD_K)
@pytest.mark.parametrize("flags", list(GRAD_FLAGS), ids=list(GRAD_FLAGS))
def test_field_gradients_per_gaussian_at_every_width(K, flags):
    P = 3000
    t, knn = _fscene(P, K, seed=7 + K)
    kw = _field_grad_kw(GRAD_FLAGS[flags], K)
    N = 20_000
    out = _field_grads(t, knn, N, seed=K, kw=kw)
    _, gidx = _field_samples(t[0], t[1], t[2], N, seed=K, edge_cases=True)
    referenced = torch.zeros(P, dtype=torch.bool, device=DEV)
    referenced[knn[gidx].reshape(-1)] = True
    assert not referenced[-UNUSED:].any()
    _check_field_grads(out, "K=%d %s" % (K, flags), referenced, t[1], beta=kw["return_beta"] or kw["return_sdf"])


@pytest.mark.parametrize("K", [3, 16])
@pytest.mark.parametrize("flags", ["density", "beta_sdf"])
def test_field_non_unit_quaternions(K, flags):
    """Norms in [0.3, 3]: the forward within the bounds, the gradients (through quat_to_matrix_vjp's -t^2 su q term) by the rule."""
    sf = _sf()
    t, knn = _fscene(3000, K, seed=40 + K, unit=False)
    assert (t[2].norm(dim=-1) - 1).abs().max() > 0.5
    kw = _field_grad_kw(GRAD_FLAGS[flags], K)
    m32, m64 = SF.Getters(t[0], t[1], t[2], t[3][:, None], knn), SF.Getters(*(v.double() for v in t[:3]), t[3][:, None].double(), knn)
    x, gidx = _field_samples(t[0], t[1], t[2], 5000, seed=3, edge_cases=True)
    want = SF.get_field_values(m64, x.double(), gidx, **kw)
    b = _field_bound(m64, x, knn[gidx], kw["density_factor"])
    _check_fields(sf.get_field_values(m32, x, gidx, **kw), want, b, "cuda non-unit q")
    _check_fields(SF.get_field_values(m32, x, gidx, **kw), want, b, "torch float32 non-unit q")
    _check_field_grads(_field_grads(t, knn, 20_000, seed=11, kw=kw), "non-unit q K=%d %s" % (K, flags))


def _normal_grads(t, knn, N, K, seed):
    """dL/dx, dL/dpoints, dL/dquaternions of sum(g_l loss) + sum(g_e est): CUDA, torch float32 and float64, all with the pinned
    sign decisions."""
    sf = _sf()
    x, gidx, o = _normal_samples(*t, N, K, seed=seed)
    P = t[0].shape[0]
    sign = SN.pinned_signs(SN.Getters(t[0], t[1], t[2], torch.ones(P, 1, device=DEV), knn), gidx)
    gen = torch.Generator().manual_seed(seed + 1)
    gl, ge = torch.randn(N, generator=gen).to(DEV), torch.randn(N, generator=gen).to(DEV)
    out = {}
    for name, dtype in (("cuda", torch.float32), ("torch32", torch.float32), ("f64", torch.float64)):
        leaves = [v.detach().to(dtype).clone().requires_grad_(True) for v in (x, t[0], t[2])]
        m = SN.Getters(leaves[1], t[1].to(dtype), leaves[2], torch.ones(P, 1, device=DEV, dtype=dtype), knn)
        if name == "cuda":
            loss, est = sf.better_normal_loss(m, leaves[0], gidx, o), sf.projection_estimate(m, leaves[0], gidx)
        else:
            loss = SN.better_normal_loss(m, leaves[0], gidx, o.to(dtype), sign=sign)
            est = SN.projection_estimate(m, leaves[0], gidx)
        ((gl.to(dtype) * loss).sum() + (ge.to(dtype) * est).sum()).backward()
        out[name] = [v.grad for v in leaves]
    return out, (x, gidx, o, gl, ge)


@pytest.mark.parametrize("unit", [True, False], ids=["unit_q", "non_unit_q"])
@pytest.mark.parametrize("K", GRAD_K)
def test_normal_gradients_per_gaussian_at_every_width(K, unit):
    t, knn = _nscene(3000, K, seed=9 + K, unit=unit)
    out, _ = _normal_grads(t, knn, 20_000, K, seed=K)
    for i, n in enumerate(NORMAL_NAMES):
        _grad_rule("K=%d %s %s" % (K, "unit" if unit else "non-unit", n), out["cuda"][i], out["torch32"][i], out["f64"][i])


@pytest.mark.parametrize("K", [3, 8, 17])
def test_normal_forward_non_unit_quaternions(K):
    sf = _sf()
    t, knn = _nscene(4000, K, seed=50 + K, unit=False)
    m32 = SN.Getters(t[0], t[1], t[2], torch.ones(4000, 1, device=DEV), knn)
    m64 = SN.Getters(*(v.double() for v in t), torch.ones(4000, 1, device=DEV, dtype=torch.float64), knn)
    x, gidx, o = _normal_samples(*t, 10_007, K, seed=K)
    sign = SN.pinned_signs(m32, gidx)
    b_loss, b_est = _normal_bound(m64, x, gidx, o, sign)
    _check(sf.better_normal_loss(m32, x, gidx, o), SN.better_normal_loss(m64, x.double(), gidx, o.double(), sign=sign), b_loss,
           "non-unit loss")
    _check(sf.projection_estimate(m32, x, gidx), SN.projection_estimate(m64, x.double(), gidx), b_est, "non-unit estimate")


# ------------------------------------------------------------------------------------------------ 4. C-ABI combinations
@pytest.mark.parametrize("K", [1, 3, 8, 13, 32])
def test_field_abi_output_subsets_and_null_dx(K):
    """Forward: any subset of the outputs (out_density NULL included) is bitwise the full call's.  Backward: dL_dx NULL leaves
    the other gradients bitwise unchanged, and rows[row_idx[n]] given as row_idx == NULL gives the same values bitwise."""
    t, x, rows, row_idx = _unique_scene(3001, K, seed=K)
    df = 0.9 / K
    full = _field_fwd(t, x, rows, row_idx, df, ("density", "opac", "beta", "sdf"))
    m = SF.Getters(t[0], t[1], t[2], t[3][:, None], rows)
    wrapped = _sf().get_field_values(m, x, row_idx, return_sdf=True, return_beta=True, return_closest_gaussian_opacities=True,
                                     density_factor=df)
    for k, w in (("density", "density"), ("opac", "closest_gaussian_opacities"), ("beta", "beta"), ("sdf", "sdf")):
        assert torch.isfinite(full[k]).all() and torch.equal(full[k], wrapped[w]), k
    for sub in (("opac",), ("beta",), ("sdf",), ("opac", "beta"), ("beta", "sdf"), ("opac", "sdf"), ("opac", "beta", "sdf"),
                ("density",), ("density", "sdf")):
        got = _field_fwd(t, x, rows, row_idx, df, sub)
        for k in sub:
            assert torch.equal(got[k], full[k]), (sub, k)
    direct = _field_fwd(t, x, rows[row_idx].contiguous(), None, df, ("density", "opac", "beta", "sdf"))
    for k in full:
        assert torch.equal(direct[k], full[k]), k
    gen = torch.Generator().manual_seed(K)
    g = {k: torch.randn(v.shape, generator=gen).to(DEV) for k, v in full.items()}
    for sub in (("density",), ("opac",), ("beta",), ("sdf",), ("beta", "sdf"), ("density", "opac", "beta", "sdf")):
        gs = {k: g[k] for k in sub}
        a = _field_bwd(t, x, rows, row_idx, df, gs)
        b = _field_bwd(t, x, rows, row_idx, df, gs, want_dx=False)
        c = _field_bwd(t, x, rows[row_idx].contiguous(), None, df, gs)
        assert b[0] is None and torch.isfinite(a[0]).all()
        for i in range(1, 5):
            assert torch.isfinite(a[i]).all() and torch.equal(a[i], b[i]) and torch.equal(a[i], c[i]), (sub, FIELD_NAMES[i])
        assert torch.equal(a[0], c[0]), sub


@pytest.mark.parametrize("K", [1, 3, 8, 16, 31])
def test_normal_abi_both_outputs_and_both_gradients(K):
    """Forward with both outputs is bitwise the two separate calls.  Backward with dL_dloss and dL_destimate together against
    float64 by the gradient rule: the estimate's dn_i is added to the loss's before one RED.ADD."""
    t, knn = _nscene(3000, K, seed=60 + K)
    out, (x, gidx, o, gl, ge) = _normal_grads(t, knn, 20_000, K, seed=60 + K)
    loss, est = _normal_fwd(t, x, gidx, knn, o, True, True)
    assert torch.equal(loss, _normal_fwd(t, x, gidx, knn, o, True, False)[0])
    assert torch.equal(est, _normal_fwd(t, x, gidx, knn, o, False, True)[1])
    both = _normal_bwd(t, x, gidx, knn, o, gl, ge)
    for i, n in enumerate(NORMAL_NAMES):
        _grad_rule("both K=%d %s" % (K, n), both[i], out["torch32"][i], out["f64"][i])
    # the estimate alone with knn_idx given runs at W = 1 and equals the wrapper's (K = 1) call bitwise where no atomics race
    est_only = _normal_bwd(t, x, gidx, knn, o, None, ge)
    est_k1 = _normal_bwd(t, x, gidx, None, None, None, ge)
    assert torch.equal(est_only[0], est_k1[0])


# ------------------------------------------------------------------------------------------------ 5. contention
@pytest.mark.parametrize("flags", ["density", "beta_sdf"])
def test_field_repeated_indices_and_one_gaussian_in_100k_pairs(flags):
    """compute_density-style explicit rows (the row_idx == NULL path): repeats within rows, and Gaussian 0 in four of the five
    pairs of each of 25k samples.  Gradients by the rule."""
    K, N = 5, 25_000
    t, knn = _fscene(3000, K, seed=70)
    t = [v.clone() for v in t]
    t[1][0] = 0.5  # large enough that every sample sees it
    x, gidx = _field_samples(t[0], t[1], t[2], N, seed=70, edge_cases=True)
    rows = knn[gidx].clone()
    rows[:, 1:] = 0
    rows[:N // 2, 1] = rows[:N // 2, 0]  # repeats of the sample's own nearest Gaussian
    rows[:, 0] = torch.where(torch.arange(N, device=DEV) % 3 == 0, rows[:, 0], 0)
    assert int((rows == 0).sum()) >= 100_000
    kw = _field_grad_kw(GRAD_FLAGS[flags], K)
    out = _field_grads(t, knn, N, seed=70, kw=kw, rows=rows.contiguous())
    _check_field_grads(out, "contention %s" % flags)


def test_normal_one_gaussian_in_100k_pairs():
    K, N = 8, 20_000
    t, knn = _nscene(3000, K, seed=80)
    knn = knn.clone()
    knn[:, 2:7] = 5  # Gaussian 5 five times in every row, and every sample's row is a row of knn
    out, _ = _normal_grads(t, knn.contiguous(), N, K, seed=80)
    for i, n in enumerate(NORMAL_NAMES):
        _grad_rule("contention %s" % n, out["cuda"][i], out["torch32"][i], out["f64"][i])


# ------------------------------------------------------------------------------------------------ 6. out-of-range indices
@pytest.mark.parametrize("K", [1, 3, 16, 32])
def test_field_out_of_range_indices(K):
    """Rows of -1, R, P and 1 << 40 through row_idx and Gaussian indices of -1, -5, P, P + 3 and 1 << 40 in the rows.  Forward: NaN in
    exactly the density, beta and sdf of the bad samples and the opacities of the bad pairs; every other value bitwise the run
    without the bad samples.  Backward, for every combination of output gradients: dL/dx NaN exactly on the bad samples, every
    per-Gaussian gradient finite and bitwise the run without them (each Gaussian is in at most one pair).  The torch
    restatement never sees a bad index."""
    N = 1000
    t, x, rows, row_idx = _unique_scene(N, K, seed=90 + K)
    P, R = t[0].shape[0], rows.shape[0]
    row_idx, rows = row_idx.clone(), rows.clone()
    bad_row = torch.zeros(N, dtype=torch.bool, device=DEV)
    for n, v in ((0, -1), (5, R), (9, P), (17, 1 << 40)):
        row_idx[n] = v
        bad_row[n] = True
    bad_pair = torch.zeros(N, K, dtype=torch.bool, device=DEV)
    for n, k, v in ((40, 0, -1), (41, K - 1, P), (42, K // 2, P + 3), (43, 0, 1 << 40), (N - 1, K - 1, -5)):
        rows[row_idx[n], k] = v
        bad_pair[n, k] = True
    bad = bad_row | bad_pair.any(1)
    bad_pair |= bad_row[:, None]
    good = (~bad).nonzero()[:, 0]
    df = 0.9 / K
    outs = ("density", "opac", "beta", "sdf")
    f = _field_fwd(t, x, rows, row_idx, df, outs)
    ref = _field_fwd(t, x[good].contiguous(), rows, row_idx[good].contiguous(), df, outs)
    for k in ("density", "beta", "sdf"):
        assert torch.equal(torch.isnan(f[k]), bad), k
        assert torch.equal(f[k][good], ref[k]), k
    assert torch.equal(torch.isnan(f["opac"]), bad_pair)
    assert torch.equal(f["opac"][good], ref["opac"])
    assert torch.isfinite(f["opac"][bad & ~bad_row][~bad_pair[bad & ~bad_row]]).all()  # valid pairs of a bad sample
    gen = torch.Generator().manual_seed(K)
    g = {k: torch.randn(v.shape, generator=gen).to(DEV) for k, v in f.items()}
    combos = [tuple(k for j, k in enumerate(outs) if m >> j & 1) for m in range(1, 16)]
    for sub in combos:
        a = _field_bwd(t, x, rows, row_idx, df, {k: g[k] for k in sub})
        b = _field_bwd(t, x[good].contiguous(), rows, row_idx[good].contiguous(), df, {k: g[k][good].contiguous() for k in sub})
        assert torch.equal(torch.isnan(a[0]).any(1), bad) and torch.isnan(a[0][bad]).all(), sub
        assert torch.equal(a[0][good], b[0]), sub
        for i in range(1, 5):
            assert torch.isfinite(a[i]).all(), (sub, FIELD_NAMES[i])
            assert torch.equal(a[i], b[i]), (sub, FIELD_NAMES[i])
    # the same through autograd with the bad samples' outputs masked out of the loss (their upstream gradients are 0)
    sf = _sf()
    leaves = [v.clone().requires_grad_(True) for v in (x, t[0], t[1], t[2], t[3][:, None])]
    m = SF.Getters(*leaves[1:], rows)
    out = sf.get_field_values(m, leaves[0], row_idx, return_sdf=True, return_beta=True, density_factor=df)
    (out["sdf"].nan_to_num() + out["beta"].nan_to_num()).sum().backward()
    for i in range(1, 5):
        assert torch.isfinite(leaves[i].grad).all(), FIELD_NAMES[i]
    assert torch.equal(torch.isnan(leaves[0].grad).any(1), bad)
