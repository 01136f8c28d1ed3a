"""CPU checks of render_raw(), the differentiable render() from a GaussianModel's raw parameters: the closed-form backward of
the activations and shading normals (activate_backward below, the formula gsr_activate_gaussians_backward implements) against
fp64 autograd, the input checks, and the new C export.  Its numbers on the GPU are checked in tests/test_gpu_raw_render.py."""
import os
import re
import types

import numpy as np
import pytest
import torch

from tests import wrapper_ref as WR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def raw_rows(P, M, seed, ties=True, tiny=4):
    """Raw parameters with quaternion norms spread over 0.1..10, `tiny` rows below F.normalize's 1e-12 clamp, rows with two or
    three equal log-scales, and positions on both sides of the camera's view direction (both flip signs)."""
    g = np.random.default_rng(seed)
    q = g.normal(size=(P, 4))
    q *= (10.0 ** g.uniform(-1, 1, size=P) / np.linalg.norm(q, axis=1))[:, None]
    q[:tiny] *= 1e-14
    sc = g.normal(-3.0, 0.7, size=(P, 3))
    if ties:
        sc[tiny:tiny + 8, 1] = sc[tiny:tiny + 8, 0]  # two equal smallest scales
        sc[tiny:tiny + 8, 2] = sc[tiny:tiny + 8, 0] + 1.0
        sc[tiny + 8:tiny + 16] = sc[tiny + 8:tiny + 16, :1]  # isotropic rows
    return {"xyz": g.normal(size=(P, 3)), "f_dc": g.normal(size=(P, 1, 3)), "f_rest": g.normal(size=(P, M - 1, 3)),
            "opacity": g.normal(size=(P, 1)), "scaling": sc, "rotation": q}


def activate_backward(xyz: np.ndarray, campos: np.ndarray, scaling_raw: np.ndarray, rotation_raw: np.ndarray, opacity_raw: np.ndarray,
                      g_s: np.ndarray, g_r: np.ndarray, g_o: np.ndarray, g_sh=None, g_e=None, k=None, sgn=None) -> dict:
    """Closed-form VJP of the activations (scene/gaussian_model.py:95-115) followed by get_normal(...) * 0.5 + 0.5 (:120-128),
    in the dtype of the inputs.  g_s, g_r, g_o, g_sh [P,M,3] and g_e [P,3] are the gradients of the activated scales, rotations, opacities, SH rows
    and remapped normals (g_sh / g_e may be None).  The axis k (smallest activated scale, first on ties) and the flip sign sgn are
    the forward's piecewise-constant decisions; either may be forced.  Returns d_scaling, d_rotation, d_opacity and, with g_sh,
    d_f_dc / d_f_rest."""
    dt = np.result_type(scaling_raw, rotation_raw, np.float32)
    s = np.exp(scaling_raw.astype(dt))
    rho = rotation_raw.astype(dt)
    rho_n = np.sqrt((rho * rho).sum(-1))
    r = rho / np.maximum(rho_n, dt.type(1e-12))[:, None]
    o = 1 / (1 + np.exp(-opacity_raw.astype(dt)))
    out = {"d_scaling": g_s * s, "d_opacity": g_o * o * (1 - o)}
    rb = g_r.astype(dt).copy()
    if g_e is not None:
        P = r.shape[0]
        if k is None:
            k = np.argmin(s, axis=-1)
        qn = np.sqrt((r * r).sum(-1))
        q = r / qn[:, None]
        w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        # build_rotation's matrix and its derivative d R[i, j] / d q_c, for the columns of the smallest axis
        Rm = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                       np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                       np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
        zero = np.zeros_like(w)
        dR = np.stack([  # [P, 4 (w,x,y,z), 3, 3]
            np.stack([np.stack([zero, -2 * z, 2 * y], -1), np.stack([2 * z, zero, -2 * x], -1), np.stack([-2 * y, 2 * x, zero], -1)], 1),
            np.stack([np.stack([zero, 2 * y, 2 * z], -1), np.stack([2 * y, -4 * x, -2 * w], -1), np.stack([2 * z, 2 * w, -4 * x], -1)], 1),
            np.stack([np.stack([-4 * y, 2 * x, 2 * w], -1), np.stack([2 * x, zero, 2 * z], -1), np.stack([-2 * w, 2 * z, -4 * y], -1)], 1),
            np.stack([np.stack([-4 * z, -2 * w, 2 * x], -1), np.stack([2 * w, -4 * z, 2 * y], -1), np.stack([2 * x, 2 * y, zero], -1)], 1)], 1)
        idx = np.arange(P)
        a = Rm[idx, :, k]
        if sgn is None:
            d = xyz.astype(dt) - campos.astype(dt)[None, :]
            d = d / np.sqrt((d * d).sum(-1))[:, None]
            sgn = np.where((a * -d).sum(-1) >= 0, 1, -1)
        sgn = np.asarray(sgn, dtype=dt)
        an = np.sqrt((a * a).sum(-1))
        n = sgn[:, None] * a / an[:, None]
        nb = 0.5 * g_e.astype(dt)
        ab = sgn[:, None] * (nb - n * (n * nb).sum(-1, keepdims=True)) / an[:, None]
        qb = np.einsum("pci,pi->pc", dR[idx, :, :, k], ab)
        rb = rb + (qb - q * (q * qb).sum(-1, keepdims=True)) / qn[:, None]
    clamped = rho_n < dt.type(1e-12)
    proj = (rb - r * (r * rb).sum(-1, keepdims=True)) / np.where(clamped, 1, rho_n)[:, None]
    out["d_rotation"] = np.where(clamped[:, None], rb / dt.type(1e-12), proj)
    if g_sh is not None:
        out["d_f_dc"], out["d_f_rest"] = g_sh[:, :1].copy(), g_sh[:, 1:].copy()
    return out


def fp64_autograd(raw, campos, grads, k, sgn):
    """exp / F.normalize / sigmoid / cat and get_normal(...) * 0.5 + 0.5 in torch fp64 with the axis k and flip sgn forced."""
    t = {n: torch.tensor(v, dtype=torch.float64, requires_grad=n != "xyz") for n, v in raw.items()}
    s, r, o = torch.exp(t["scaling"]), torch.nn.functional.normalize(t["rotation"]), torch.sigmoid(t["opacity"])
    shs = torch.cat((t["f_dc"], t["f_rest"]), dim=1)
    a = WR.build_rotation(r)[torch.arange(r.shape[0]), :, torch.as_tensor(k)]
    n = a * torch.as_tensor(sgn, dtype=torch.float64)[:, None]
    e = n / n.norm(dim=1, keepdim=True) * 0.5 + 0.5
    loss = sum((x * torch.as_tensor(grads[n_])).sum() for x, n_ in ((s, "g_s"), (r, "g_r"), (o, "g_o"), (shs, "g_sh"), (e, "g_e"))
               if grads.get(n_) is not None)
    loss.backward()
    return {"d_scaling": t["scaling"].grad, "d_rotation": t["rotation"].grad, "d_opacity": t["opacity"].grad,
            "d_f_dc": t["f_dc"].grad, "d_f_rest": t["f_rest"].grad}


@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("with_normals", [True, False], ids=["normals", "no_normals"])
def test_activate_backward_against_fp64_autograd(M, with_normals):
    P = 400
    raw = raw_rows(P, M, seed=M)
    campos = np.array([0.1, -0.2, 0.3])
    g = np.random.default_rng(99)
    grads = {"g_s": g.normal(size=(P, 3)), "g_r": g.normal(size=(P, 4)), "g_o": g.normal(size=(P, 1)), "g_sh": g.normal(size=(P, M, 3)),
             "g_e": g.normal(size=(P, 3)) if with_normals else None}
    got = activate_backward(raw["xyz"], campos, raw["scaling"], raw["rotation"], raw["opacity"], **grads)
    s = torch.exp(torch.tensor(raw["scaling"]))
    k = torch.argsort(s, dim=-1, stable=True)[:, 0].numpy()
    # activate_backward's decisions: first minimum on ties, and both flip signs occur
    assert np.array_equal(k, np.argmin(np.exp(raw["scaling"]), axis=-1))
    assert (k[4:20] == 0).all()
    r = raw["rotation"] / np.maximum(np.linalg.norm(raw["rotation"], axis=1), 1e-12)[:, None]
    a = WR.build_rotation(torch.tensor(r))[torch.arange(P), :, torch.tensor(k)].numpy()
    d = raw["xyz"] - campos
    sgn = np.where((a * -(d / np.linalg.norm(d, axis=1)[:, None])).sum(-1) >= 0, 1.0, -1.0)
    assert (sgn > 0).sum() > 50 and (sgn < 0).sum() > 50
    want = fp64_autograd(raw, campos, grads, k, sgn)
    assert set(got) == set(want)
    for name, w in want.items():
        w = w.numpy()
        err = np.linalg.norm((got[name] - w).reshape(P, -1), axis=1)
        ref = np.linalg.norm(w.reshape(P, -1), axis=1)
        assert (err <= 1e-12 * ref + 1e-300).all(), (name, float((err / np.maximum(ref, 1e-300)).max()))
    assert np.abs(got["d_rotation"][:4]).max() > 1e6  # the clamped rows: r = rho / 1e-12
    if not with_normals:
        # without the normal image the rotation gradient is F.normalize's Jacobian of g_r alone
        rn = np.linalg.norm(raw["rotation"], axis=1)[4:]
        gr, rr = grads["g_r"][4:], r[4:]
        assert np.allclose(got["d_rotation"][4:], (gr - rr * (rr * gr).sum(-1, keepdims=True)) / rn[:, None], rtol=1e-12, atol=0)


# ---- render_raw's input checks --------------------------------------------------------------------------------------------------
class _RawModel:
    """The raw fields and activation attributes of the reference's GaussianModel (scene/gaussian_model.py:32-61)."""

    def __init__(self, P=4, M=16, device="cpu"):
        f = dict(dtype=torch.float32, device=device)
        self._xyz, self._features_dc, self._features_rest = torch.zeros(P, 3, **f), torch.zeros(P, 1, 3, **f), torch.zeros(P, M - 1, 3, **f)
        self._opacity, self._scaling, self._rotation = torch.zeros(P, 1, **f), torch.zeros(P, 3, **f), torch.ones(P, 4, **f)
        self.scaling_activation, self.opacity_activation = torch.exp, torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize
        self.active_sh_degree, self.max_sh_degree = 3, 3


def _pipe(**kw):
    return types.SimpleNamespace(**dict(dict(debug=False, compute_cov3D_python=False, convert_SHs_python=False), **kw))


def _cam():
    return types.SimpleNamespace(FoVx=1.0, FoVy=1.0, image_height=8, image_width=8, world_view_transform=torch.eye(4),
                                 full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))


def _call(pc, pipe=None):
    from autovfx_b200.renderer import render_raw
    return render_raw(_cam(), pc, pipe or _pipe(), torch.zeros(3))


@pytest.mark.parametrize("field", ["_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"])
def test_render_raw_rejects_a_model_without_raw_fields(field):
    pc = _RawModel()
    delattr(pc, field)
    with pytest.raises(ValueError, match=field):
        _call(pc)


@pytest.mark.parametrize("attr,fn", [("scaling_activation", torch.nn.functional.softplus), ("opacity_activation", torch.tanh),
                                     ("rotation_activation", lambda x: x), ("scaling_activation", None)])
def test_render_raw_rejects_other_activations(attr, fn):
    pc = _RawModel()
    if fn is None:
        delattr(pc, attr)
    else:
        setattr(pc, attr, fn)
    with pytest.raises(ValueError, match=attr):
        _call(pc)


@pytest.mark.parametrize("flag", ["compute_cov3D_python", "convert_SHs_python"])
def test_render_raw_rejects_python_pipe_paths(flag):
    with pytest.raises(ValueError, match=flag):
        _call(_RawModel(), _pipe(**{flag: True}))


def test_render_raw_rejects_cpu_tensors():
    with pytest.raises(RuntimeError, match="no CPU path"):
        _call(_RawModel())


def test_render_raw_rejects_bad_shapes():
    pc = _RawModel()
    pc._opacity = torch.zeros(4)
    with pytest.raises(ValueError, match="_opacity"):
        _call(pc)


def test_activate_backward_export_is_declared_bound_and_listed():
    from autovfx_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    assert re.search(r"int gsr_activate_gaussians_backward\(", hdr)
    assert "gsr_activate_gaussians_backward" in _lib.EXPORTS
    fn = _lib.lib.gsr_activate_gaussians_backward
    assert len(fn.argtypes) == 19 and _lib.ABI_VERSION == 4
