"""CPU checks of render_sugar_raw()'s colour path: SuGaR's get_points_rgb (eval_sh, degrees 0-4) stated in numpy float32 with one
rounding per torch op (tests/sugar_colors_ref.py, the arithmetic gsr_sugar_colors implements) against torch on the CPU; the closed-form
backward gsr_sugar_colors_backward implements against fp64 autograd; the degree-4 basis pinned by its orthonormality on the sphere;
render_sugar_raw's input validation; and the new C exports.  The GPU side is checked in tests/test_gpu_sugar_colors.py."""
import os
import re
import types

import numpy as np
import pytest
import torch

from tests import sugar_colors_ref as SC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFGS = [(deg, M) for deg in range(5) for M in (1, 4, 9, 16, 25) if M >= (deg + 1) ** 2]
ZERO_DC = np.float32(-1.7724538)  # fl(fl(C0 * ZERO_DC) + 0.5) == 0 exactly: a pre-clamp colour of 0 when the other coefficients are 0


def rows(P, M, seed, unit=True):
    """SH rows [P,M,3], positions, camera centre and directions; rows 0-7 have a negative pre-clamp colour in every channel, rows
    8-11 an exact 0 (dc = ZERO_DC, the rest 0), rows 12-13 sit at the camera centre."""
    g = np.random.default_rng(seed)
    sh = g.normal(0.0, 0.6, size=(P, M, 3)).astype(np.float32)
    sh[0:8, 0] = -6.0
    sh[0:8, 1:] *= 0.01
    sh[8:12, 0], sh[8:12, 1:] = ZERO_DC, 0.0
    campos = np.array([0.25, -0.5, 0.125], dtype=np.float32)
    pos = g.normal(size=(P, 3)).astype(np.float32)
    pos[12:14] = campos
    d = g.normal(size=(P, 3))
    if unit:
        d /= np.linalg.norm(d, axis=1, keepdims=True)
    else:
        d *= g.uniform(0.5, 1.5, size=(P, 1))
    return sh, pos, campos, d.astype(np.float32)


def torch_colors(deg, sh, dirs):
    """SuGaR's get_points_rgb in directions mode on the CPU (SS/:711-755 with tests/sugar_colors_ref.eval_sh)."""
    n = (deg + 1) ** 2
    shs_view = torch.from_numpy(sh)[:, :n].transpose(-1, -2).reshape(-1, 3, n)
    return torch.clamp_min(SC.eval_sh(deg, shs_view, torch.from_numpy(dirs)) + 0.5, 0.0).view(-1, 3).numpy()


@pytest.mark.parametrize("deg,M", CFGS)
@pytest.mark.parametrize("unit", [True, False], ids=["unit", "scaled"])
def test_float32_restatement_is_torch_cpu_bit_for_bit(deg, M, unit):
    sh, pos, campos, d = rows(2048, M, seed=deg * 31 + M, unit=unit)
    got, pre = SC.colors_np(deg, sh, d)
    want = torch_colors(deg, sh, d)
    assert np.array_equal(got, want), np.abs(got - want).max()
    assert (pre[0:8] < 0).all() and (got[0:8] == 0).all() and (pre[8:12] == 0).all()
    # camera-centre mode: torch's F.normalize against the left-to-right norm; the colours agree to rounding
    dirs_t = torch.nn.functional.normalize(torch.from_numpy(pos) - torch.from_numpy(campos).reshape(1, 3), dim=-1).numpy()
    dirs_n = SC.view_dirs_np(pos, campos)
    assert np.abs(dirs_t - dirs_n).max() <= 2.4e-7 and np.array_equal(dirs_n[12:14], np.zeros((2, 3), np.float32))
    assert np.abs(SC.colors_np(deg, sh, dirs_n)[0] - torch_colors(deg, sh, dirs_t)).max() <= 1e-5


def _autograd(deg, sh, g, passed, directions=None, positions=None, campos=None):
    sh64 = torch.from_numpy(sh).double().requires_grad_(True)
    src = torch.from_numpy(directions if directions is not None else positions).double().requires_grad_(True)
    out = SC.colors_forced(deg, sh64, torch.from_numpy(passed).double(), **(
        {"directions": src} if directions is not None else {"positions": src, "campos": torch.from_numpy(campos).double().reshape(1, 3)}))
    out.backward(torch.from_numpy(g))
    return sh64.grad.numpy(), (np.zeros(src.shape) if src.grad is None else src.grad.numpy())  # degree 0 never reads the direction


def _rows_close(got, want, rel=1e-9):
    got, want = got.reshape(got.shape[0], -1), want.reshape(want.shape[0], -1)
    err = np.linalg.norm(got - want, axis=1)
    return bool((err <= rel * np.linalg.norm(want, axis=1) + 1e-300).all())


@pytest.mark.parametrize("deg,M", CFGS)
@pytest.mark.parametrize("mode", ["camera", "directions"])
def test_closed_form_backward_against_fp64_autograd(deg, M, mode):
    P = 512
    sh, pos, campos, d = rows(P, M, seed=100 + deg * 7 + M, unit=False)
    dirs = d if mode == "directions" else SC.view_dirs_np(pos, campos)
    _, pre = SC.colors_np(deg, sh, dirs)
    passed = (pre >= 0).astype(np.float64)  # torch's clamp_min passes the gradient at equality
    assert passed[8:12].all() and not passed[0:8].any()
    g = np.random.default_rng(deg + M).normal(size=(P, 3))
    kw = {"directions": d} if mode == "directions" else {"positions": pos, "campos": campos}
    want_sh, want_src = _autograd(deg, sh, g, passed, **kw)
    got_sh, got_src = SC.colors_vjp(deg, sh[:, :(deg + 1) ** 2], g, passed, **kw)
    n = (deg + 1) ** 2
    assert np.abs(want_sh[:, n:]).max(initial=0.0) == 0.0  # the slice's backward: zeros beyond the active degree
    assert _rows_close(got_sh, want_sh[:, :n]) and _rows_close(got_src, want_src)
    if mode == "camera" and deg > 0:
        # at the camera centre F.normalize divides by the constant 1e-12: the gradient is dL/ddir / 1e-12, with no norm term
        gd = SC.colors_vjp(deg, sh[12:14, :n], g[12:14], passed[12:14], directions=np.zeros((2, 3)))[1]
        assert np.allclose(want_src[12:14], gd / 1e-12, rtol=1e-12, atol=0) and np.abs(want_src[12:14]).max() > 1e9


def test_degree_4_basis_is_orthonormal_on_the_sphere():
    """The 25 restated polynomials times their constants are the real orthonormal spherical harmonics: their Gram matrix under a
    40 x 80 Gauss-Legendre x uniform-azimuth quadrature (exact for these degree-8 products) is the identity, to 2.4e-14 in float64
    with this evaluation order (a constant off in its 9th digit would show as 1e-9)."""
    mu, w = np.polynomial.legendre.leggauss(40)
    phi = 2 * np.pi * np.arange(80) / 80
    s = np.sqrt(1 - mu ** 2)
    x, y, z = (s[:, None] * np.cos(phi)[None]).ravel(), (s[:, None] * np.sin(phi)[None]).ravel(), np.repeat(mu, 80)
    wt = np.repeat(w, 80) * (2 * np.pi / 80)
    B = np.stack([SC.SIGN[k] * b for k, b in enumerate(SC.basis(4, x, y, z, np.float64))], 0)
    gram = (B * wt) @ B.T
    assert np.abs(gram - np.eye(25)).max() <= 5e-14


# ---- input validation --------------------------------------------------------------------------------------------------------------
def _model(P=6, M=16, device="cpu", **over):
    m = types.SimpleNamespace(device=device, _sh_coordinates_dc=torch.zeros(P, 1, 3), _sh_coordinates_rest=torch.zeros(P, M - 1, 3),
                              all_densities=torch.zeros(P, 1))
    for k, v in over.items():
        setattr(m, k, v)
    return m


@pytest.mark.parametrize("over,kw,field", [
    (dict(_sh_coordinates_dc=None), {}, "_sh_coordinates_dc"),
    (dict(all_densities=torch.zeros(6, 1, dtype=torch.float64)), {}, "all_densities"),
    (dict(_sh_coordinates_rest=torch.zeros(6, 15, 3, dtype=torch.float16)), {}, "_sh_coordinates_rest"),
    (dict(device="cuda:0"), {}, "_sh_coordinates_dc"),  # leaves on the CPU, model on a GPU
    (dict(_sh_coordinates_dc=torch.zeros(6, 3)), {}, "_sh_coordinates_dc"),
    (dict(_sh_coordinates_dc=torch.zeros(6, 2, 3)), {}, "_sh_coordinates_dc"),
    (dict(_sh_coordinates_rest=torch.zeros(6, 15, 4)), {}, "_sh_coordinates_rest"),
    (dict(_sh_coordinates_rest=torch.zeros(5, 15, 3)), {}, "_sh_coordinates_rest"),
    (dict(all_densities=torch.zeros(7)), {}, "all_densities"),
    (dict(return_one_densities=True), {}, "return_one_densities"),
    ({}, dict(sh_deg=4), "sh_deg"),   # 25 coefficients, M = 16
    ({}, dict(sh_deg=5), "sh_deg"),
    ({}, dict(sh_deg=-1), "sh_deg"),
    ({}, dict(sh_deg=None), "sh_deg"),
])
def test_render_sugar_raw_rejects_bad_inputs(over, kw, field):
    from autovfx_b200.renderer import render_sugar_raw
    kw = dict(dict(sh_deg=3), **kw)
    with pytest.raises(ValueError, match=field):
        render_sugar_raw(_model(**over), **kw)


def test_render_sugar_raw_checks_sh_deg_only_where_colours_are_evaluated():
    from autovfx_b200.renderer import render_sugar_raw
    # the point_colors and compute_color_in_rasterizer branches never call eval_sh; on the CPU they stop at the missing CUDA path
    for kw in (dict(point_colors=torch.zeros(6, 3)), dict(compute_color_in_rasterizer=True)):
        with pytest.raises(RuntimeError, match="no CPU path"):
            render_sugar_raw(_model(), sh_deg=9, **kw)
    with pytest.raises(RuntimeError, match="no CPU path"):
        render_sugar_raw(_model(M=25), sh_deg=4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        render_sugar_raw(_model(M=1), sh_deg=0)


def test_sugar_color_exports():
    from autovfx_b200 import _lib, renderer
    assert {"gsr_sugar_colors", "gsr_sugar_colors_backward"} <= set(_lib.EXPORTS) and _lib.ABI_VERSION == 4
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsr_b200.h")).read(), flags=re.S)
    assert re.search(r"int gsr_sugar_colors\(", hdr) and re.search(r"int gsr_sugar_colors_backward\(", hdr)
    L = _lib.lib
    assert L.gsr_abi_version() == 4
    assert len(L.gsr_sugar_colors.argtypes) == 12 and len(L.gsr_sugar_colors_backward.argtypes) == 16
    assert "render_sugar_raw" in renderer.__all__
    n = [None] * 8
    assert L.gsr_sugar_colors(0, 16, 3, *n, None) == 0  # P = 0 is a no-op
    assert L.gsr_sugar_colors_backward(0, 25, 4, *n, *n[:5]) == 0
    assert L.gsr_sugar_colors(4, 16, 3, *n[:6], None, None, None) == 0  # nothing requested
    # the reference's asserts: deg in 0..4, M >= (deg+1)^2
    for P, M, deg in ((4, 16, 5), (4, 16, -1), (4, 8, 3), (4, 24, 4), (-1, 16, 3)):
        assert L.gsr_sugar_colors(P, M, deg, *n[:6], 16, 16, None) != 0
        assert "gsr_sugar_colors" in L.gsr_last_error().decode()
        assert L.gsr_sugar_colors_backward(P, M, deg, *n[:6], 16, 16, None, 16, 16, 16, None) != 0
    # partly-NULL argument lists are rejected before any launch
    assert L.gsr_sugar_colors(4, 16, 3, 16, None, None, 16, 16, 16, 16, None, None) != 0  # no campos, no directions
    assert L.gsr_sugar_colors(4, 16, 3, None, None, 16, 16, None, 16, 16, None, None) != 0  # no sh_rest at M = 16
    assert L.gsr_sugar_colors(4, 16, 3, None, None, 16, 16, 16, None, None, 16, None) != 0  # opacities without densities
    assert L.gsr_sugar_colors_backward(4, 16, 3, None, None, 16, 16, 16, 16, 16, None, 16, 16, None, None, None) != 0  # no dL_dpositions
    assert L.gsr_sugar_colors_backward(4, 16, 3, None, None, 16, 16, 16, 16, None, 16, None, None, None, None, None) != 0  # no dL_ddensities
