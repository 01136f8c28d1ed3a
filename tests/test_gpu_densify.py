"""Densification on the GPU (autovfx_b200.densify): the statistics and densify_and_prune drop-ins against the reference's own
GaussianModel (oracle/ref_py: live where it is staged, replayed from tests/golden/ref/ elsewhere) and against the torch
restatements of tests/densify_ref.py (always).  Run with -m gpu on an H100.

Every parameter and both Adam moments must be bit-identical, except the xyz of split children: torch computes R(q) @ samples with
cuBLAS bmm, whose summation order is its own.  Two 3-term dot products of the same float operands differ by at most
2 * gamma_3 * sum_k |R_ck| |s_k| (gamma_3 = 3u / (1 - 3u), u = 2^-24, |R_ck| <= 1 + 1e-6), and the final "+ xyz" adds one rounding
to each side: u * (|ours| + |ref|).  SuGaR's rotation (quaternion_to_matrix of F.normalize(q)) sums |q|^2 in torch's reduction order;
the kernel's pairwise order may move each element of R by a few ulps, so its bound adds 8u * sum_k |s_k|.
"""
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

from tests import densify_ref as DR  # noqa: E402
from tests import helpers as Hh  # noqa: E402
from tests.test_densify_cpu import CASES, make_case  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
GAMMA3 = 3 * U / (1 - 3 * U)
SEED = 1234
GS_GROUPS = (("xyz", "_xyz"), ("f_dc", "_features_dc"), ("f_rest", "_features_rest"), ("opacity", "_opacity"),
             ("scaling", "_scaling"), ("rotation", "_rotation"))
LRS = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 0.05, "scaling": 5e-3, "rotation": 1e-3}
PIPE = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)


@pytest.fixture(scope="module", autouse=True)
def _lib():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import densify  # noqa: F401  (fails loudly if the CUDA library is missing)


def _adam_state(params, state, seed):
    """An Adam optimizer over named groups (as training_setup builds it) after two real steps.  state: 'all', 'some' (three groups
    stepped, the others without state) or 'none'."""
    opt = torch.optim.Adam([{"params": [p], "lr": LRS[n], "name": n} for n, p in params], lr=0.0, eps=1e-15)
    if state != "none":
        g = torch.Generator().manual_seed(seed)
        for _ in range(2):
            for n, p in params:
                gr = torch.randn(p.shape, generator=g)
                p.grad = gr.to(p.device) if state == "all" or n in ("xyz", "f_rest", "scaling") else None
            opt.step()
        for _, p in params:
            p.grad = None
    return opt


def _gs_model(obj, raw, accum, denom, state, seed):
    for n, a in GS_GROUPS:
        setattr(obj, a, nn.Parameter(raw[n].detach().clone().to(DEV).contiguous().requires_grad_(True)))
    obj.optimizer = _adam_state([(n, getattr(obj, a)) for n, a in GS_GROUPS], state, seed)
    obj.xyz_gradient_accum, obj.denom = accum.clone().to(DEV), denom.clone().to(DEV)
    obj.max_radii2D = torch.zeros(accum.shape[0], device=DEV)
    obj.percent_dense = 0.01
    return obj


def _snapshot(opt):
    """{group name: (param, exp_avg, exp_avg_sq or None, step object)} copies before densification."""
    out = {}
    for g in opt.param_groups:
        p = g["params"][0]
        st = opt.state.get(p)
        out[g["name"]] = (p.detach().clone(), *((st["exp_avg"].clone(), st["exp_avg_sq"].clone(), st["step"]) if st else (None,) * 3))
    return out


def _split_rows(accum, denom, scaling, max_grad, extent, pd):
    g = (accum / denom).reshape(-1)
    g = torch.where(g.isnan(), torch.zeros_like(g), g)
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    return (g >= f32(max_grad)) & (torch.exp(scaling).max(dim=1).values > f32(pd * extent))


def _child_bound(tags, P, split, scaling, extra):
    """Per-element bound on |ours - torch| for the xyz of the final rows that are split children (module docstring)."""
    torch.cuda.manual_seed(SEED)
    S = int(split.sum())
    eps = torch.randn((2 * S, 3), device=DEV)
    j = torch.cumsum(split.long(), 0) - 1
    kind, src = tags // P, tags % P
    ch = kind >= 2
    row = (kind[ch] - 2) * S + j[src[ch]]
    smp = (eps[row] * torch.exp(scaling[src[ch]])).abs().sum(-1, keepdim=True)
    return ch, (2 * GAMMA3 * (1 + 1e-6) + extra) * smp


def _check_against_restatement(new, new_m, tags, opt_groups, snap, P, bound_fn, names_xyz):
    """ours (params from opt_groups, moments from the optimizer) == the restatement, children's xyz within the bound."""
    ch, bound = bound_fn(tags)
    for name, (p, st) in opt_groups.items():
        want = new[name]
        assert p.shape == want.shape, name
        if name == names_xyz:
            assert torch.equal(p[~ch], want[~ch]), name
            d = (p[ch] - want[ch]).abs()
            assert bool((d <= bound + U * (p[ch].abs() + want[ch].abs())).all()), (name, float(d.max()) if d.numel() else 0.0)
        else:
            assert torch.equal(p, want), name
        if snap[name][1] is None:
            assert st is None, name
        else:
            assert st is not None and st["step"] is snap[name][3], name
            assert torch.equal(st["exp_avg"], new_m[name][0]) and torch.equal(st["exp_avg_sq"], new_m[name][1]), name


def _gs_case(name, M, P, state, seed):
    from autovfx_b200 import densify
    raw, accum, denom, max_grad, min_opacity, mss = make_case(name, P, M, seed)
    extent, pd = 1.0, 0.01
    ours = _gs_model(types.SimpleNamespace(), raw, accum, denom, state, seed)
    snap = _snapshot(ours.optimizer)
    torch.cuda.manual_seed(SEED)
    with torch.no_grad():
        densify.densify_and_prune(ours, max_grad, min_opacity, extent, mss)
    rng = torch.cuda.get_rng_state()
    # the param groups hold the model's attributes, the state is keyed by them
    groups = {}
    for g in ours.optimizer.param_groups:
        p = g["params"][0]
        assert p is getattr(ours, dict(GS_GROUPS)[g["name"]]) and isinstance(p, nn.Parameter) and p.requires_grad
        groups[g["name"]] = (p.detach(), ours.optimizer.state.get(p))
    P2 = ours._xyz.shape[0]
    for t, shape in ((ours.xyz_gradient_accum, (P2, 1)), (ours.denom, (P2, 1)), (ours.max_radii2D, (P2,))):
        assert t.shape == shape and not t.any()
    # the restatement on the same inputs, from the same generator state
    moments = {n: (s[1], s[2]) for n, s in snap.items() if s[1] is not None}
    torch.cuda.manual_seed(SEED)
    with torch.no_grad():
        new, new_m, tags = DR.sequential({n: s[0] for n, s in snap.items()}, moments, accum.to(DEV), denom.to(DEV), max_grad,
                                         min_opacity, extent, mss, pd, DR.build_rotation)
    assert torch.equal(rng, torch.cuda.get_rng_state())
    split = _split_rows(accum.to(DEV), denom.to(DEV), snap["scaling"][0], max_grad, extent, pd)
    _check_against_restatement(new, new_m, tags, groups, snap, P,
                               lambda tg: _child_bound(tg, P, split, snap["scaling"][0], 0.0), "xyz")
    # the reference's own GaussianModel: live where staged, replayed elsewhere
    Hh.use_ref_python()
    if Hh.have_ref():
        def ref_run():
            from oracle import ref_py
            ns = ref_py.load("ref")
            m = _gs_model(ns.gaussian_model.GaussianModel(3), raw, accum, denom, state, seed)
            torch.cuda.manual_seed(SEED)
            with torch.no_grad():
                m.densify_and_prune(max_grad, min_opacity, extent, mss)
            out = {g["name"]: (g["params"][0], m.optimizer.state.get(g["params"][0])) for g in m.optimizer.param_groups}
            out["_rng"] = torch.cuda.get_rng_state()
            return out
        ref = _once(ref_run)
        ch, bound = _child_bound(tags, P, split, snap["scaling"][0], 0.0)
        assert Hh.ref_value(lambda: int(ref()["xyz"][0].shape[0])) == P2
        assert Hh.ref_same(rng, lambda: ref()["_rng"])
        for n, (p, st) in sorted(groups.items()):
            if n == "xyz":
                assert Hh.ref_same(p[~ch], lambda: ref()[n][0][~ch]), n
                if ch.any():
                    d = Hh.ref_maxabs(p[ch], lambda: ref()[n][0][ch])
                    assert d <= float((bound + 2 * U * p[ch].abs()).max()) * 1.01, (n, d)
            else:
                assert Hh.ref_same(p, lambda: ref()[n][0]), n
            if st is not None:
                assert Hh.ref_same(st["exp_avg"], lambda: ref()[n][1]["exp_avg"]), n
                assert Hh.ref_same(st["exp_avg_sq"], lambda: ref()[n][1]["exp_avg_sq"]), n
    return ours


def _once(fn):
    box = []
    return lambda: box[0] if box else (box.append(fn()) or box[0])


@pytest.mark.parametrize("name", sorted(CASES))
def test_densify_and_prune_matches_reference(name):
    _gs_case(name, 16, 3000, "all", seed=len(name))


@pytest.mark.parametrize("M", [1, 16, 25])
@pytest.mark.parametrize("state", ["all", "some", "none"])
def test_densify_and_prune_sh_widths_and_state(M, state):
    _gs_case("default", M, 2500, state, seed=M)


def test_densify_and_prune_3m_gaussians():
    _gs_case("default", 16, 3_000_000, "all", seed=3)


def test_densified_model_trains():
    """One Adam step and one render_raw step (forward + backward) on the densified model."""
    from autovfx_b200 import densify, renderer
    from tests.test_gpu_fused_grads import _cam
    ours = _gs_case("default", 16, 3000, "all", seed=9)
    ours.scaling_activation, ours.opacity_activation = torch.exp, torch.sigmoid
    ours.rotation_activation = torch.nn.functional.normalize
    ours.active_sh_degree, ours.max_sh_degree = 3, 3
    c = Hh.case_inputs("config1")
    cam, bg = _cam(c["cam"], torch.device(DEV)), torch.tensor(c["bg"], device=DEV)
    for _ in range(2):
        out = renderer.render_raw(cam, ours, PIPE, bg)
        out["render"].square().mean().backward()
        with torch.no_grad():
            densify.update_densification_stats(ours, out["viewspace_points"], out["radii"], out["visibility_filter"])
        ours.optimizer.step()
        ours.optimizer.zero_grad(set_to_none=True)
    assert torch.isfinite(ours._xyz).all()


def test_stats_match_reference_lines():
    """Three render_raw backward steps: update_densification_stats (GaussianModel and SuGaR accumulator names) and
    add_densification_stats equal the trainer's max-radii line plus the reference's add_densification_stats bit for bit, and
    issue no host synchronisation."""
    from autovfx_b200 import densify, renderer
    from tests.test_gpu_raw_render import _case, _RawPC
    raw, cam, bg, D, mod, _ = _case("config1", torch.device(DEV))
    pc = _RawPC(raw, D)
    P = raw["_xyz"].shape[0]
    z = lambda *s: torch.zeros(s, device=DEV)  # noqa: E731
    gs = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1), max_radii2D=z(P))
    sugar = types.SimpleNamespace(points_gradient_accum=z(P, 1), denom=z(P, 1), max_radii2D=z(P))
    add = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1))
    want = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1), max_radii2D=z(P))
    live = None
    from oracle import ref_py
    if ref_py.available():
        live = (ref_py.load("ref").gaussian_model.GaussianModel, types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1)))
    g = torch.Generator().manual_seed(4)
    for step in range(3):
        out = renderer.render_raw(cam, pc, PIPE, bg, scaling_modifier=mod)
        w = torch.randn(out["render"].shape, generator=g).to(DEV)
        (out["render"] * w).sum().backward()
        vs, radii, vis = out["viewspace_points"], out["radii"], out["visibility_filter"]
        assert radii.dtype == torch.int32
        with torch.no_grad():
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                densify.update_densification_stats(gs, vs, radii, vis)
                densify.update_densification_stats(sugar, vs, radii, vis)
                densify.add_densification_stats(add, vs, vis)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            want.max_radii2D[vis] = torch.max(want.max_radii2D[vis], radii[vis])
            want.xyz_gradient_accum[vis] += torch.norm(vs.grad[vis, :2], dim=-1, keepdim=True)
            want.denom[vis] += 1
            if live is not None:
                live[0].add_densification_stats(live[1], vs, vis)
        for t in (gs.xyz_gradient_accum, sugar.points_gradient_accum, add.xyz_gradient_accum):
            assert torch.equal(t, want.xyz_gradient_accum), step
        for m in (gs, sugar, add):
            assert torch.equal(m.denom, want.denom)
        assert torch.equal(gs.max_radii2D, want.max_radii2D) and torch.equal(sugar.max_radii2D, want.max_radii2D)
        if live is not None:
            assert torch.equal(live[1].xyz_gradient_accum, want.xyz_gradient_accum) and torch.equal(live[1].denom, want.denom)
        for k in pc.leaves.values():
            k.grad = None
    assert int(want.denom.max()) == 3 and bool((want.xyz_gradient_accum > 0).any())


@pytest.mark.parametrize("name", ["default", "split_only", "screen_none", "all_pruned"])
@pytest.mark.parametrize("M", [1, 16])
def test_sugar_densify_and_prune_matches_restatement(name, M):
    from autovfx_b200 import densify
    raw, accum, denom, max_grad, min_opacity, mss = make_case(name, 3000, M, seed=11 + M)
    names = (("points", "_points", "xyz"), ("all_densities", "all_densities", "opacity"), ("scales", "_scales", "scaling"),
             ("quaternions", "_quaternions", "rotation"), ("sh_coordinates_dc", "_sh_coordinates_dc", "f_dc"),
             ("sh_coordinates_rest", "_sh_coordinates_rest", "f_rest"))
    model = types.SimpleNamespace(binded_to_surface_mesh=False)
    for n, a, r in names:
        setattr(model, a, nn.Parameter(raw[r].clone().to(DEV).requires_grad_(True)))
    LRS.update({n: LRS[r] for n, _, r in names})
    opt = _adam_state([(n, getattr(model, a)) for n, a, _ in names], "all", 3)
    dens = types.SimpleNamespace(model=model, optimizer=opt, points_gradient_accum=accum.clone().to(DEV), denom=denom.clone().to(DEV),
                                 max_radii2D=torch.zeros(3000, device=DEV), max_grad=max_grad, min_opacity=min_opacity,
                                 scene_extent=1.0, percent_dense=0.01, params_to_densify=[n for n, _, _ in names])
    snap = _snapshot(opt)
    torch.cuda.manual_seed(SEED)
    with torch.no_grad():
        densify.sugar_densify_and_prune(dens, max_screen_size=mss)  # max_grad, min_opacity and extent from the densifier
    rng = torch.cuda.get_rng_state()
    for g in opt.param_groups:
        assert g["params"][0] is dict((n, getattr(model, a)) for n, a, _ in names)[g["name"]]
    groups = {g["name"]: (g["params"][0].detach(), opt.state.get(g["params"][0])) for g in opt.param_groups}
    moments = {n: (s[1], s[2]) for n, s in snap.items()}
    torch.cuda.manual_seed(SEED)
    with torch.no_grad():
        new, new_m, tags = DR.sequential({n: s[0] for n, s in snap.items()}, moments, accum.to(DEV), denom.to(DEV), max_grad,
                                         min_opacity, 1.0, mss, 0.01, DR.sugar_rotation,
                                         names=("points", "all_densities", "scales", "quaternions"))
    assert torch.equal(rng, torch.cuda.get_rng_state())
    split = _split_rows(accum.to(DEV), denom.to(DEV), snap["scales"][0], max_grad, 1.0, 0.01)
    _check_against_restatement(new, new_m, tags, groups, snap, 3000,
                               lambda tg: _child_bound(tg, 3000, split, snap["scales"][0], 8 * U), "points")
    assert dens.points_gradient_accum.shape == (tags.numel(), 1) and not dens.points_gradient_accum.any()


def test_errors():
    from autovfx_b200 import densify
    raw, accum, denom, *_ = make_case("default", 100, 4, seed=1)
    m = _gs_model(types.SimpleNamespace(), raw, accum, denom, "none", 1)
    m.optimizer.param_groups.pop(2)
    with pytest.raises(ValueError, match="f_rest"):
        densify.densify_and_prune(m, 2e-4, 0.005, 1.0, 20)
    m = _gs_model(types.SimpleNamespace(), raw, accum, denom, "none", 1)
    m.optimizer.param_groups[0]["params"][0] = nn.Parameter(m._xyz.detach().double())
    with pytest.raises(ValueError, match="xyz"):
        densify.densify_and_prune(m, 2e-4, 0.005, 1.0, 20)
    m = _gs_model(types.SimpleNamespace(), raw, accum, denom, "none", 1)
    m.optimizer.param_groups[4]["params"][0] = nn.Parameter(m._scaling.detach().t().contiguous().t())
    with pytest.raises(ValueError, match="scaling"):
        densify.densify_and_prune(m, 2e-4, 0.005, 1.0, 20)
