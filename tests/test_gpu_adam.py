"""The CUDA Adam step (autovfx_b200.optim) against torch.optim.Adam with the trainers' arguments (lr=0.0, eps=1e-15, every other
option at its default: the foreach path) in the same process.  Run with -m gpu on an H100.

Twin models start from the same values and receive the same gradients; after every step each parameter, exp_avg and exp_avg_sq
must be bit-identical (compared as int32 bits, NaN by position) and every step count equal.
"""
import copy
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gs_layout(P, M):
    """GaussianModel.training_setup's groups (gaussian_model.py:164-173), spatial_lr_scale 5."""
    return [("xyz", (P, 3), 0.00016 * 5.0), ("f_dc", (P, 1, 3), 0.0025), ("f_rest", (P, M - 1, 3), 0.0025 / 20.0),
            ("opacity", (P, 1), 0.05), ("scaling", (P, 3), 0.005), ("rotation", (P, 4), 0.001)]


def sugar_layout(P, M):
    """SuGaROptimizer's groups (sugar_optimizer.py:68-85), spatial_lr_scale 5."""
    return [("points", (P, 3), 0.00016 * 5.0), ("sh_coordinates_dc", (P, 1, 3), 0.0025),
            ("sh_coordinates_rest", (P, M - 1, 3), 0.0025 / 20.0), ("all_densities", (P, 1), 0.05), ("scales", (P, 3), 0.005),
            ("quaternions", (P, 4), 0.001)]


def _optimizers(layout, seed, views=False):
    """(torch Adam, library Adam) over two identical sets of parameters.  views: each parameter is a view at a 4-byte offset into a
    larger tensor, so that its descriptor takes the scalar path."""
    from autovfx_b200.optim import use_cuda_adam
    g = torch.Generator().manual_seed(seed)
    init = [torch.randn(shape, generator=g) for _, shape, _ in layout]
    out = []
    for _ in range(2):
        ps = []
        for x in init:
            if views:
                buf = torch.empty(x.numel() + 1, device=DEV)
                buf[1:] = x.flatten().to(DEV)
                ps.append(nn.Parameter(buf[1:].view(x.shape)))
            else:
                ps.append(nn.Parameter(x.clone().to(DEV)))
        out.append(torch.optim.Adam([{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(ps, layout)], lr=0.0, eps=1e-15))
    out[1] = use_cuda_adam(out[1])
    return out


def _params(opt):
    return [p for grp in opt.param_groups for p in grp["params"]]


def assert_bits_equal(a, b, what):
    a, b = a.detach().contiguous(), b.detach().contiguous()
    assert a.shape == b.shape and a.dtype == b.dtype == torch.float32, what
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN at different positions" % what
    ia, ib = a.view(torch.int32)[~na], b.view(torch.int32)[~nb]
    bad = int((ia != ib).sum())
    assert bad == 0, "%s: %d of %d elements differ, first %s vs %s" % (what, bad, ia.numel(), a[~na][ia != ib][:4].tolist(),
                                                                        b[~nb][ia != ib][:4].tolist())


def assert_same(ref, ours, what=""):
    for gi, (ga, gb) in enumerate(zip(ref.param_groups, ours.param_groups)):
        for pa, pb in zip(ga["params"], gb["params"]):
            name = "%s group %s" % (what, ga.get("name", gi))
            assert_bits_equal(pa, pb, name + " param")
            sa, sb = ref.state.get(pa, {}), ours.state.get(pb, {})
            assert set(sa) == set(sb), name
            if sa:
                assert_bits_equal(sa["exp_avg"], sb["exp_avg"], name + " exp_avg")
                assert_bits_equal(sa["exp_avg_sq"], sb["exp_avg_sq"], name + " exp_avg_sq")
                assert sb["step"].device.type == "cpu" and sb["step"].dtype == sa["step"].dtype
                assert float(sa["step"]) == float(sb["step"]), name


def _grad(shape, gen, kind):
    x = torch.randn(shape, generator=gen) * 1e-3
    if kind == "plain":
        return x
    flat = x.view(-1)
    n = flat.numel()
    sel = torch.randint(0, 8, (n,), generator=gen)
    specials = torch.tensor([0.0, -0.0, 1e-40, -3e-42, 3e38, -1e30, float("inf"), float("nan")])
    pick = torch.rand(n, generator=gen) < 0.3
    flat[pick] = specials[sel[pick]]
    return x


def run_twins(ref, ours, steps, seed, lr_schedule=None, skip=None, kinds=None, check_every=True):
    """Step both optimizers `steps` times with the same gradients.  lr_schedule(it) -> xyz lr; skip(it, gi) -> True leaves group
    gi without a gradient; kinds(it) -> gradient kind."""
    gen = torch.Generator().manual_seed(seed)
    pr, po = _params(ref), _params(ours)
    for it in range(steps):
        if lr_schedule is not None:
            ref.param_groups[0]["lr"] = ours.param_groups[0]["lr"] = lr_schedule(it)
        for gi, (a, b) in enumerate(zip(pr, po)):
            if skip is not None and skip(it, gi):
                a.grad = b.grad = None
                continue
            gr = _grad(a.shape, gen, kinds(it) if kinds else "plain").to(DEV)
            a.grad, b.grad = gr.clone(), gr.clone()
        ref.step()
        ours.step()
        if check_every or it == steps - 1:
            torch.cuda.synchronize()
            assert_same(ref, ours, "step %d" % (it + 1))


def _xyz_lr(it):  # the exponential schedule of get_expon_lr_func, sampled at different iterations
    return 0.00016 * 5.0 * (0.01 ** (it / 30.0))


@pytest.fixture(scope="module", autouse=True)
def _device():
    assert torch.cuda.is_available()
    torch.cuda.set_device(DEV)


@pytest.mark.parametrize("layout", [gs_layout, sugar_layout], ids=["3dgs", "sugar"])
@pytest.mark.parametrize("P", [1, 1003, 4098])
@pytest.mark.parametrize("steps", [1, 2, 20])
def test_steps_match_torch(layout, P, steps):
    ref, ours = _optimizers(layout(P, 16), seed=P + steps)
    run_twins(ref, ours, steps, seed=steps, lr_schedule=_xyz_lr)


@pytest.mark.parametrize("M", [1, 4, 25])
def test_sh_widths_and_scalar_path(M):
    ref, ours = _optimizers(gs_layout(517, M), seed=M)
    run_twins(ref, ours, 5, seed=M, lr_schedule=_xyz_lr)
    ref, ours = _optimizers(gs_layout(517, M), seed=M, views=True)
    assert all(p.data_ptr() % 16 != 0 for p in _params(ours) if p.numel() > 0)
    run_twins(ref, ours, 5, seed=M, lr_schedule=_xyz_lr)


def test_skipped_groups_and_zero_lr():
    """Opacity without a gradient on every third step (reset_opacity), every group on step 4 (a densify iteration), rotation at
    lr 0: skipped tensors keep their values, moments and step count."""
    layout = gs_layout(1501, 16)
    layout[5] = ("rotation", layout[5][1], 0.0)
    ref, ours = _optimizers(layout, seed=3)

    def skip(it, gi):
        return it == 4 or (gi == 3 and it % 3 == 0)
    run_twins(ref, ours, 12, seed=5, lr_schedule=_xyz_lr, skip=skip)
    steps = [float(ours.state[p]["step"]) for p in _params(ours)]
    assert steps[3] == 7.0 and steps[0] == 11.0
    # the group first seen without a gradient has no state until its first gradient
    ref, ours = _optimizers(layout, seed=4)
    run_twins(ref, ours, 3, seed=6, skip=lambda it, gi: gi == 2 and it < 2)
    assert float(ours.state[_params(ours)[2]]["step"]) == 1.0


def test_special_gradients():
    """Gradients that are +-0, subnormal, huge, +-Inf or NaN on 30 % of the elements, every other step."""
    ref, ours = _optimizers(gs_layout(2049, 16), seed=11)
    run_twins(ref, ours, 8, seed=12, lr_schedule=_xyz_lr, kinds=lambda it: "specials" if it % 2 == 0 else "plain")
    st = ours.state[_params(ours)[2]]
    assert torch.isnan(st["exp_avg"]).any() and torch.isinf(st["exp_avg_sq"]).any()


def test_more_tensors_than_one_launch_takes():
    from autovfx_b200 import _lib
    n = _lib.GSR_ADAM_MAX_TENSORS + 9
    layout = [("t%d" % i, (37 + i,), 10.0 ** -(1 + i % 4)) for i in range(n)]
    ref, ours = _optimizers(layout, seed=2)
    run_twins(ref, ours, 3, seed=2)


def _seed_state(opt, step, seed):
    gen = torch.Generator().manual_seed(seed)
    for p in _params(opt):
        opt.state[p] = {"step": torch.tensor(float(step)), "exp_avg": (torch.randn(p.shape, generator=gen) * 1e-3).to(DEV),
                        "exp_avg_sq": (torch.rand(p.shape, generator=gen) * 1e-6).to(DEV)}


@pytest.mark.parametrize("layout", [gs_layout, sugar_layout], ids=["3dgs", "sugar"])
def test_state_dict_round_trips_at_step_15000(layout):
    from autovfx_b200.optim import use_cuda_adam
    lay = layout(1003, 16)
    ref, ours = _optimizers(lay, seed=21)
    _seed_state(ref, 14999, 22)
    sd = copy.deepcopy(ref.state_dict())  # load_state_dict keeps tensors that are already on the device: no aliasing of moments
    # torch -> library: ours resumes from torch's state_dict
    ours.load_state_dict(sd)
    assert_same(ref, ours, "loaded")
    run_twins(ref, ours, 3, seed=23, lr_schedule=lambda it: 1.6e-6 * (it + 1))
    assert float(ours.state[_params(ours)[0]]["step"]) == 15002.0
    # library -> torch: a fresh torch Adam resumes from ours' state_dict, a fresh library Adam from torch's
    ref2 = torch.optim.Adam([{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(_params(ours), lay)], lr=0.0, eps=1e-15)
    ref2.load_state_dict(copy.deepcopy(ours.state_dict()))
    ours2 = use_cuda_adam(torch.optim.Adam([{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(_params(ref), lay)],
                                           lr=0.0, eps=1e-15))
    ours2.load_state_dict(copy.deepcopy(ref.state_dict()))
    assert type(ref2) is torch.optim.Adam
    run_twins(ref2, ours2, 3, seed=24, lr_schedule=lambda it: 1.6e-6)


def _gs_model(opt, names, attrs):
    m = types.SimpleNamespace(optimizer=opt, percent_dense=0.01)
    for grp, attr in zip(opt.param_groups, attrs):
        setattr(m, attr, grp["params"][0])
    P = m._xyz.shape[0]
    gen = torch.Generator().manual_seed(P)
    denom = torch.randint(0, 6, (P, 1), generator=gen).float()
    m.xyz_gradient_accum = (torch.rand(P, 1, generator=gen) * 5e-4 * denom).to(DEV)
    m.denom = denom.to(DEV)
    m.max_radii2D = torch.zeros(P, device=DEV)
    return m


def test_densify_and_prune_then_skipped_step_then_more_steps():
    """Train, densify_and_prune (which re-keys the state dicts onto new Parameters), a step on which no parameter has a gradient
    (torch updates nothing), then more steps: the library's optimizer stays bit-identical to torch's throughout."""
    from autovfx_b200 import densify
    attrs = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
    lay = gs_layout(3001, 16)
    ref, ours = _optimizers(lay, seed=31)
    with torch.no_grad():
        for opt in (ref, ours):
            _params(opt)[4].mul_(0.5).sub_(4.0)  # log-scales around exp(-4): some clone, some split
    run_twins(ref, ours, 4, seed=32, lr_schedule=_xyz_lr)
    models = [_gs_model(opt, [n for n, _, _ in lay], attrs) for opt in (ref, ours)]
    for m in models:
        torch.manual_seed(33)
        densify.densify_and_prune(m, 2e-4, 0.005, 1.0, 20)
    P2 = models[1]._xyz.shape[0]
    assert P2 != 3001 and type(ours) is not torch.optim.Adam
    assert all(ours.state[p]["exp_avg"].shape == p.shape for p in _params(ours))
    assert_same(ref, ours, "densified")
    run_twins(ref, ours, 1, seed=34, skip=lambda it, gi: True)
    assert float(ours.state[_params(ours)[0]]["step"]) == 4.0
    run_twins(ref, ours, 5, seed=35, lr_schedule=_xyz_lr)


def test_3m_gaussians_two_steps():
    ref, ours = _optimizers(gs_layout(3_000_001, 16), seed=41)
    run_twins(ref, ours, 2, seed=42, lr_schedule=_xyz_lr, check_every=False)
    del ref, ours
    torch.cuda.empty_cache()


def test_no_host_synchronisation():
    """A step with gradients issues no device synchronisation (torch.cuda.set_sync_debug_mode('error'))."""
    ref, ours = _optimizers(gs_layout(1003, 16), seed=51)
    run_twins(ref, ours, 1, seed=52)
    for p in _params(ours):
        p.grad = torch.ones_like(p)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ours.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
