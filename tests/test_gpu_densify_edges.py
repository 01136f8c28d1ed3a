"""Densification on the GPU at its decision boundaries: gsr_densify_plan through the C ABI against densify_ref.plan_map run on
the device, and the densify_and_prune drop-ins against densify_ref.sequential run on CUDA, on rows exactly on a threshold and one
float32 ulp either side (tests/test_densify_sample_edges_cpu.tie_case), on non-finite rows, at every block and scan-chunk edge
of the plan, and gsr_densify_stats at its edges.  Run with -m gpu on an H100.

Clone tests torch.norm(grads, dim=-1) >= max_grad and split tests grads >= max_grad.  Over grads' single column torch.norm is
|g|; a rounded sqrt(g * g) equals |g| except where g * g is subnormal or overflows, so the rows that tell the two apart sit at a
max_grad near 1e-21.
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
from tests import test_densify_sample_edges_cpu as E  # noqa: E402
from tests import test_gpu_densify as TG  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = TG.U
SUGAR_NAMES = (("points", "_points", "xyz"), ("all_densities", "all_densities", "opacity"), ("scales", "_scales", "scaling"),
               ("quaternions", "_quaternions", "rotation"), ("sh_coordinates_dc", "_sh_coordinates_dc", "f_dc"),
               ("sh_coordinates_rest", "_sh_coordinates_rest", "f_rest"))


@pytest.fixture(scope="module", autouse=True)
def _lib():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import densify  # noqa: F401  (fails loudly if the CUDA library is missing)


def _same_bits(a, b, what=""):
    """NaN exactly where b has NaN, the same bit pattern everywhere else."""
    assert a.shape == b.shape, what
    nan = b.isnan()
    assert torch.equal(a.isnan(), nan), what
    assert torch.equal(a.view(torch.int32)[~nan], b.view(torch.int32)[~nan]), what


# ------------------------------------------------------------------------------------------------------------ the plan (C ABI)
def _plan(accum, denom, scaling, opacity, max_grad, dense_thr, min_opacity, use_screen, mss, big_thr):
    from autovfx_b200 import _lib as L
    P = scaling.shape[0]
    dst = torch.full((5, P), -7, dtype=torch.int32, device=DEV)
    totals = torch.full((2,), -7, dtype=torch.int32, device=DEV)
    nbytes = L.lib.gsr_densify_plan_bytes(P)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=DEV)
    rc = L.lib.gsr_densify_plan(P, accum.data_ptr(), denom.data_ptr(), scaling.data_ptr(), opacity.data_ptr(), max_grad, dense_thr,
                                min_opacity, int(use_screen), mss, big_thr, dst.data_ptr(), totals.data_ptr(), ws.data_ptr(), nbytes,
                                L.stream_ptr(torch.device(DEV)))
    L.check(rc, "gsr_densify_plan")
    return dst, totals


def _tags(dst, totals):
    """The final row -> source tag map the plan's four streams describe; checks the split-index stream on the way."""
    P = dst.shape[1]
    S, P2 = totals.tolist()
    rows = torch.arange(P, device=DEV)
    out = torch.full((P2,), -1, dtype=torch.int64, device=DEV)
    n = 0
    for s in range(4):
        keep = dst[s] >= 0
        n += int(keep.sum())
        out[dst[s][keep].long()] = s * P + rows[keep]
    assert n == P2 and bool((out >= 0).all())
    split = dst[4] >= 0
    assert int(split.sum()) == S and torch.equal(dst[4][split].long(), torch.arange(S, device=DEV))
    return out, S


def _check_plan(accum, denom, scaling, opacity, max_grad, dense_thr, min_opacity, mss, big_thr):
    """The kernel's plan equals plan_map on the device; returns the tags."""
    extent, pd = E.extent_pd(dense_thr, big_thr)
    dst, totals = _plan(accum, denom, scaling, opacity, max_grad, dense_thr, min_opacity, bool(mss), float(mss or 0.0), big_thr)
    got, S = _tags(dst, totals)
    want, S_want = DR.plan_map(accum, denom, scaling, opacity, max_grad, min_opacity, extent, mss, pd)
    assert S == S_want and torch.equal(got, want)
    return got


@pytest.mark.parametrize("mss", [20, None])
@pytest.mark.parametrize("grad", ["exact", "sqrt_up", "sqrt_down"])
def test_plan_at_the_ties(grad, mss):
    c = E.tie_case(DEV, grad)
    E.assert_ties(c)
    tags = _check_plan(c["accum"], c["denom"], c["scaling"], c["opacity"], c["max_grad"], c["dense_thr"], c["min_opacity"], mss,
                       c["big_thr"])
    if grad != "exact":
        # torch.norm over the single column is |g|; rows one ulp from max_grad where a rounded sqrt(g * g) would decide otherwise
        g = (c["accum"] / c["denom"]).reshape(-1)
        assert torch.equal(torch.norm(g[:, None], dim=-1), g.abs())
        sq, M = torch.sqrt(g * g), c["max_grad"]
        near = (g == E.pred(M)) | (g == M) | (g == E.succ(M))
        odd = (sq >= M) & (g < M) if grad == "sqrt_up" else (sq < M) & (g >= M)
        small = torch.exp(c["scaling"]).max(1).values <= c["dense_thr"]
        assert bool((near & odd & small).any()) and bool((near & odd & ~small).any())
        # and the literal replay (torch.norm) agrees
        extent, pd = E.extent_pd(c["dense_thr"], c["big_thr"])
        params = {k: v.to(DEV) for k, v in E.rest_of_model(g.numel(), 1).items()}
        params.update(scaling=c["scaling"], opacity=c["opacity"])
        _, _, want = DR.sequential(params, {}, c["accum"], c["denom"], M, c["min_opacity"], extent, mss, pd, DR.build_rotation)
        assert torch.equal(tags, want)


def test_plan_screen_size_zero_prunes_nothing_for_screen_size():
    """use_screen with max_screen_size 0: the screen-space test compares max_radii2D = 0 (reset by the postfix) with 0, which
    prunes nothing; the world-space test still applies."""
    c = E.tie_case(DEV)
    extent, pd = E.extent_pd(c["dense_thr"], c["big_thr"])
    dst, totals = _plan(c["accum"], c["denom"], c["scaling"], c["opacity"], c["max_grad"], c["dense_thr"], c["min_opacity"], True, 0.0,
                        c["big_thr"])
    got, _ = _tags(dst, totals)
    want, _ = DR.plan_map(c["accum"], c["denom"], c["scaling"], c["opacity"], c["max_grad"], c["min_opacity"], extent, 1e-30, pd)
    assert torch.equal(got, want)


# the five kinds of row of the block-edge plans: kept, kept + clone, pruned, split with children kept, split with children pruned
KINDS = [(E.S_SMALL, E.O_OK, 0.0), (E.S_SMALL, E.O_OK, E.G_HI), (E.S_SMALL, E.O_LOW, 0.0), (E.S_SPLIT, E.O_OK, E.G_HI),
         (E.S_SPLIT, E.O_LOW, E.G_HI)]


def _kinds(P, seed):
    """A kind per row: random, lane 31 and the next lane 0 always of different kinds, every fourth block (from block 1) all
    pruned and every fourth (from block 2) all split with children kept."""
    g = torch.Generator().manual_seed(seed)
    k = torch.randint(0, 5, (P,), generator=g)
    i = torch.arange(P)
    w = i // 32
    k = torch.where(i % 32 == 31, w % 5, k)
    k = torch.where(i % 32 == 0, (w + 2) % 5, k)
    b = i // 1024
    k = torch.where(b % 4 == 1, torch.full_like(k, 2), k)
    k = torch.where(b % 4 == 2, torch.full_like(k, 3), k)
    return k


def _kind_rows(k):
    t = torch.tensor(KINDS, dtype=torch.float32)[k]
    P = k.shape[0]
    scaling = t[:, :1].expand(P, 3).contiguous()
    scaling[:, 1] = E.S_SMALL
    return (t[:, 2:3].contiguous().to(DEV), torch.ones(P, 1, device=DEV), scaling.to(DEV), t[:, 1:2].contiguous().to(DEV))


@pytest.mark.parametrize("P", [1, 2, 31, 32, 33, 1023, 1024, 1025, 2049, 204 * 1024, 205 * 1024 + 1, 1_100_000])
def test_plan_block_edges(P):
    """5 * nb + 1 scan entries: P = 204 * 1024 fits k_rs_scan's first 1024-entry chunk, 205 * 1024 + 1 does not."""
    k = _kinds(P, seed=P)
    accum, denom, scaling, opacity = _kind_rows(k)
    tags = _check_plan(accum, denom, scaling, opacity, float(E.F32(1.5e-4)), 0.5, 0.005, 20, 2.0)
    counts = torch.bincount(k, minlength=5).tolist()
    assert tags.numel() == counts[0] + 2 * counts[1] + 2 * counts[3]
    if P >= 1025:
        assert bool((k[1024:2048] == 2).all()) and int(k[1023]) != int(k[1024])
    if P >= 2049:
        assert bool((k[2048:3072] == 3).all())


# ------------------------------------------------------------------------------------------------------- the drop-ins (full)
def _split_mask(accum, denom, scaling, max_grad, extent, pd):
    from autovfx_b200 import densify
    g = (accum / denom).reshape(-1)
    g = torch.where(g.isnan(), torch.zeros_like(g), g)
    return (g >= densify._f32(max_grad)) & (torch.exp(scaling).max(dim=1).values > densify._f32(densify._times(pd, extent)))


def _check_bits(new, new_m, tags, groups, snap, bound_fn, name_xyz):
    """_check_against_restatement with NaN where the replay has NaN: bit patterns elsewhere, and the split children's xyz within
    the bound where both are finite, the same infinities and NaNs where not."""
    ch, bound = bound_fn(tags)
    for name, (p, st) in groups.items():
        want = new[name]
        if name == name_xyz:
            _same_bits(p[~ch], want[~ch], name)
            a, b = p[ch], want[ch]
            assert torch.equal(a.isnan(), b.isnan()), name
            fin = torch.isfinite(a) & torch.isfinite(b)
            assert torch.equal(a[~fin & ~a.isnan()], b[~fin & ~b.isnan()]), name
            lim = (bound.expand_as(a) + U * (a.abs() + b.abs()))
            assert bool(((a - b).abs()[fin] <= lim[fin]).all()), name
        else:
            _same_bits(p, want, name)
        if snap[name][1] is None:
            assert st is None, name
        else:
            assert st is not None and st["step"] is snap[name][3], name
            _same_bits(st["exp_avg"], new_m[name][0], name)
            _same_bits(st["exp_avg_sq"], new_m[name][1], name)


def _raw(scaling, opacity, seed):
    raw = {k: v.to(DEV) for k, v in E.rest_of_model(scaling.shape[0], seed).items()}
    raw.update(scaling=scaling.to(DEV), opacity=opacity.to(DEV))
    return raw


def _gs_full(raw, accum, denom, max_grad, min_opacity, extent, mss, pd, state="all", bits=False):
    """densify_and_prune on a GaussianModel-like object against sequential on CUDA; returns the replay's tags."""
    from autovfx_b200 import densify
    P = accum.shape[0]
    ours = TG._gs_model(types.SimpleNamespace(), raw, accum, denom, state, seed=5)
    ours.percent_dense = pd
    with torch.no_grad():  # the Adam steps that built the state moved the parameters off their constructed values
        for n, a in TG.GS_GROUPS:
            getattr(ours, a).copy_(raw[n])
    snap = TG._snapshot(ours.optimizer)
    torch.cuda.manual_seed(TG.SEED)
    with torch.no_grad():
        densify.densify_and_prune(ours, max_grad, min_opacity, extent, mss)
    groups = {g["name"]: (g["params"][0].detach(), ours.optimizer.state.get(g["params"][0])) for g in ours.optimizer.param_groups}
    moments = {n: (s[1], s[2]) for n, s in snap.items() if s[1] is not None}
    torch.cuda.manual_seed(TG.SEED)
    with torch.no_grad():
        new, new_m, tags = DR.sequential({n: s[0] for n, s in snap.items()}, moments, accum.to(DEV), denom.to(DEV), max_grad,
                                         min_opacity, extent, mss, pd, DR.build_rotation)
    split = _split_mask(accum.to(DEV), denom.to(DEV), snap["scaling"][0], max_grad, extent, pd)
    bound_fn = lambda tg: TG._child_bound(tg, P, split, snap["scaling"][0], 0.0)  # noqa: E731
    check = _check_bits if bits else TG._check_against_restatement
    if bits:
        check(new, new_m, tags, groups, snap, bound_fn, "xyz")
    else:
        check(new, new_m, tags, groups, snap, P, bound_fn, "xyz")
    assert ours.xyz_gradient_accum.shape == (tags.numel(), 1)
    return tags


def _sugar_full(raw, accum, denom, max_grad, min_opacity, extent, mss, pd, wanted=None, bits=False):
    """sugar_densify_and_prune on a SuGaRDensifier-like object (params_to_densify = wanted, all groups by default) against
    sequential on CUDA over the rebuilt groups; the other groups must be untouched.  Returns the replay's tags."""
    from autovfx_b200 import densify
    P = accum.shape[0]
    model = types.SimpleNamespace(binded_to_surface_mesh=False)
    for n, a, r in SUGAR_NAMES:
        setattr(model, a, nn.Parameter(raw[r].clone().to(DEV).contiguous().requires_grad_(True)))
        TG.LRS.setdefault(n, TG.LRS[r])
    opt = TG._adam_state([(n, getattr(model, a)) for n, a, _ in SUGAR_NAMES], "all", 3)
    with torch.no_grad():  # the Adam steps that built the state moved the parameters off their constructed values
        for n, a, r in SUGAR_NAMES:
            getattr(model, a).copy_(raw[r])
    wanted = [n for n, _, _ in SUGAR_NAMES] if wanted is None else wanted
    dens = types.SimpleNamespace(model=model, optimizer=opt, points_gradient_accum=accum.clone().to(DEV), denom=denom.clone().to(DEV),
                                 max_radii2D=torch.zeros(P, device=DEV), max_grad=max_grad, min_opacity=min_opacity,
                                 scene_extent=extent, percent_dense=pd, params_to_densify=wanted)
    snap = TG._snapshot(opt)
    before = {g["name"]: (g["params"][0], opt.state[g["params"][0]]) for g in opt.param_groups}
    torch.cuda.manual_seed(TG.SEED)
    with torch.no_grad():
        densify.sugar_densify_and_prune(dens, max_screen_size=mss)
    groups = {}
    for g in opt.param_groups:
        p, n = g["params"][0], g["name"]
        assert p is getattr(model, dict((k, a) for k, a, _ in SUGAR_NAMES)[n])
        if n in wanted:
            groups[n] = (p.detach(), opt.state.get(p))
        else:  # untouched: the same parameter, values and state
            assert p is before[n][0] and opt.state[p] is before[n][1], n
            _same_bits(p.detach(), snap[n][0], n)
            _same_bits(before[n][1]["exp_avg"], snap[n][1], n)
            _same_bits(before[n][1]["exp_avg_sq"], snap[n][2], n)
    moments = {n: (s[1], s[2]) for n, s in snap.items() if n in wanted}
    torch.cuda.manual_seed(TG.SEED)
    with torch.no_grad():
        new, new_m, tags = DR.sequential({n: s[0] for n, s in snap.items() if n in wanted}, moments, accum.to(DEV), denom.to(DEV),
                                         max_grad, min_opacity, extent, mss, pd, DR.sugar_rotation,
                                         names=("points", "all_densities", "scales", "quaternions"))
    split = _split_mask(accum.to(DEV), denom.to(DEV), snap["scales"][0], max_grad, extent, pd)
    bound_fn = lambda tg: TG._child_bound(tg, P, split, snap["scales"][0], 8 * U)  # noqa: E731
    if bits:
        _check_bits(new, new_m, tags, groups, snap, bound_fn, "points")
    else:
        TG._check_against_restatement(new, new_m, tags, groups, snap, P, bound_fn, "points")
    assert dens.points_gradient_accum.shape == (tags.numel(), 1)
    return tags


@pytest.mark.parametrize("mode", ["3dgs", "sugar"])
@pytest.mark.parametrize("mss", [20, None])
def test_drop_ins_at_the_ties(mode, mss):
    c = E.tie_case(DEV)
    E.assert_ties(c)
    extent, pd = E.extent_pd(c["dense_thr"], c["big_thr"])
    raw = _raw(c["scaling"], c["opacity"], seed=2)
    run = _gs_full if mode == "3dgs" else _sugar_full
    tags = run(raw, c["accum"], c["denom"], c["max_grad"], c["min_opacity"], extent, mss, pd)
    assert (tags // c["scaling"].shape[0] >= 2).any()


def _extent_pair():
    """A float extent e for which f32(0.01 * e) (double product, a Python extent) and f32(f32(0.01) * f32(e)) (a tensor extent)
    differ, with both in the range where exp reaches every float."""
    for e in np.arange(100.0, 140.0, 0.37):
        e = float(E.F32(e))
        a, b = float(E.F32(0.01 * e)), float(E.F32(E.F32(0.01) * E.F32(e)))
        if a != b:
            return e, a, b
    raise AssertionError("no extent found")


@pytest.mark.parametrize("mode", ["3dgs", "sugar"])
def test_python_and_tensor_extents_round_differently(mode):
    from autovfx_b200 import densify
    e, a, b = _extent_pair()
    et = torch.tensor(e, dtype=torch.float32)
    assert densify._f32(densify._times(0.01, e)) == a and densify._f32(densify._times(0.01, et)) == b and a != b
    # rows with their largest scale on each rounding and one ulp either side, all with a gradient above max_grad
    targets = sorted({E.pred(min(a, b)), a, b, E.succ(max(a, b))})
    s = E.preimages(torch.exp, float(np.log(a)), targets, DEV)
    P = 4 * len(s)
    scaling = torch.full((P, 3), E.S_SMALL, device=DEV)
    scaling[:, 0] = torch.tensor(s, device=DEV).repeat(4)
    opacity = torch.full((P, 1), E.O_OK, device=DEV)
    accum, denom = torch.full((P, 1), E.G_HI, device=DEV), torch.ones(P, 1, device=DEV)
    mx = torch.exp(scaling).max(1).values
    assert bool(((mx <= a) != (mx <= b)).any())  # some row is cloned under one rounding and split under the other
    raw = _raw(scaling, opacity, seed=4)
    run = _gs_full if mode == "3dgs" else _sugar_full
    t_float = run(raw, accum, denom, 2e-4, 0.005, e, 20, 0.01)
    t_tensor = run(raw, accum, denom, 2e-4, 0.005, et, 20, 0.01)
    assert not torch.equal(t_float, t_tensor), (mx.tolist(), a, b, t_float.tolist())


def _non_finite_case():
    """Rows with NaN, +inf and -inf scaling components and raw opacities, accum > 0 over denom 0, and split rows with a zero and
    a NaN quaternion, among ordinary rows."""
    nan, inf = float("nan"), float("inf")
    rows = []  # (s3, o, accum, denom, quaternion or None)
    for v in (nan, inf, -inf):
        for c in range(3):
            for s_other, acc in ((E.S_SMALL, 0.0), (E.S_SMALL, E.G_HI), (E.S_SPLIT, E.G_HI)):
                s3 = [s_other] * 3
                s3[c] = v
                rows.append((s3, E.O_OK, acc, 1.0, None))
        for s, acc in ((E.S_SMALL, 0.0), (E.S_SMALL, E.G_HI), (E.S_SPLIT, E.G_HI)):
            rows.append(([s] * 3, v, acc, 1.0, None))
    for s in (E.S_SMALL, E.S_SPLIT):
        rows.append(([s] * 3, E.O_OK, E.G_HI, 0.0, None))   # accum / 0 = inf
        rows.append(([s] * 3, E.O_OK, 0.0, 0.0, None))      # 0 / 0 = NaN -> 0
    for q in ([0.0, 0.0, 0.0, 0.0], [nan, 0.5, 0.5, 0.5], [0.5, 0.5, nan, 0.5]):
        rows.append(([E.S_SPLIT, E.S_SMALL, E.S_SMALL], E.O_OK, E.G_HI, 1.0, q))
    for o in (E.O_OK, E.O_LOW):
        for s, acc in ((E.S_SMALL, 0.0), (E.S_SMALL, E.G_HI), (E.S_SPLIT, E.G_HI)):
            rows.append(([s] * 3, o, acc, 1.0, None))
    f = lambda x: torch.tensor(x, dtype=torch.float32, device=DEV)  # noqa: E731
    scaling, opacity = f([r[0] for r in rows]), f([[r[1]] for r in rows])
    accum, denom = f([[r[2]] for r in rows]), f([[r[3]] for r in rows])
    raw = _raw(scaling, opacity, seed=6)
    for i, r in enumerate(rows):
        if r[4] is not None:
            raw["rotation"][i] = f(r[4])
    return raw, accum, denom


@pytest.mark.parametrize("mode", ["3dgs", "sugar"])
@pytest.mark.parametrize("mss", [20, None])
def test_non_finite_rows(mode, mss):
    raw, accum, denom = _non_finite_case()
    P = accum.shape[0]
    E_, pd = E.extent_pd(0.5, 2.0)
    _check_plan(accum, denom, raw["scaling"], raw["opacity"], float(E.F32(1.5e-4)), 0.5, 0.005, mss, 2.0)
    run = _gs_full if mode == "3dgs" else _sugar_full
    tags = run(raw, accum, denom, 1.5e-4, 0.005, E_, mss, pd, bits=True)
    # the zero- and NaN-quaternion rows were split and their children's xyz are NaN in the replay
    q_bad = (raw["rotation"] == 0).all(1) | raw["rotation"].isnan().any(1)
    kind, src = tags // P, tags % P
    assert bool((q_bad[src] & (kind >= 2)).sum() == 2 * int(q_bad.sum()))


@pytest.mark.parametrize("P", [1, 1025])
@pytest.mark.parametrize("mode", ["3dgs", "sugar"])
def test_drop_ins_at_block_edges(P, mode):
    k = _kinds(P, seed=7 + P)
    if P == 1:
        k[:] = 3  # the one row is split
    accum, denom, scaling, opacity = _kind_rows(k)
    E_, pd = E.extent_pd(0.5, 2.0)
    run = _gs_full if mode == "3dgs" else _sugar_full
    tags = run(_raw(scaling, opacity, seed=8), accum, denom, 1.5e-4, 0.005, E_, 20, pd)
    assert tags.numel() == 2 if P == 1 else tags.numel() > 0


@pytest.mark.parametrize("missing", [("sh_coordinates_rest",), ("sh_coordinates_dc", "sh_coordinates_rest")])
def test_sugar_params_to_densify_subset(missing):
    c = E.tie_case(DEV)
    extent, pd = E.extent_pd(c["dense_thr"], c["big_thr"])
    raw = _raw(c["scaling"], c["opacity"], seed=9)
    wanted = [n for n, _, _ in SUGAR_NAMES if n not in missing]
    _sugar_full(raw, c["accum"], c["denom"], c["max_grad"], c["min_opacity"], extent, 20, pd, wanted=wanted)


# -------------------------------------------------------------------------------------------------------------- statistics
@pytest.mark.parametrize("C", [2, 3, 4])
@pytest.mark.parametrize("P", [1, 255, 256, 257, 1025])
def test_stats_edges(P, C):
    """update_densification_stats and add_densification_stats against the trainer's torch lines, bit for bit, over three steps:
    random grads with inf and NaN rows, a step with an all-False mask, NaN max_radii2D, radii = 16_777_217."""
    from autovfx_b200 import densify
    g = torch.Generator().manual_seed(P * 10 + C)
    z = lambda *s: torch.zeros(s, device=DEV)  # noqa: E731
    max_r = (torch.rand(P, generator=g) * 40).to(DEV)
    radii = torch.randint(0, 60, (P,), generator=g, dtype=torch.int32).to(DEV)
    special = [(16_777_217, 16_777_215.0), (16_777_217, float("nan")), (3, float("nan"))]
    for i, (r, m) in enumerate(special if P > 1 else special[1:2]):
        radii[(i * 97) % P], max_r[(i * 97) % P] = r, m
    gs = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1), max_radii2D=max_r.clone())
    add = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1))
    want = types.SimpleNamespace(xyz_gradient_accum=z(P, 1), denom=z(P, 1), max_radii2D=max_r.clone())
    for step in range(3):
        grad = torch.randn(P, C, generator=g) * 1e-3
        if step == 1:
            grad[:: 5, 0] = float("inf")
            grad[2:: 7, 1] = -float("inf")
            grad[3:: 11, 0] = float("nan")
        vis = torch.rand(P, generator=g) < 0.6
        vis[0] = True
        if step == 2:
            vis[:] = False
        vs = types.SimpleNamespace(grad=grad.to(DEV).contiguous())
        vis, r = vis.to(DEV), radii
        with torch.no_grad():
            densify.update_densification_stats(gs, vs, r, vis)
            densify.add_densification_stats(add, vs, vis)
            want.max_radii2D[vis] = torch.max(want.max_radii2D[vis], r[vis])
            want.xyz_gradient_accum[vis] += torch.norm(vs.grad[vis, :2], dim=-1, keepdim=True)
            want.denom[vis] += 1
        for m in (gs, add):
            _same_bits(m.xyz_gradient_accum, want.xyz_gradient_accum, step)
            _same_bits(m.denom, want.denom, step)
        _same_bits(gs.max_radii2D, want.max_radii2D, step)
    assert bool(want.max_radii2D.isnan()[0]) if P == 1 else bool(want.max_radii2D.isnan().any())
    if P > 1:
        assert bool((want.max_radii2D == 16_777_216.0).any())
    if P >= 5:
        assert bool(want.xyz_gradient_accum.isinf().any()) and bool(want.xyz_gradient_accum.isnan().any())
