"""Decision boundaries of densification and of SuGaR's sampler: the constructions the GPU edge tests
(test_gpu_densify_edges.py, test_gpu_sugar_sample_edges.py) build their ties with, checked on the CPU.

Densification: rows whose gradient, largest scale, split-child scale or opacity sits exactly on its threshold or one float32
ulp either side.  Every tie is found on the float grid with torch's own op on the device the test runs on (exp, sigmoid,
accum / denom), so the constructed row meets the threshold bit for bit.  Here the one-pass plan's restatement
(densify_ref.plan_map) must equal the literal clone -> split -> prune replay (densify_ref.sequential) on those rows.

Sampling: integer weights, so that every prefix T is exact in float64 and the total is a power of two; then u = T_k / total is
exact, u * total == T_k, and the search must return the next row of positive weight.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import densify_ref as DR  # noqa: E402
from tests import sugar_sample_ref as SR  # noqa: E402

F32 = np.float32


def pred(x):
    return float(np.nextafter(F32(x), F32(-np.inf)))


def succ(x):
    return float(np.nextafter(F32(x), F32(np.inf)))


def f32_grid(x0, device, n=1 << 15):
    """The 2n consecutive float32 values around float32(x0), on `device`."""
    base = int(torch.tensor([x0], dtype=torch.float32).view(torch.int32))
    return torch.arange(base - n, base + n, dtype=torch.int32).view(torch.float32).to(device)


def preimages(fn, x0, targets, device):
    """For each target, a float32 input s near x0 with fn(s) == target bit for bit (fn evaluated on `device`)."""
    grid = f32_grid(x0, device)
    y = fn(grid)
    out = []
    for t in targets:
        hit = torch.nonzero(y == t)
        assert hit.numel() > 0, ("no float32 input near %r reaches %r" % (x0, t))
        out.append(float(grid[hit[0, 0]]))
    return out


def threshold_ties(pairs, device):
    """(thr, [inputs reaching pred(thr), thr and succ(thr)] for each (fn, x0) in pairs): thr is the output nearest fn(x0) of the
    first pair that every fn reaches, with both float32 neighbours, from an input near its x0.  exp is not correctly rounded,
    so even where an input step moves it by a fraction of an ulp some outputs are never produced."""
    evals, common = [], None
    for fn, x0 in pairs:
        grid = f32_grid(x0, device)
        y = fn(grid)
        yi = torch.unique(y[y > 0]).view(torch.int32)  # positive floats: consecutive bit patterns are ulp neighbours
        good = yi[1:-1][(yi[1:-1] - yi[:-2] == 1) & (yi[2:] - yi[1:-1] == 1)]
        common = good if common is None else common[torch.isin(common, good)]
        evals.append((x0, grid, y))
    assert common.numel() > 0, "no output has both neighbours reachable"
    mid = evals[0][2][evals[0][1].numel() // 2].view(torch.int32)
    thr = float(common[(common - mid).abs().argmin()].view(torch.float32))
    out = []
    for x0, grid, y in evals:
        ins = []
        for t in (pred(thr), thr, succ(thr)):
            hit = torch.nonzero(y == t)
            assert hit.numel() > 0, ("no float32 input near %r reaches %r" % (x0, t))
            ins.append(float(grid[hit[0, 0]]))
        out.append(ins)
    return thr, out


def solve_accum(g, denom, device):
    """accum (float32) with fl(accum / denom) == g for every (g, denom) pair, searched around g * denom on `device`."""
    gt = torch.tensor(g, dtype=torch.float32)
    dt = torch.tensor(denom, dtype=torch.float32)
    base = (gt * dt).view(torch.int32)
    cand = (base[:, None] + torch.arange(-16, 17, dtype=torch.int32)).view(torch.float32).to(device)
    ok = (cand / dt.to(device)[:, None]) == gt.to(device)[:, None]
    assert bool(ok.any(1).all()), "some accum / denom cannot reach its target"
    return cand.gather(1, ok.int().argmax(1, keepdim=True)).squeeze(1)


def extent_pd(dense_thr, big_thr):
    """(extent, percent_dense) whose float32 thresholds are exactly dense_thr = f32(pd * extent) and big_thr = f32(0.1 * extent)."""
    extent = big_thr / 0.1
    pd = dense_thr / extent
    assert float(F32(pd * extent)) == dense_thr and float(F32(0.1 * extent)) == big_thr
    return extent, pd


def child_max_fn(s):
    """A split child's largest scale, as torch computes it: exp(log(exp(s) * (1 / 1.6f)))."""
    return torch.exp(torch.log(torch.exp(s) * (1.0 / torch.tensor(1.6, dtype=torch.float32, device=s.device))))


def sqrt_threshold(device, up):
    """A positive max_grad at which a rounded sqrt(fl(g * g)) and torch.norm's |g| decide differently for a row one ulp away
    (torch.norm over grads' single column is |g|, which the GPU tests assert).  In binary floating
    point sqrt(fl(g * g)) == |g| whenever g * g neither underflows nor overflows, so the threshold sits near 1e-21, where g * g
    is subnormal.  up: g = pred(M) has sqrt(fl(g * g)) >= M.  Otherwise g = M has sqrt(fl(g * g)) < M."""
    g = f32_grid(1e-21, device)
    h = torch.sqrt(g * g)
    k = int(torch.nonzero(h > g if up else h < g)[0, 0])
    return float(g[k + 1] if up else g[k])


# row values away from every threshold
S_SMALL, S_SPLIT, O_OK, O_LOW, G_HI = -1.0, 0.0, 3.0, -8.0, 1e-3
# the data the thresholds are taken from: dense_thr = exp(S_D), big_thr = exp(S_B), min_opacity = sigmoid(O_M).  Near these
# values a one-ulp step of the input moves exp, sigmoid and a child's scale (whose parent lies in [1.6, 2)) by less than one
# ulp of the output, so every float32 threshold and its two neighbours are reached.
S_D, S_B, O_M = -0.2, 0.15, 0.7


def tie_case(device, grad="exact"):
    """Rows on every threshold of the plan and one ulp either side, and the thresholds.  grad: 'exact' (max_grad =
    f32(1.5e-4): 3 * max_grad lies in [2, 4) * 2^e, so accum / 3 reaches every float near it), 'sqrt_up' or 'sqrt_down'
    (sqrt_threshold).  Returns a dict of scaling [R,3], opacity [R,1], accum [R,1], denom [R,1] on
    `device` and max_grad, dense_thr, big_thr, min_opacity (Python floats, exact float32 values)."""
    dev = torch.device(device)
    D, (s_D,) = threshold_ties([(torch.exp, S_D)], dev)
    B, (s_B, s_C) = threshold_ties([(torch.exp, S_B), (child_max_fn, float(np.log(np.exp(S_B) * 1.6)))], dev)
    m, (o_m,) = threshold_ties([(torch.sigmoid, O_M)], dev)
    M = float(F32(1.5e-4)) if grad == "exact" else sqrt_threshold(dev, grad == "sqrt_up")
    rows = []

    def add(s3, o=O_OK, g=0.0, den=1.0):
        rows.append((list(s3), o, g, den))

    def at(c, v):
        s3 = [S_SMALL] * 3
        s3[c] = v
        return s3

    # gradient ties, on the clone path (small scale) and the split path, through three denominators
    for gv in (pred(M), M, succ(M)):
        for den in (1.0, 3.0, 4.0):
            add([S_SMALL] * 3, g=gv, den=den)
            add([S_SPLIT, S_SMALL, S_SPLIT], g=gv, den=den)
    # largest scale on dense_thr: cloned at or below it, split above it; in each component
    for sv in s_D:
        for c in range(3):
            add(at(c, sv), g=G_HI)
            add(at(c, sv))
    # largest scale of an original row on big_thr (not split: its gradient is 0)
    for sv in s_B:
        for c in range(3):
            add(at(c, sv))
    # largest scale of a split child on big_thr
    for sv in s_C:
        for c in range(3):
            add(at(c, sv), g=G_HI)
    # opacity on min_opacity: kept, cloned and split rows
    for ov in o_m:
        add([S_SMALL] * 3, o=ov)
        add([S_SMALL] * 3, o=ov, g=G_HI)
        add([S_SPLIT] * 3, o=ov, g=G_HI)
    # rows away from every threshold
    for o in (O_OK, O_LOW):
        add([S_SMALL] * 3, o=o)
        add([S_SMALL] * 3, o=o, g=G_HI)
        add([S_SPLIT] * 3, o=o, g=G_HI)
    f = lambda x: torch.tensor(x, dtype=torch.float32, device=dev)  # noqa: E731
    return dict(scaling=f([r[0] for r in rows]).contiguous(), opacity=f([[r[1]] for r in rows]),
                accum=solve_accum([r[2] for r in rows], [r[3] for r in rows], dev)[:, None].contiguous(),
                denom=f([[r[3]] for r in rows]), max_grad=M, dense_thr=D, big_thr=B, min_opacity=m)


def assert_ties(c):
    """The case holds every tie it claims, and its two neighbours, evaluated on the case's device."""
    g = (c["accum"] / c["denom"]).reshape(-1)
    mx = torch.exp(c["scaling"]).max(1).values
    mxc = child_max_fn(c["scaling"]).max(1).values
    op = torch.sigmoid(c["opacity"]).reshape(-1)
    for vals, thr in ((g, c["max_grad"]), (mx, c["dense_thr"]), (mx, c["big_thr"]), (mxc, c["big_thr"]), (op, c["min_opacity"])):
        for t in (pred(thr), thr, succ(thr)):
            assert bool((vals == t).any()), (thr, t)
    for den in (1.0, 3.0, 4.0):
        assert bool(((g == c["max_grad"]) & (c["denom"].reshape(-1) == den)).any()), den


def rest_of_model(P, seed, M=4):
    """xyz, SH and raw rotation groups for P rows."""
    g = torch.Generator().manual_seed(seed)
    return {"xyz": torch.randn(P, 3, generator=g) * 2, "f_dc": torch.randn(P, 1, 3, generator=g),
            "f_rest": torch.randn(P, M - 1, 3, generator=g), "rotation": torch.randn(P, 4, generator=g)}


@pytest.mark.parametrize("mss", [20, None])
def test_plan_map_equals_sequential_at_the_ties(mss):
    c = tie_case("cpu")
    assert_ties(c)
    extent, pd = extent_pd(c["dense_thr"], c["big_thr"])
    P = c["scaling"].shape[0]
    params = rest_of_model(P, 1)
    params.update(scaling=c["scaling"], opacity=c["opacity"])
    torch.manual_seed(0)
    _, _, tags = DR.sequential(params, {}, c["accum"], c["denom"], c["max_grad"], c["min_opacity"], extent, mss, pd,
                               DR.build_rotation)
    want, S = DR.plan_map(c["accum"], c["denom"], c["scaling"], c["opacity"], c["max_grad"], c["min_opacity"], extent, mss, pd)
    assert torch.equal(tags, want)
    kind = tags // P
    assert S > 0 and (kind == 1).any() and (kind >= 2).any() and tags.numel() < 2 * P


def test_ulp_neighbours_decide_both_ways():
    """At each threshold the row on it and its two neighbours are not all decided alike: the ties are where decisions flip."""
    c = tie_case("cpu")
    extent, pd = extent_pd(c["dense_thr"], c["big_thr"])
    P = c["scaling"].shape[0]
    tags, _ = DR.plan_map(c["accum"], c["denom"], c["scaling"], c["opacity"], c["max_grad"], c["min_opacity"], extent, 20, pd)
    kind, src = tags // P, tags % P
    mx = torch.exp(c["scaling"]).max(1).values
    g = (c["accum"] / c["denom"]).reshape(-1)
    cloned = torch.zeros(P, dtype=torch.bool)
    cloned[src[kind == 1]] = True
    split_kept = torch.zeros(P, dtype=torch.bool)
    split_kept[src[kind == 2]] = True
    small = mx <= c["dense_thr"]
    assert cloned[(g == c["max_grad"]) & small].all() and not cloned[(g == pred(c["max_grad"])) & small].any()
    assert cloned[(mx == c["dense_thr"]) & (g > c["max_grad"])].all()
    assert split_kept[(mx == succ(c["dense_thr"])) & (g > c["max_grad"])].all()
    mxc = child_max_fn(c["scaling"]).max(1).values
    assert split_kept[(mxc == c["big_thr"]) & (g > c["max_grad"])].all()
    assert not split_kept[(mxc == succ(c["big_thr"])) & (g > c["max_grad"])].any()


# ------------------------------------------------------------------------------------------------------------------ sampling
def dyadic_case(seed=0, n_mid=2300):
    """Integer weights (strengths, volume=False) over ~2400 rows: leading selected zero-weight rows and unselected rows, a middle
    of weights 0..2 with a mask, one last selected row whose weight makes the total a power of two, then unselected rows.
    Every C and T is an integer below 2^25, exact in float64 in any order of addition.  Returns (strengths [P], mask [P],
    T as Python ints, total, index of the last positive row)."""
    rng = np.random.default_rng(seed)
    w = [0, 5, 0, 7]                 # rows 0 and 2 selected with weight 0 (C = 0), rows 1 and 3 unselected
    sel = [True, False, True, False]
    w += [int(x) for x in rng.integers(0, 3, n_mid)]
    sel += [bool(x) for x in rng.random(n_mid) < 0.8]
    C = T = 0
    for wi, si in zip(w, sel):
        if si:
            C += wi
            T += C
    m = int(np.ceil(np.log2(T + C + 1)))
    w.append(2 ** m - T - C)         # t = C + w, so the total is 2^m
    sel.append(True)
    assert 0 < w[-1] <= 2 ** 24      # exact in float32
    last = len(w) - 1
    w += [3, 9, 1]
    sel += [False, False, False]
    C = T = 0
    Ts = []
    for wi, si in zip(w, sel):
        if si:
            C += wi
            T += C
        Ts.append(T)
    assert Ts[-1] == 2 ** m
    return torch.tensor(w, dtype=torch.float32), torch.tensor(sel), Ts, 2 ** m, last


def tie_draws(Ts, total):
    """u = T_k / total for every distinct positive T_k below the total (exact), and the row each must select: the first row
    whose T exceeds T_k."""
    us, rows = [], []
    for k, t in enumerate(Ts):
        if 0 < t < total and (k == 0 or Ts[k - 1] != t):
            us.append(t / total)
            assert us[-1] * total == t
            rows.append(next(j for j in range(k + 1, len(Ts)) if Ts[j] > t))
    return us, rows


def test_dyadic_prefix_is_exact_and_ties_select_the_next_row():
    w, mask, Ts, total, last = dyadic_case()
    T = SR.prefix(SR.weights(torch.ones(w.shape[0], 3), w[:, None], mask, volume=False), mask)
    assert T.tolist() == [float(t) for t in Ts]
    us, rows = tie_draws(Ts, total)
    assert len(us) > 1000
    got, tot = SR.select_rows(T, torch.tensor(us, dtype=torch.float64))
    assert float(tot) == total and got.tolist() == rows
    # a tie always skips rows of zero weight: some selected row follows an unselected one
    assert any(Ts[r - 1] == Ts[r - 2] for r in rows if r >= 2)


def test_u_edges_select_the_first_and_last_positive_rows():
    w, mask, Ts, total, last = dyadic_case()
    first = next(k for k, t in enumerate(Ts) if t > 0)
    assert first >= 4 and Ts[:first] == [0] * first  # leading zero-weight and unselected rows
    assert not mask[last + 1:].any() and Ts[last] == total
    T = SR.prefix(SR.weights(torch.ones(w.shape[0], 3), w[:, None], mask, volume=False), mask)
    got, _ = SR.select_rows(T, torch.tensor([0.0, 1.0 - 2.0 ** -53], dtype=torch.float64))
    assert got.tolist() == [first, last]
