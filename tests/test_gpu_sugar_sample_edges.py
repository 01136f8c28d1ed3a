"""gsr_sugar_sample at its decision boundaries, through the C ABI with chosen u and z: exact ties u * total == T_k, u = 0 and
u = 1 - 2^-53, the step back from a zero-weight row that rounding raised above its predecessor, every block edge of the float64
prefix and of k_rs_scan's 1024-entry chunk (more than 1024 blocks), and a selection of one row, forward and backward.  Run with
-m gpu on an H100.

The workspace of gsr_sugar_sample starts with T [P] (float64): the prefix over all rows of t_i = mask_i C_i, stored as -T_i on
rows with t_i = 0.  The tests read it there and check |T| against sugar_sample_ref.prefix.
"""
import numpy as np
import pytest
import torch

from tests import sugar_sample_ref as SR
from tests import test_densify_sample_edges_cpu as E
from tests import test_gpu_sugar_sample as TS

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ptr(t):
    return None if t is None else t.data_ptr()


def _forward(N, f, volume, mask, strengths, u, z, points, scaling, quats):
    """sugar_field._sample_forward, keeping the workspace: returns (samples, rows, total, T)."""
    from autovfx_b200 import _lib
    P = points.shape[0]
    out = torch.empty((N, 3), dtype=torch.float32, device=DEV)
    idx = torch.empty(N, dtype=torch.int64, device=DEV)
    total = torch.empty(1, dtype=torch.float64, device=DEV)
    nbytes = _lib.lib.gsr_sugar_sample_bytes(P)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    rc = _lib.lib.gsr_sugar_sample(N, P, f, int(volume), _ptr(mask), _ptr(strengths), u.data_ptr(), z.data_ptr(), points.data_ptr(),
                                   scaling.data_ptr(), quats.data_ptr(), out.data_ptr(), idx.data_ptr(), total.data_ptr(),
                                   ws.data_ptr(), nbytes, _lib.stream_ptr(torch.device(DEV)))
    _lib.check(rc, "gsr_sugar_sample")
    return out, idx, total, ws[: 8 * P].view(torch.float64)


def _z(N, seed):
    return torch.randn(N, 3, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _same_bits(a, b):
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _dyadic():
    w, mask, Ts, total, last = E.dyadic_case()
    points, scaling, quats, _ = TS._scene(w.shape[0], seed=1, zero_volume=False)
    return w.to(DEV), mask.to(DEV), Ts, total, last, points, scaling, quats


def test_exact_ties_select_the_next_positive_row():
    """u = T_k / total with a power-of-two total: u * total == T_k exactly, and the row drawn is the first whose T exceeds it.
    u = 1 - 2^-53 draws the last positive row, which unselected rows follow."""
    w, mask, Ts, total, last, points, scaling, quats = _dyadic()
    us, rows = E.tie_draws(Ts, total)
    us.append(1.0 - 2.0 ** -53)
    rows.append(last)
    N = len(us)
    u, z = torch.tensor(us, dtype=torch.float64, device=DEV), _z(N, 2)
    x, idx, tot, T = _forward(N, 1.5, False, mask, w, u, z, points, scaling, quats)
    Tref = torch.tensor(Ts, dtype=torch.float64, device=DEV)
    assert torch.equal(T.abs(), Tref) and float(tot) == total
    t_pos = torch.diff(Tref, prepend=Tref.new_zeros(1)) > 0
    assert torch.equal(T > 0, t_pos)  # the sign marks the rows of zero weight
    assert not bool(mask[last + 1:].any()) and last + 1 < w.shape[0]
    assert idx.tolist() == rows
    _same_bits(x, SR.place(points, scaling, quats, idx, z, 1.5))


def test_u_zero_selects_the_first_positive_row():
    """u = 0: leading rows of zero weight (selected with C = 0, and unselected) have T = 0 and are passed over."""
    w, mask, Ts, total, last, points, scaling, quats = _dyadic()
    first = next(k for k, t in enumerate(Ts) if t > 0)
    assert first >= 4 and bool(mask[:first].any()) and not bool(mask[:first].all())
    N = 64
    x, idx, _, _ = _forward(N, 1.5, False, mask, w, torch.zeros(N, dtype=torch.float64, device=DEV), _z(N, 3), points, scaling, quats)
    assert bool((idx == first).all())
    _same_bits(x, SR.place(points, scaling, quats, idx, _z(N, 3), 1.5))


def _search(a, x):
    """k_sample_points' binary search over |T|: the first crossing of x."""
    lo, hi = 0, len(a) - 1
    while lo < hi:
        mid = (lo + hi) >> 1
        if a[mid] > x:
            hi = mid
        else:
            lo = mid + 1
    return lo


def test_step_back_from_a_raised_zero_weight_row():
    """Weights from 1e-30 to 1e30 and half the rows unselected: the parallel scan's roundings leave some unselected rows (t = 0)
    with |T_i| > |T_{i-1}|.  A u whose u * total lands in [|T_{i-1}|, |T_i|) finds row i, and the kernel must step back to the
    last row of positive weight before it."""
    P = 8192
    g = torch.Generator().manual_seed(3)
    w = (10.0 ** (torch.rand(P, generator=g, dtype=torch.float64) * 60 - 30)).float().to(DEV)
    mask = (torch.rand(P, generator=g) < 0.5).to(DEV)
    points, scaling, quats, _ = TS._scene(P, seed=4, zero_volume=False)
    one = torch.full((1,), 0.5, dtype=torch.float64, device=DEV)
    _, _, _, T0 = _forward(1, 1.0, False, mask, w, one, _z(1, 0), points, scaling, quats)
    T = T0.cpu().numpy().copy()
    a, zero = np.abs(T), ~(T > 0)
    total = a[-1]
    assert np.allclose(a, SR.prefix(SR.weights(scaling, w, mask, False), mask).cpu().numpy(), rtol=1e-12, atol=0)
    raised = np.nonzero(zero[1:] & (a[1:] > a[:-1]))[0] + 1
    assert raised.size > 0
    us, want = [], []
    for i in raised:
        u0 = np.array([a[i - 1] / total])
        for k in (0, 1, -1, 2, -2, 3, -3):
            u = float((u0.view(np.int64) + k).view(np.float64)[0])
            x = u * total
            if not (0 <= u < 1 and x < total):
                continue
            land = _search(a, x)
            if zero[land] and a[i - 1] <= x < a[i]:
                j = land
                while not T[j] > 0:
                    j -= 1
                us.append(u)
                want.append(j)
                break
    assert len(us) > 0, "no u lands on a raised zero-weight row"
    N = len(us)
    u, z = torch.tensor(us, dtype=torch.float64, device=DEV), _z(N, 5)
    x, idx, _, T1 = _forward(N, 1.5, False, mask, w, u, z, points, scaling, quats)
    assert torch.equal(T1.view(torch.int64), T0.view(torch.int64))  # deterministic
    assert idx.tolist() == want
    assert bool((T1[idx] > 0).all())
    _same_bits(x, SR.place(points, scaling, quats, idx, z, 1.5))


@pytest.mark.parametrize("how", ["all", "masked", "boundary"])
@pytest.mark.parametrize("P", [1, 1023, 1024, 1025, 2049, 1_048_577, 2_100_000])
def test_block_edges(P, how):
    """Rows against the float64 search (test_gpu_sugar_sample._check_rows), |T| against the float64 prefix; 'boundary' selects
    only the two rows around the last block boundary (for P = 1,048,577 that is also k_rs_scan's chunk boundary)."""
    if how == "boundary" and P <= 1024:
        pytest.skip("one block: no boundary")
    points, scaling, quats, strengths = TS._scene(P, seed=P % 97)
    opacity = how == "masked" and P > 1  # _scene gives the last row strength 0
    st = strengths.reshape(P).contiguous() if opacity else None
    mask = None
    if how == "masked":
        mask = TS._mask(P, seed=P % 89)
    elif how == "boundary":
        b = ((P - 1) // 1024) * 1024
        mask = torch.zeros(P, dtype=torch.bool, device=DEV)
        mask[b - 1: b + 1] = True
    N, seed = 100_000, P % 101
    u, z = SR.draws(N, DEV, seed)
    x, idx, tot, T = _forward(N, 1.5, True, mask, st, u, z, points, scaling, quats)
    w = SR.weights(scaling, st, mask, True)
    Tref = SR.prefix(w, mask)
    total = Tref[-1]
    assert bool(((T.abs() - Tref).abs() <= 1e-12 * total).all())
    c = w.double().cumsum(0)
    t = c if mask is None else torch.where(mask, c, torch.zeros_like(c))
    assert torch.equal(T > 0, t > 0)
    ref_rows, _ = SR.select_rows(Tref, u)
    TS._check_rows(idx, ref_rows, Tref, u)
    _same_bits(x, SR.place(points, scaling, quats, idx, z, 1.5))
    if how == "boundary":
        assert set(idx.unique().tolist()) == {b - 1, b}


@pytest.mark.parametrize("P,row", [(1, 0), (3000, 1500), (1_048_577, 1_048_576)])
def test_single_positive_row(P, row):
    """One selected row: every sample takes it, and all N gradient contributions land on its address (float64 autograd)."""
    from autovfx_b200.sugar_field import sample_points_in_gaussians
    points, scaling, quats, strengths = TS._scene(P, seed=6, zero_volume=False)
    mask = torch.zeros(P, dtype=torch.bool, device=DEV)
    mask[row] = True
    leaves = [t.clone().requires_grad_(True) for t in (points, scaling, quats)]
    N, f = 50_000, 1.5
    torch.manual_seed(71)
    x, idx = sample_points_in_gaussians(SR.Getters(*leaves, strengths), N, f, mask=mask)
    assert bool((idx == row).all())
    _, z = SR.draws(N, DEV, 71)
    _same_bits(x.detach(), SR.place(points, scaling, quats, idx, z, f))
    gr = torch.randn(N, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    (x * gr).sum().backward()
    l64 = [t.detach().double().requires_grad_(True) for t in (points, scaling, quats)]
    (SR.place_pytorch3d(*l64, idx, z.double(), f) * gr.double()).sum().backward()
    bound, hits = TS._row_bound(l64[1].detach(), l64[2].detach(), z, gr, idx, f, P)
    assert int(hits[row]) == N
    for a, b in zip(leaves, l64):
        err = (a.grad.double() - b.grad).abs().amax(-1)
        assert bool((err <= bound).all()), (err / bound).max().item()
        assert not bool(a.grad[torch.arange(P, device=DEV) != row].any())
