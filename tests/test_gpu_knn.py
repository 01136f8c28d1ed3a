"""GPU tests of knn_points / gsr_knn (run with -m gpu on an H100).  Distances are compared bit for bit and indices exactly
against the float32 brute-force restatement (tests/knn_ref.py) run on the same GPU; the full-size case is also checked
against a float64 k-d tree."""
import numpy as np
import pytest
import torch

from tests import knn_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import knn  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


def _knn(q, p, K, **kw):
    from autovfx_b200.knn import knn_points
    return knn_points(q[None], p[None], K=K, **kw)


def _assert_exact(dists, idx, want_d, want_i, what=""):
    assert dists.dtype == torch.float32 and idx.dtype == torch.int64
    assert dists.shape == want_d.shape and idx.shape == want_i.shape, (dists.shape, want_d.shape)
    bad_d = dists.view(torch.int32) != want_d.view(torch.int32)
    bad_i = idx != want_i
    rows = (bad_d | bad_i).any(dim=1).nonzero().flatten()
    assert len(rows) == 0, "%s: %d rows differ, e.g. row %d: %s %s vs %s %s" % (
        what, len(rows), int(rows[0]), dists[rows[0]].tolist(), idx[rows[0]].tolist(), want_d[rows[0]].tolist(), want_i[rows[0]].tolist())


def _check_self(p, K, what=""):
    r = _knn(p, p, K)
    wd, wi = knn_ref.knn_brute(p, p, K)
    _assert_exact(r.dists[0], r.idx[0], wd, wi, what)
    return r


def _check_general(q, p, K, what=""):
    r = _knn(q, p, K)
    wd, wi = knn_ref.knn_brute(q, p, K)
    _assert_exact(r.dists[0], r.idx[0], wd, wi, what)
    return r


@pytest.fixture(scope="module")
def uniform60k(dev):
    p = (torch.rand(60_000, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1).to(dev)
    return p, knn_ref.knn_brute(p, p, 32)


@pytest.mark.parametrize("K", [1, 2, 3, 4, 8, 15, 16, 17, 31, 32])
def test_self_mode_every_capacity(uniform60k, K):
    """Each register capacity (4, 8, 16, 32) at and below its size."""
    p, (wd, wi) = uniform60k
    r = _knn(p, p, K)
    _assert_exact(r.dists[0], r.idx[0], wd[:, :K].contiguous(), wi[:, :K].contiguous(), "K=%d" % K)
    assert (r.idx[0, :, 0] == torch.arange(len(p), device=p.device)).all()  # distinct points: self first, at 0


@pytest.mark.parametrize("K", [1, 5, 16, 32])
def test_general_queries_inside_on_and_far_outside(dev, K):
    gen = torch.Generator().manual_seed(2)
    p = torch.rand(50_000, 3, generator=gen) * 2 - 1
    inside = torch.rand(40_000, 3, generator=gen) * 2 - 1
    on = p[torch.randint(0, 50_000, (30_000,), generator=gen)] + torch.randn(30_000, 3, generator=gen) * 1e-3 * (torch.rand(30_000, 1, generator=gen) < 0.5)
    far = torch.randn(10_000, 3, generator=gen) * 40  # mostly outside the points' box: the all-boxes fall-back
    q = torch.cat([inside, on, far])[torch.randperm(80_000, generator=gen)]
    _check_general(q.to(dev), p.to(dev), K, "general K=%d" % K)


def test_coincident_copies_take_the_lowest_indices(dev):
    gen = torch.Generator().manual_seed(5)
    pts = torch.cat([torch.tensor([[0.3, -0.2, 0.1]]).expand(5000, 3), torch.randn(3000, 3, generator=gen) * 0.5])
    pts = pts[torch.randperm(len(pts), generator=gen)].contiguous().to(dev)
    r = _check_self(pts, 16, "coincident")
    copies = (pts == torch.tensor([0.3, -0.2, 0.1], device=dev)).all(dim=1).nonzero().flatten()
    assert len(copies) == 5000
    assert (r.idx[0][copies] == copies[:16][None]).all() and (r.dists[0][copies] == 0).all()


def test_densify_style_duplicate_pairs(dev):
    """SuGaR's clone densification appends exact copies of selected points: every copy ties with its original at 0."""
    gen = torch.Generator().manual_seed(6)
    p = torch.rand(30_000, 3, generator=gen) * 2 - 1
    sel = torch.rand(30_000, generator=gen) < 0.3
    pts = torch.cat([p, p[sel]]).to(dev)
    r = _check_self(pts, 8, "duplicates")
    _check_general(p[:5000].to(dev), pts, 8, "duplicates general")
    n = len(p)
    orig = sel.nonzero().flatten().to(dev)
    copy = torch.arange(n, n + len(orig), device=dev)
    assert (r.idx[0][copy, 0] == orig).all() and (r.idx[0][copy, 1] == copy).all() and (r.dists[0][copy, :2] == 0).all()


def test_planar_cloud(dev):
    """z == 0 everywhere: the box has no extent along z (the Morton code divides 0 by 0 there)."""
    xy = torch.rand(20_000, 2, generator=torch.Generator().manual_seed(7)) * 4 - 2
    pts = torch.cat([xy, torch.zeros(20_000, 1)], dim=1).to(dev)
    _check_self(pts, 16, "planar")
    q = torch.cat([xy[:3000] + 0.01, torch.rand(3000, 1) - 0.5], dim=1).to(dev)
    _check_general(q, pts, 16, "planar general")


def test_candidate_list_overflow_both_modes(dev):
    """1.2M uniform points and far outliers: CTAs holding an outlier list more boxes than fit and test every box.  The rows
    checked are every outlier and a random sample, against a brute force over all 1.2M points."""
    from autovfx_b200.knn import knn_points
    gen = torch.Generator().manual_seed(8)
    pts = torch.rand(1_200_000, 3, generator=gen) * 2 - 1
    out = torch.arange(0, 1_200_000, 240_000)
    pts[out] = torch.tensor([[40.0, 35.0, -30.0], [-45.0, 30.0, 38.0], [33.0, -41.0, 44.0], [-39.0, -37.0, -36.0], [50.0, 0.0, 0.0]])
    pts = pts.to(dev)
    rows = torch.cat([out, torch.randint(0, 1_200_000, (8192,), generator=gen)]).to(dev)
    r = knn_points(pts[None], pts[None], K=16)
    wd, wi = knn_ref.knn_brute(pts[rows], pts, 16)
    _assert_exact(r.dists[0][rows], r.idx[0][rows], wd, wi, "overflow self")
    q = torch.cat([torch.rand(200_000, 3, generator=gen) * 2 - 1, torch.randn(2000, 3, generator=gen) * 60]).to(dev)
    r = knn_points(q[None], pts[None], K=16)
    qrows = torch.cat([torch.arange(200_000, 202_000), torch.randint(0, 200_000, (4096,), generator=gen)]).to(dev)
    wd, wi = knn_ref.knn_brute(q[qrows], pts, 16)
    _assert_exact(r.dists[0][qrows], r.idx[0][qrows], wd, wi, "overflow general")


@pytest.mark.parametrize("K", [1, 16, 32])
def test_small_sizes(dev, K):
    gen = torch.Generator().manual_seed(9 + K)
    for P2 in (K, K + 1):
        p = (torch.randn(P2, 3, generator=gen)).to(dev)
        _check_self(p, K, "P2=%d K=%d" % (P2, K))
        _check_general(torch.randn(700, 3, generator=gen).to(dev), p, K, "general P2=%d K=%d" % (P2, K))
    r = _knn(torch.empty(0, 3, device=dev), torch.randn(50, 3, generator=gen).to(dev), K, return_nn=True)
    assert r.dists.shape == r.idx.shape == (1, 0, K) and r.knn.shape == (1, 0, K, 3)


def test_one_to_five_points(dev):
    gen = torch.Generator().manual_seed(10)
    for P in range(1, 6):
        p = torch.randn(P, 3, generator=gen).to(dev)
        for K in sorted({1, P}):
            _check_self(p, K, "P=%d K=%d" % (P, K))
            _check_general(torch.randn(3, 3, generator=gen).to(dev), p, K, "general P=%d K=%d" % (P, K))


def test_full_size_config3_k16(dev):
    """config-3's 3M positions, self mode, K = 16: 65,536 sampled rows exactly against a brute force over all 3M points,
    and their distances against a float64 k-d tree."""
    from scipy.spatial import cKDTree
    from autovfx_b200 import scene
    pts_cpu = scene.config3_scene()["means3D"]
    pts = pts_cpu.to(dev)
    r = _knn(pts, pts, 16)
    rows = torch.randperm(len(pts), generator=torch.Generator().manual_seed(11))[:65_536]
    wd, wi = knn_ref.knn_brute(pts[rows.to(dev)], pts, 16)
    got_d, got_i = r.dists[0][rows.to(dev)], r.idx[0][rows.to(dev)]
    _assert_exact(got_d, got_i, wd, wi, "config3")
    p64 = pts_cpu.double().numpy()
    dd, _ = cKDTree(p64).query(p64[rows.numpy()], k=16)
    np.testing.assert_allclose(got_d.double().cpu().numpy(), dd * dd, rtol=1e-6, atol=1e-14)


def test_deterministic_and_permutation_equivariant(dev):
    gen = torch.Generator().manual_seed(12)
    p = (torch.rand(100_000, 3, generator=gen) * 2 - 1).to(dev)
    q = (torch.rand(70_000, 3, generator=gen) * 2.2 - 1.1).to(dev)
    a, b = _knn(q, p, 16), _knn(q, p, 16)
    assert torch.equal(a.dists.view(torch.int32), b.dists.view(torch.int32)) and torch.equal(a.idx, b.idx)
    a, b = _knn(p, p, 16), _knn(p, p, 16)
    assert torch.equal(a.dists.view(torch.int32), b.dists.view(torch.int32)) and torch.equal(a.idx, b.idx)
    perm = torch.randperm(len(q), generator=gen).to(dev)
    c = _knn(q[perm], p, 16)
    r = _knn(q, p, 16)
    assert torch.equal(c.dists[0].view(torch.int32), r.dists[0][perm].view(torch.int32)) and torch.equal(c.idx[0], r.idx[0][perm])
    # self mode (the same storage) and a copy of the points as queries find the same neighbours
    s, g = _knn(p, p, 16), _knn(p.clone(), p, 16)
    assert torch.equal(s.dists.view(torch.int32), g.dists.view(torch.int32)) and torch.equal(s.idx, g.idx)


def test_pytorch3d_return_contract(dev):
    from autovfx_b200.knn import knn_points
    gen = torch.Generator().manual_seed(13)
    p1 = torch.randn(1, 900, 3, generator=gen).to(dev)
    p2 = torch.randn(1, 1200, 3, generator=gen).to(dev)
    res = knn_points(p1, p2, K=6)
    dists, idx, nn = res
    assert nn is None and res.knn is None and res.dists is dists and res.idx is idx
    assert dists.shape == (1, 900, 6) and dists.dtype == torch.float32 and dists.device == p1.device
    assert idx.shape == (1, 900, 6) and idx.dtype == torch.int64
    res = knn_points(p1, p2, K=6, return_nn=True, return_sorted=False, version=0)
    assert res.knn.shape == (1, 900, 6, 3) and torch.equal(res.knn[0], p2[0][res.idx[0]])
    assert torch.equal(res.dists, dists) and torch.equal(res.idx, idx)
    assert torch.all(dists[..., 1:] >= dists[..., :-1])
    q_strided = torch.randn(1, 900, 6, generator=gen).to(dev)[..., ::2]  # non-contiguous input
    _assert_exact(knn_points(q_strided, p2, K=6).dists[0], knn_points(q_strided, p2, K=6).idx[0],
                  *knn_ref.knn_brute(q_strided[0], p2[0], 6), "strided")


def test_sugar_call_patterns(dev):
    """sugar_model.py:233 (K = 16 under no_grad on an nn.Parameter) and :47 (K = 4, dists[..., 1:] skips the point itself)."""
    from autovfx_b200.knn import knn_points
    gen = torch.Generator().manual_seed(14)
    points = torch.nn.Parameter((torch.rand(40_000, 3, generator=gen) * 2 - 1).to(dev))
    with torch.no_grad():
        knn_idx = knn_points(points[None], points[None], K=16).idx[0]
    wd, wi = knn_ref.knn_brute(points.detach(), points.detach(), 16)
    assert torch.equal(knn_idx, wi)
    dists = knn_points(points[None], points[None], K=4).dists
    assert (dists[..., 0] == 0).all()
    radii = dists[..., 1:].mean(dim=-1)  # SuGaR's initial radii
    assert torch.equal(dists[0].view(torch.int32), wd[:, :4].contiguous().view(torch.int32))
    assert radii.shape == (1, 40_000) and (radii > 0).all()


def test_gradients_against_fp64_autograd(dev):
    from autovfx_b200.knn import knn_points
    gen = torch.Generator().manual_seed(15)
    p1 = torch.randn(1, 300, 3, generator=gen).to(dev).requires_grad_(True)
    p2 = torch.randn(1, 500, 3, generator=gen).to(dev).requires_grad_(True)
    w = torch.randn(1, 300, 8, generator=gen).to(dev)
    res = knn_points(p1, p2, K=8)
    (res.dists * w).sum().backward()
    a = p1.detach().double().requires_grad_(True)
    b = p2.detach().double().requires_grad_(True)
    d64 = ((a[0][:, None, :] - b[0][res.idx[0]]) ** 2).sum(-1)
    (d64 * w[0].double()).sum().backward()
    torch.testing.assert_close(p1.grad.double(), a.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(p2.grad.double(), b.grad, rtol=1e-5, atol=1e-6)
    # self mode: both gradients reach the same leaf
    p = torch.randn(400, 3, generator=gen).to(dev).requires_grad_(True)
    res = knn_points(p[None], p[None], K=5)
    assert res.dists.requires_grad and not res.idx.requires_grad
    (res.dists[0] * w[0, :, :5].repeat(2, 1)[:400]).sum().backward()
    c = p.detach().double().requires_grad_(True)
    d64 = ((c[:, None, :] - c[res.idx[0]]) ** 2).sum(-1)
    (d64 * w[0, :, :5].repeat(2, 1)[:400].double()).sum().backward()
    torch.testing.assert_close(p.grad.double(), c.grad, rtol=1e-5, atol=1e-6)
    # without grad mode the dists carry no graph
    with torch.no_grad():
        assert not knn_points(p1, p2, K=8).dists.requires_grad
