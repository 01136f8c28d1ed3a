"""CPU tests of knn_points' host side and of its float32 oracle (tests/knn_ref.py): the restatement against a float64 k-d
tree, its tie rule, the argument checks (no device is touched) and the C-ABI size query and validation."""
import numpy as np
import pytest
import torch

from tests import knn_ref


def test_restatement_matches_kdtree_within_float32_rounding():
    from scipy.spatial import cKDTree
    gen = torch.Generator().manual_seed(11)
    p = torch.rand(2000, 3, generator=gen) * 2 - 1
    q = torch.cat([p[:500], torch.randn(700, 3, generator=gen) * 1.5])
    K = 16
    d, i = knn_ref.knn_brute(q, p, K)
    assert d.dtype == torch.float32 and i.dtype == torch.int64 and d.shape == i.shape == (1200, K)
    assert torch.all(d[:, 1:] >= d[:, :-1])
    dd, ii = cKDTree(p.double().numpy()).query(q.double().numpy(), k=K)
    want = dd * dd
    np.testing.assert_allclose(d.double().numpy(), want, rtol=1e-6, atol=1e-12)
    # the float32 distance of the returned index is the restatement's own: the indices are a set of true nearest up to rounding
    again = knn_ref.pinned_d2(q, p).gather(1, i)
    assert torch.equal(again, d)
    assert (i[:500, 0] == torch.arange(500)).all()  # self at distance 0 for the queries that are points


def test_restatement_resolves_ties_to_the_lowest_index():
    base = torch.tensor([[0.0, 0.0, 0.0]])
    # four points at distance exactly 1 (one per axis direction), two coincident copies at distance 0.25^2, one far point
    p = torch.tensor([[5.0, 5.0, 5.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.25, 0.0, 0.0], [0.0, 0.0, -1.0], [0.25, 0.0, 0.0],
                      [-1.0, 0.0, 0.0]])
    d, i = knn_ref.knn_brute(base, p, 5)
    assert i[0].tolist() == [3, 5, 1, 2, 4]
    assert d[0].tolist() == [0.0625, 0.0625, 1.0, 1.0, 1.0]
    # many copies: the K lowest-index copies win, in index order
    p = torch.zeros(40, 3)
    d, i = knn_ref.knn_brute(p[:3], p, 16)
    assert (i == torch.arange(16)).all() and (d == 0).all()


def test_pinned_distance_rounds_each_op_once():
    """(dx*dx + dy*dy) + dz*dz in float32, never the float64 value rounded once."""
    q = torch.tensor([[0.1, 0.2, 0.3]])
    p = torch.tensor([[0.7, -0.4, 1.3]])
    dx, dy, dz = (np.float32(a) - np.float32(b) for a, b in zip(p[0].numpy(), q[0].numpy()))
    want = np.float32(np.float32(np.float32(dx * dx) + np.float32(dy * dy)) + np.float32(dz * dz))
    assert knn_ref.pinned_d2(q, p).item() == want


def _cloud(P=8):
    return torch.rand(1, P, 3)


@pytest.mark.parametrize("kwargs, match", [
    (dict(p1=torch.rand(8, 3)), "p1"),
    (dict(p2=torch.rand(8, 3)), "p2"),
    (dict(p1=torch.rand(2, 8, 3)), "p1 has N = 2"),
    (dict(p2=torch.rand(2, 8, 3)), "p2 has N = 2"),
    (dict(p1=torch.rand(1, 8, 2)), "p1 has D = 2"),
    (dict(p2=torch.rand(1, 8, 4)), "p2 has D = 4"),
    (dict(p1=torch.rand(1, 8, 3, dtype=torch.float64)), "p1 must be float32"),
    (dict(p2=torch.rand(1, 8, 3).half()), "p2 must be float32"),
    (dict(p1=[[0.0, 0.0, 0.0]]), "p1 must be a torch.Tensor"),
    (dict(lengths1=torch.tensor([8])), "lengths1"),
    (dict(lengths2=torch.tensor([8])), "lengths2"),
    (dict(norm=1), "norm"),
    (dict(K=0), "K = 0"),
    (dict(K=33, p2=torch.rand(1, 40, 3)), "K = 33"),
    (dict(K=9), "K = 9"),  # K > P2 = 8: pytorch3d pads, this does not
    (dict(K=2.0), "K = 2.0"),
    (dict(K=True), "K = True"),
])
def test_unsupported_arguments_raise_value_error(kwargs, match):
    from autovfx_b200.knn import knn_points
    args = dict(p1=_cloud(), p2=_cloud(), K=4)
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        knn_points(**args)


def test_cpu_tensors_raise_runtime_error():
    from autovfx_b200.knn import knn_points
    with pytest.raises(RuntimeError, match="CUDA"):
        knn_points(_cloud(), _cloud(), K=4)
    p = _cloud()
    with pytest.raises(RuntimeError, match="CUDA"):
        knn_points(p, p, K=1, return_nn=True)


def test_knn_workspace_size_and_argument_validation():
    import ctypes as C
    from autovfx_b200._lib import lib
    # the points' Morton layout (as distCUDA2's) plus, for a second query cloud, the queries' own
    assert lib.gsr_knn_bytes(0, 100000, 16) == lib.gsr_dist2_bytes(100000) + lib.gsr_dist2_bytes(0) < 100000 * 40
    assert lib.gsr_knn_bytes(50000, 100000, 16) == lib.gsr_dist2_bytes(100000) + lib.gsr_dist2_bytes(50000)
    assert lib.gsr_knn_bytes(3_000_000, 3_000_000, 32) < 3_000_000 * 2 * 40
    assert lib.gsr_knn_bytes(-5, -5, 1) == 2 * lib.gsr_dist2_bytes(0)
    fake = C.c_void_p(256)  # never dereferenced: every call below fails validation before any launch
    for P1, P2, K, q, msg in [(-1, 10, 1, fake, b"negative"), (10, -1, 1, fake, b"negative"), (10, 10, 0, None, b"K = 0"),
                              (10, 40, 33, fake, b"K = 33"), (10, 4, 5, fake, b"K = 5 > P2"), (10, 12, 4, None, b"P1 == P2")]:
        assert lib.gsr_knn(P1, P2, K, q, fake, fake, fake, fake, 1 << 30, None) == -1
        assert msg in lib.gsr_last_error()
    assert lib.gsr_knn(0, 10, 4, fake, fake, None, None, None, 0, None) == 0  # P1 = 0 launches nothing
    assert lib.gsr_knn(10, 10, 4, None, None, fake, fake, fake, 1 << 30, None) == -1
    assert b"null" in lib.gsr_last_error()
    assert lib.gsr_knn(10, 10, 4, None, fake, fake, fake, fake, 16, None) == -2
    assert b"workspace" in lib.gsr_last_error()
