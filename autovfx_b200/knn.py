"""``distCUDA2`` — drop-in for ``simple_knn._C.distCUDA2`` (reference KNN/spatial.cu:15-26, KNN/ext.cpp:15-17) — and
``knn_points``, a drop-in for ``pytorch3d.ops.knn_points`` as SuGaR calls it (one cloud pair, 3-D, K <= 32)."""
from __future__ import annotations

from collections import namedtuple

import torch

from . import _lib
from ._lib import lib as _L

KNN_MAX_K = 32

# pytorch3d.ops.knn's return type: dists [N,P1,K] squared, idx [N,P1,K] int64, knn [N,P1,K,D] or None
KNN = namedtuple("KNN", "dists idx knn")


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """Mean squared distance of every point to its 3 nearest neighbours; [P,3] CUDA fp32 -> [P] fp32."""
    if not points.is_cuda:
        raise RuntimeError("autovfx_b200.distCUDA2: points must be a CUDA tensor (there is no CPU path)")
    device = points.device
    with torch.cuda.device(device):
        pts = points.to(torch.float32).contiguous()
        P = pts.size(0)
        means = torch.zeros((P,), dtype=torch.float32, device=device)  # torch::full({P}, 0.0), spatial.cu:21
        if P == 0:
            return means
        nbytes = _L.gsr_dist2_bytes(P)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        rc = _L.gsr_dist2(P, pts.data_ptr(), means.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr(device))
        _lib.check(rc, "gsr_dist2")
    return means


def _search(q: torch.Tensor, p: torch.Tensor, K: int, same: bool):
    """gsr_knn on [P1,3] queries and [P2,3] points (contiguous fp32, no grad) -> dists [P1,K], idx [P1,K] int64."""
    device = p.device
    P1, P2 = q.size(0), p.size(0)
    dists = torch.empty((P1, K), dtype=torch.float32, device=device)
    idx = torch.empty((P1, K), dtype=torch.int64, device=device)
    if P1 == 0:
        return dists, idx
    nbytes = _L.gsr_knn_bytes(0 if same else P1, P2, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
    rc = _L.gsr_knn(P1, P2, K, None if same else q.data_ptr(), p.data_ptr(), dists.data_ptr(), idx.data_ptr(), ws.data_ptr(), nbytes,
                    _lib.stream_ptr(device))
    _lib.check(rc, "gsr_knn")
    return dists, idx


class _KnnPoints(torch.autograd.Function):
    """The search runs detached; dists = |p1_i - p2_idx|^2 carries pytorch3d's analytic backward."""

    @staticmethod
    def forward(ctx, p1, p2, K, same):
        q, p = p1[0].detach().contiguous(), p2[0].detach().contiguous()
        dists, idx = _search(q, p, K, same)
        ctx.save_for_backward(p1, p2, idx)
        ctx.mark_non_differentiable(idx)
        return dists[None], idx[None]

    @staticmethod
    def backward(ctx, g, _gidx):
        p1, p2, idx = ctx.saved_tensors
        terms = 2.0 * g[0][..., None] * (p1[0][:, None, :] - p2[0][idx])  # [P1,K,3]
        g1 = terms.sum(dim=1)[None] if ctx.needs_input_grad[0] else None
        g2 = None
        if ctx.needs_input_grad[1]:
            g2 = torch.zeros_like(p2[0]).index_add_(0, idx.reshape(-1), terms.reshape(-1, 3), alpha=-1.0)[None]
        return g1, g2, None, None


def _check_cloud(name: str, t) -> None:
    if not isinstance(t, torch.Tensor):
        raise ValueError("knn_points: %s must be a torch.Tensor" % name)
    if t.dim() != 3:
        raise ValueError("knn_points: %s must be [N, P, 3], got shape %s" % (name, tuple(t.shape)))
    if t.size(0) != 1:
        raise ValueError("knn_points: %s has N = %d; only N = 1 is supported" % (name, t.size(0)))
    if t.size(2) != 3:
        raise ValueError("knn_points: %s has D = %d; only D = 3 is supported" % (name, t.size(2)))
    if t.dtype != torch.float32:
        raise ValueError("knn_points: %s must be float32, got %s" % (name, t.dtype))


def knn_points(p1: torch.Tensor, p2: torch.Tensor, lengths1=None, lengths2=None, norm: int = 2, K: int = 1, version: int = -1,
               return_nn: bool = False, return_sorted: bool = True) -> KNN:
    """pytorch3d.ops.knn_points for N = 1, D = 3, float32 CUDA tensors, norm = 2 and 1 <= K <= min(32, P2).

    Returns KNN(dists [1,P1,K] squared distances, ascending; idx [1,P1,K] int64 into p2; knn = p2[0][idx] [1,P1,K,3] with
    return_nn, else None).  The search is exact: d = (dx*dx + dy*dy) + dz*dz in float32, each operation rounded once, ties to
    the lower index, the query itself not excluded when p1 is p2.  ``version`` is ignored and the output is always sorted.
    Anything else raises ValueError naming the argument; K > P2, which pytorch3d pads with zeros, is not supported.  CPU tensors
    raise RuntimeError (there is no CPU path).  With grad enabled, dists are differentiable with respect to p1 and p2 as in
    pytorch3d (dL/dp1_i = sum_k 2 g_ik (p1_i - p2_idx), dL/dp2 the negated scatter of the same terms).
    """
    _check_cloud("p1", p1)
    _check_cloud("p2", p2)
    if lengths1 is not None:
        raise ValueError("knn_points: lengths1 is not supported (one cloud per batch: pass None)")
    if lengths2 is not None:
        raise ValueError("knn_points: lengths2 is not supported (one cloud per batch: pass None)")
    if norm != 2:
        raise ValueError("knn_points: norm = %r is not supported (only 2, squared L2)" % (norm,))
    P2 = p2.size(1)
    if isinstance(K, bool) or not isinstance(K, int) or not 1 <= K <= min(KNN_MAX_K, P2):
        raise ValueError("knn_points: K = %r must be an int in 1..min(%d, P2 = %d) (padding for K > P2 is not reproduced)"
                         % (K, KNN_MAX_K, P2))
    if not (p1.is_cuda and p2.is_cuda):
        raise RuntimeError("autovfx_b200.knn_points: p1 and p2 must be CUDA tensors (there is no CPU path)")
    if p1.device != p2.device:
        raise ValueError("knn_points: p2 is on %s, p1 on %s" % (p2.device, p1.device))
    # SuGaR's knn_points(points[None], points[None]): the queries are the points, which the search seeds from their own order
    same = p1.data_ptr() == p2.data_ptr() and p1.shape == p2.shape and p1.stride() == p2.stride()
    with torch.cuda.device(p1.device):
        if torch.is_grad_enabled() and (p1.requires_grad or p2.requires_grad):
            dists, idx = _KnnPoints.apply(p1, p2, K, same)
        else:
            d, i = _search(p1[0].detach().contiguous(), p2[0].detach().contiguous(), K, same)
            dists, idx = d[None], i[None]
        knn = p2[0][idx[0]][None] if return_nn else None
    return KNN(dists, idx, knn)
