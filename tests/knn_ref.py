"""Float32 brute-force restatement of gsr_knn / knn_points, the oracle of tests/test_knn_cpu.py and tests/test_gpu_knn.py.

The distance is the pinned one, d = (dx*dx + dy*dy) + dz*dz with dx = p.x - q.x, as separate float32 torch ops (each rounded
once, never fused), and ranking is on the int64 key (float bits << 32) | index: for d >= 0 the float bits order like the
values, so ties go to the lower index.  Runs on any device: on the GPU it reproduces the kernel bit for bit.
"""
from __future__ import annotations

import torch


def pinned_d2(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """[Q,3] x [P,3] float32 -> [Q,P] squared distances with the kernel's rounding sequence."""
    dx = p[None, :, 0] - q[:, None, 0]
    dy = p[None, :, 1] - q[:, None, 1]
    dz = p[None, :, 2] - q[:, None, 2]
    return (dx * dx + dy * dy) + dz * dz


def knn_brute(q: torch.Tensor, p: torch.Tensor, K: int):
    """Exact K nearest of p for every row of q: (dists [Q,K] float32, idx [Q,K] int64), ascending by (distance, index)."""
    q, p = q.float(), p.float()
    chunk = max(1, (1 << 27) // max(1, p.size(0)))  # about 1 GiB of int64 keys per chunk
    idx_all = torch.arange(p.size(0), dtype=torch.int64, device=p.device)
    ds, ix = [], []
    for s in range(0, q.size(0), chunk):
        d = pinned_d2(q[s:s + chunk], p)
        key = (d.view(torch.int32).to(torch.int64) << 32) | idx_all[None]
        del d
        best = torch.topk(key, K, dim=1, largest=False, sorted=True).values
        del key
        ix.append(best & 0xFFFFFFFF)
        ds.append((best >> 32).to(torch.int32).view(torch.float32))
    if not ds:
        return torch.empty((0, K), dtype=torch.float32, device=p.device), torch.empty((0, K), dtype=torch.int64, device=p.device)
    return torch.cat(ds), torch.cat(ix)
