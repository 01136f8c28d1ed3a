"""``distCUDA2`` — drop-in for ``simple_knn._C.distCUDA2`` (reference KNN/spatial.cu:15-26, KNN/ext.cpp:15-17)."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib as _L


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
