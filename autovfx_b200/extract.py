"""Scoring of extract_object's candidate Gaussian subsets on the GPU (extract/extract_object.py:168-224, :287-343).

For every ratio the reference deep-copies the model, boolean-indexes it, calls the full ``render()`` for every tracked view and
counts ``(alpha >= 0.8) XOR (mask == 255)`` in numpy on the host.  Here, with the masks packed once per object::

    scorer = MaskScorer(gaussians, camera_views, obj_masks, pipe)   # once per object
    total_missed_pixels = int(scorer.count(mask3d))                 # replaces :195-221 and :314-340

``count`` compacts the subset's rows in one pass (gsr_select_rows), reads back the row count, and issues one exact-mode forward
per tracked view (``colors_precomp`` zero, so no SH is read), each followed by gsr_mask_disagreement on the alpha plane, without
a host synchronisation per frame.  Exact mode gives the reference CUDA's alpha bit for bit (the default blend is only within
1e-5, which could move a pixel across the threshold), so the count equals the reference loop's.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from . import rasterizer as R
from ._lib import lib as _L
from .renderer import _setup

__all__ = ["MaskScorer", "ALPHA_THRESHOLD", "tracked_views"]

# `object_alpha_image >= 0.8` on a float32 array: numpy (NEP 50) compares in float32, so the threshold is float32(0.8)
ALPHA_THRESHOLD = np.float32(0.8)


def tracked_views(camera_views: Sequence, obj_masks: Dict[str, object]) -> List[Tuple[int, object, object]]:
    """(idx, view, mask) of every view the reference loop scores: view ``idx`` counts only if ``"{idx:05d}.png"`` is a key of
    ``obj_masks`` (:208-212)."""
    return [(idx, view, obj_masks["{0:05d}.png".format(idx)]) for idx, view in enumerate(camera_views)
            if "{0:05d}.png".format(idx) in obj_masks]


def _mask_u8(mask, idx: int, H: int, W: int) -> torch.Tensor:
    name = "obj_masks[%r]" % "{0:05d}.png".format(idx)
    t = mask if isinstance(mask, torch.Tensor) else torch.from_numpy(np.asarray(mask))
    if t.dtype != torch.uint8:
        raise ValueError("%s must be uint8 (a grayscale tracking mask), not %s" % (name, t.dtype))
    if tuple(t.shape) != (H, W):
        raise ValueError("%s has shape %s, but view %d renders (H, W) = (%d, %d)" % (name, tuple(t.shape), idx, H, W))
    return t


class MaskScorer:
    """The masked-pixel count of extract_object's ratio search for one object.

    ``gaussians``: the scene's model; ``get_xyz``, ``get_opacity``, ``get_scaling`` and ``get_rotation`` are read once (the
    activations render() uses; they act per element or per row, so selecting rows afterwards gives the bits the cropped copy
    would).  ``camera_views``: the cameras render() takes (FoVx, FoVy, image_height, image_width, world_view_transform,
    full_proj_transform, camera_center).  ``obj_masks``: file name -> uint8 [H,W] tracking mask.  ``pipe``: render()'s pipeline
    settings, or None; ``pipe.compute_cov3D_python`` is refused (its torch covariance changes the image bits).

    ValueError names the argument at fault; CPU tensors raise RuntimeError."""

    def __init__(self, gaussians, camera_views: Sequence, obj_masks: Dict[str, object], pipe=None):
        if pipe is not None and getattr(pipe, "compute_cov3D_python", False):
            raise ValueError("pipe.compute_cov3D_python: the torch covariance changes the image bits; MaskScorer renders from scales "
                             "and rotations")
        views = tracked_views(camera_views, obj_masks)
        sizes = [(int(v.image_height), int(v.image_width)) for _, v, _ in views]
        masks = [_mask_u8(m, idx, H, W) for (idx, _, m), (H, W) in zip(views, sizes)]
        xyz = gaussians.get_xyz
        if not xyz.is_cuda:
            raise RuntimeError("autovfx_b200.extract: gaussians must live on a CUDA device (there is no CPU path)")
        device = self.device = xyz.device
        P = self.P = int(xyz.shape[0])
        self.idx = [idx for idx, _, _ in views]
        rows = [xyz, gaussians.get_opacity, gaussians.get_scaling, gaussians.get_rotation]
        for name, t, w in zip(("get_xyz", "get_opacity", "get_scaling", "get_rotation"), rows, (3, 1, 3, 4)):
            if tuple(t.shape) != (P, w):
                raise ValueError("gaussians.%s has shape %s, expected (%d, %d)" % (name, tuple(t.shape), P, w))
            if t.device != device:
                raise ValueError("gaussians.%s is on %s, get_xyz on %s" % (name, t.device, device))
        f32 = dict(dtype=torch.float32, device=device)
        with torch.no_grad(), torch.cuda.device(device):
            self.rows = [t.detach().to(torch.float32).contiguous() for t in rows]
            self.sel = [torch.empty((P, w), **f32) for w in (3, 1, 3, 4)]  # the subset's rows, first P_sel of them valid
            self.colors = torch.zeros((P, 3), **f32)
            self.sel_ws = torch.empty(max(int(_L.gsr_select_rows_bytes(P)), 4), dtype=torch.uint8, device=device)
            self.sel_count = torch.zeros((), dtype=torch.int32, device=device)
            V = len(views)
            self.counts = torch.zeros((V,), dtype=torch.int64, device=device)
            bg = torch.zeros(3, **f32)
            HW = max([H * W for H, W in sizes], default=1)
            frame = torch.empty((5 * HW,), **f32)  # colour | depth | alpha of the frame in flight
            radii = torch.empty((P,), dtype=torch.int32, device=device)
            self.cams = torch.empty((V, 35), **f32)
            self.bits, self.frames, self.tan, self.alpha = [], [], [], []
            stream = _lib.stream_ptr(device)
            for v, ((_, view, _), (H, W), mask) in enumerate(zip(views, sizes, masks)):
                # the camera fields render() reads, through render()'s own settings (an empty xyz: no screen-space leaf is needed)
                _, s = _setup(view, xyz[:0], 0, pipe if pipe is not None else _NO_PIPE, bg, 1.0)
                self.cams[v] = torch.cat([R._dev_f32(s.viewmatrix, device).reshape(16), R._dev_f32(s.projmatrix, device).reshape(16),
                                          R._dev_f32(s.campos, device).reshape(3)])
                self.tan.append((float(s.tanfovx), float(s.tanfovy)))
                bits = torch.empty((H, (W + 31) // 32), dtype=torch.int32, device=device)
                m = mask.to(device).contiguous()
                _lib.check(_L.gsr_pack_masks(1, W, H, m.data_ptr(), bits.data_ptr(), stream), "gsr_pack_masks")
                self.bits.append(bits)
                out = (frame[:3 * H * W].view(3, H, W), frame[3 * H * W:4 * H * W].view(1, H, W), frame[4 * H * W:5 * H * W].view(1, H, W), radii)
                self.alpha.append(out[2])
                self.frames.append(R.PreparedForward(self.sel[0], None, self.sel[1], self.sel[2], self.sel[3], self.cams[v], W, H, bg, 0, 1.0,
                                                     out, exact=True, colors_precomp=self.colors))
            self.sizes = sizes
            self._keep = (frame, radii)
        self.rerendered = 0  # views rendered again after a binning overflow

    @property
    def num_views(self) -> int:
        """The tracked views: those with a mask."""
        return len(self.frames)

    def count(self, selection) -> torch.Tensor:
        """Total masked-pixel disagreement of the subset ``selection`` (bool [P], numpy or tensor) over the tracked views: the
        reference's ``total_missed_pixels``, as a 0-dim int64 tensor on the scene's device."""
        keep = selection if isinstance(selection, torch.Tensor) else torch.from_numpy(np.asarray(selection))
        if keep.dtype != torch.bool or tuple(keep.shape) != (self.P,):
            raise ValueError("selection must be a bool mask of shape (%d,), got %s %s" % (self.P, keep.dtype, tuple(keep.shape)))
        dev = self.device
        with torch.no_grad(), torch.cuda.device(dev):
            keep = keep.to(dev).contiguous()
            stream = _lib.stream_ptr(dev)
            p = R._ptr
            _lib.check(_L.gsr_select_rows(self.P, p(keep), *(p(t) for t in self.rows), *(p(t) for t in self.sel), self.sel_count.data_ptr(),
                                          self.sel_ws.data_ptr(), self.sel_ws.numel(), stream), "gsr_select_rows")
            n = int(self.sel_count.item())  # the frames need the subset's size on the host
            self.counts.zero_()
            tickets = [self._frame(v, n, stream) for v in range(self.num_views)]
            for v, t in enumerate(tickets):
                if t.ok():
                    continue
                # binning overflow (ok() grew the capacity): render the view again until it fits, then count it afresh
                while not self.frames[v].launch(*self.tan[v], P=n).ok():
                    pass
                self.rerendered += 1
                self.counts[v].zero_()
                self._score(v, stream)
            return self.counts.sum()

    def _frame(self, v: int, n: int, stream) -> R.FrameTicket:
        ticket = self.frames[v].launch(*self.tan[v], P=n)
        self._score(v, stream)
        return ticket

    def _score(self, v: int, stream) -> None:
        H, W = self.sizes[v]
        _lib.check(_L.gsr_mask_disagreement(W, H, self.alpha[v].data_ptr(), self.bits[v].data_ptr(), float(ALPHA_THRESHOLD),
                                            self.counts[v:].data_ptr(), stream), "gsr_mask_disagreement")


class _NoPipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


_NO_PIPE = _NoPipe()
