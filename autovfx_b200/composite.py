"""Frame compositing of the edited video in CUDA ("BA/" = blender/blend_all.py): ``composite_frame`` is the per-frame body of
``blend_frames`` (BA/:185-342) on device tensors, and ``blend_frames`` is a drop-in for the reference's function.

``composite_frame`` runs ``gsr_percentile_low`` (the smoke depth's ``np.percentile(x, 0.001)``, BA/:208) and ``gsr_composite`` (one
pass per output pixel, BA/:236-342) on the current stream; the result is bit-identical to the reference on the same decoded arrays
and nothing synchronises with the host.  Every layer must have the frame's size: the reference's Blender scripts render at that
size, where BA/:21-28 ``downsample_image`` is Pillow's identity.

Opt in with ``blend_all.blend_frames = composite.blend_frames`` (INTEGRATION.md, "Frame compositing").
"""
from __future__ import annotations

import glob
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor
from typing import Optional

import numpy as np
import torch

from . import _lib

__all__ = ["composite_frame", "percentile_low", "blend_frames"]

PERCENTILE_BYTES = 2048  # GSR_PERCENTILE_BYTES


def _check(who, name, t, dtype, shape):
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s: %s must be a tensor, got %s" % (who, name, type(t).__name__))
    if t.dtype != dtype:
        raise ValueError("%s: %s must be %s, got %s" % (who, name, dtype, t.dtype))
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s: %s has shape %s, the frame needs %s" % (who, name, tuple(t.shape), tuple(shape)))
    if not t.is_contiguous() or (dtype == torch.uint8 and t.data_ptr() % 4):
        raise ValueError("%s: %s must be contiguous (and 4-byte aligned)" % (who, name))


def percentile_low(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``np.percentile(x, 0.001)`` of a float32 CUDA tensor as a 0-dim float32 CUDA tensor (numpy's 'linear' method in float32, as
    NumPy >= 2 computes it; NaN when any element is NaN; the sign of a zero result may differ).  No host synchronisation."""
    if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or x.numel() == 0 or not x.is_contiguous():
        raise ValueError("percentile_low: x must be a non-empty contiguous float32 tensor")
    if not x.is_cuda:
        raise RuntimeError("autovfx_b200.percentile_low: x must be a CUDA tensor, got one on %s (there is no CPU path)" % x.device)
    out = torch.empty((), dtype=torch.float32, device=x.device) if out is None else out
    ws = torch.empty(PERCENTILE_BYTES, dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib.gsr_percentile_low(x.numel(), x.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(x.device)),
                   "gsr_percentile_low")
    return out


def composite_frame(rgba8, depth, obj, obj_depth, shadow, shadow_depth, all_, obj3dgs=None, obj3dgs_depth=None, smoke=None,
                    smoke_depth=None, fire=None, out=None) -> torch.Tensor:
    """The frame of blend_frames (BA/:185-342) from decoded layers, as a uint8 [H,W,4] CUDA tensor.

    ``rgba8`` [H,W,4] uint8 is the 3DGS frame (``images/*.png`` or ``FrameLoop(pack8=True)``'s ``rgba8``) and ``depth`` [H,W]
    float32 its depth, or None: the reference loads it (BA/:186) and never reads it, so it is only validated.  ``obj``, ``shadow``,
    ``all_`` (rgb_obj, rgb_shadow, rgb_all) are [H,W,4] uint8 and ``obj_depth``, ``shadow_depth`` (depth_obj, depth_shadow) [H,W]
    float32.  Optional: ``obj3dgs`` + ``obj3dgs_depth`` (rgb_obj_3dgs, depth_obj_3dgs), ``smoke`` + ``smoke_depth``
    (rgb_smoke_fire, depth_smoke_fire) and ``fire`` (rgb_smoke_fire_pre, which needs smoke; the reference fails at BA/:265 without
    it).  depth_all and depth_smoke_fire_pre never affect the frame and are not arguments.

    Wrong dtypes, shapes or sizes, mixed devices, a colour layer without its depth (or the reverse) and fire without smoke raise
    ValueError naming the argument; CPU tensors raise RuntimeError.  Runs on the current stream without host synchronisation."""
    who = "composite_frame"
    if not isinstance(rgba8, torch.Tensor) or rgba8.dim() != 3 or rgba8.shape[2] != 4:
        raise ValueError("%s: rgba8 must be a [H,W,4] tensor, got %s" % (who, tuple(rgba8.shape) if isinstance(rgba8, torch.Tensor) else type(rgba8).__name__))
    H, W = int(rgba8.shape[0]), int(rgba8.shape[1])
    if H == 0 or W == 0:
        raise ValueError("%s: rgba8 is empty (shape %s)" % (who, tuple(rgba8.shape)))
    c4, d2 = (H, W, 4), (H, W)
    for a, b, va, vb in (("obj3dgs", "obj3dgs_depth", obj3dgs, obj3dgs_depth), ("smoke", "smoke_depth", smoke, smoke_depth)):
        if (va is None) != (vb is None):
            raise ValueError("%s: %s given without %s" % (who, a if vb is None else b, b if vb is None else a))
    if fire is not None and smoke is None:
        raise ValueError("%s: fire (rgb_smoke_fire_pre) needs smoke and smoke_depth" % who)
    args = [("rgba8", rgba8, torch.uint8, c4), ("depth", depth, torch.float32, d2), ("obj", obj, torch.uint8, c4),
            ("obj_depth", obj_depth, torch.float32, d2), ("shadow", shadow, torch.uint8, c4), ("shadow_depth", shadow_depth, torch.float32, d2),
            ("all_", all_, torch.uint8, c4), ("obj3dgs", obj3dgs, torch.uint8, c4), ("obj3dgs_depth", obj3dgs_depth, torch.float32, d2),
            ("smoke", smoke, torch.uint8, c4), ("smoke_depth", smoke_depth, torch.float32, d2), ("fire", fire, torch.uint8, c4),
            ("out", out, torch.uint8, c4)]
    given = [(n, t) for n, t, dt, sh in args if t is not None]
    for n, t, dt, sh in args:
        if t is not None:
            _check(who, n, t, dt, sh)
    dev = rgba8.device
    for n, t in given:
        if t.device != dev:
            raise ValueError("%s: %s is on %s, rgba8 on %s" % (who, n, t.device, dev))
    if not rgba8.is_cuda:
        raise RuntimeError("autovfx_b200.%s: rgba8 must be a CUDA tensor, got one on %s (there is no CPU path)" % (who, dev))
    if out is None:
        out = torch.empty(c4, dtype=torch.uint8, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    with torch.cuda.device(dev):
        stream = _lib.stream_ptr(dev)
        pct = None
        if smoke is not None:
            pct = torch.empty((), dtype=torch.float32, device=dev)
            percentile_low(smoke_depth, out=pct)
        _lib.check(_lib.lib.gsr_composite(W, H, rgba8.data_ptr(), obj.data_ptr(), obj_depth.data_ptr(), shadow.data_ptr(), shadow_depth.data_ptr(),
                                          all_.data_ptr(), ptr(obj3dgs), ptr(obj3dgs_depth), ptr(smoke), ptr(smoke_depth), ptr(pct), ptr(fire),
                                          out.data_ptr(), stream), "gsr_composite")
    return out


# ------------------------------------------------------------------------------------------------------------ the drop-in
def _host_module():
    """The module whose ``blend_frames`` is this function (``blend_all.blend_frames = composite.blend_frames``): its loaders and
    its ``generate_video_from_frames`` are the reference's own."""
    for m in list(sys.modules.values()):
        if getattr(m, "blend_frames", None) is blend_frames and hasattr(m, "generate_video_from_frames") and hasattr(m, "load_rgb"):
            return m
    raise RuntimeError("composite.blend_frames: install it with `blend_all.blend_frames = composite.blend_frames`")


def _layer_paths(cache, i):
    """BA/:170-182 for frame i (1-based names), without depth_all and depth_smoke_fire_pre, which never affect the frame."""
    d = lambda name: os.path.join(cache, name, "{:0>3d}".format(i + 1), "Image{:0>4d}.exr".format(i + 1))  # noqa: E731
    c = lambda name: os.path.join(cache, name, "{:0>3d}.png".format(i + 1))  # noqa: E731
    return {"obj": c("rgb_obj"), "obj_depth": d("depth_obj"), "shadow": c("rgb_shadow"), "shadow_depth": d("depth_shadow"),
            "all_": c("rgb_all"), "obj3dgs": c("rgb_obj_3dgs"), "obj3dgs_depth": d("depth_obj_3dgs"), "smoke": c("rgb_smoke_fire"),
            "smoke_depth": d("depth_smoke_fire"), "fire": c("rgb_smoke_fire_pre")}


def blend_frames(blend_results_dir, input_config_path=None, png_writer=None):
    """Drop-in for BA/:92-348 ``blend_frames``: the same globbing and frame count (BA/:117-132), the module's own loaders
    (``load_rgb``, ``load_depth_exr``), ``composite_frame`` per frame on the current CUDA device, the same ``frames/NNNN.png`` files,
    and the module's ``generate_video_from_frames`` for ``blended.mp4``.  Frame i+1 is decoded on host threads while frame i
    composites, and the PNGs are written on host threads: by PIL by default, or, with ``png_writer`` (a ``png.PngWriter``), encoded
    on the device (same pixels, different bytes); the writer is flushed before the video is made."""
    ba = _host_module()
    root_dir = os.path.dirname(os.path.normpath(os.path.dirname(os.path.normpath(blend_results_dir))))
    input_config = None
    if input_config_path is not None:
        with open(input_config_path, 'r') as f:
            input_config = json.load(f)
    assert input_config is not None, 'input_config is required for blending frames'
    cache = os.path.join(input_config['blender_cache_dir'], input_config['output_dir_name'])
    bg_rgb = sorted(glob.glob(os.path.join(root_dir, 'images', '*.png')))
    n_frame = len(glob.glob(os.path.join(cache, 'rgb_all', '*.png')))
    out_img_dir = os.path.join(blend_results_dir, 'frames')
    os.makedirs(out_img_dir, exist_ok=True)
    dev = torch.device("cuda", torch.cuda.current_device())

    def decode(pool, i):
        paths = _layer_paths(cache, i)
        futs = {"rgba8": pool.submit(ba.load_rgb, bg_rgb[i])}
        for k, p in paths.items():
            futs[k] = pool.submit(ba.load_depth_exr if k.endswith("_depth") else ba.load_rgb, p)
        return futs

    def upload(a):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)

    frames = []
    with ThreadPoolExecutor(max_workers=12) as pool, ThreadPoolExecutor(max_workers=2) as writers:
        pending = decode(pool, 0) if n_frame else None
        saves = []
        for i in range(n_frame):
            arrays = {k: f.result() for k, f in pending.items()}
            if arrays["fire"] is not None and arrays["smoke"] is None:
                raise ValueError("blend_frames: frame %d has rgb_smoke_fire_pre without rgb_smoke_fire" % i)
            pending = decode(pool, i + 1) if i + 1 < n_frame else None
            layers = {k: upload(v) for k, v in arrays.items()}
            if layers["obj3dgs"] is None:
                layers["obj3dgs_depth"] = None
            if layers["smoke"] is None:
                layers["smoke_depth"] = None
            frame_dev = composite_frame(layers.pop("rgba8"), None, **layers)
            path = os.path.join(out_img_dir, '{:0>4d}.png'.format(i))
            if png_writer is not None:
                png_writer.submit(path, frame_dev)
            frame = frame_dev.cpu().numpy()
            frames.append(frame)
            if png_writer is None:
                saves.append(writers.submit(_save_png, frame, path))
        for s in saves:
            s.result()
        if png_writer is not None:
            png_writer.flush()
    ba.generate_video_from_frames(np.array(frames), os.path.join(blend_results_dir, 'blended.mp4'), fps=15)


def _save_png(frame, path):
    from PIL import Image
    Image.fromarray(frame).save(path)
