"""PNG files encoded on the GPU (``gsr_png_encode``): the frame loop's image, depth-colormap and normal-map files
(scene_representation.py:424-438) and blend_frames' composited frames, without a host-side encoder.

The files are standard 8-bit PNGs (grey, RGB or RGBA, not interlaced) and decode to exactly the pixels PIL's or OpenCV's files hold
for the same image; their bytes are this encoder's own and are not byte-identical to PIL's, libpng's or zlib's output.  The bytes
depend only on the pixels and the shape.

- ``encode_png`` / ``encode_pngs``: the files in device or pinned host buffers, with their sizes in an int64 tensor.
- ``save_image`` and ``imwrite``: synchronous drop-ins for ``torchvision.utils.save_image`` (one [C,H,W] image) and
  ``cv2.imwrite`` on ``.png`` paths.
- ``PngWriter``: asynchronous: ``submit`` enqueues the encode on the current stream into a ring of pinned buffers and host threads
  write each file once its event has completed; the submitting thread never synchronises with the device.
- ``FrameFiles``: a ``consume`` callback for ``FrameLoop(pack8=True, to_host=False)`` writing the reference loop's file set.
"""
from __future__ import annotations

import ctypes as C
import os
import queue
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

__all__ = ["png_bound", "encode_png", "encode_pngs", "save_image", "imwrite", "PngWriter", "FrameFiles", "turbo_lut_rgb"]

_ALIGN = 256


def png_bound(H: int, W: int, C: int) -> int:
    """The largest file ``gsr_png_encode`` writes for an H x W image with C channels in the file (3 for a lookup-table image)."""
    n = _lib.lib.gsr_png_bound(int(H), int(W), int(C))
    if n == 0:
        raise ValueError("png_bound: no PNG of shape (%d, %d, %d)" % (H, W, C))
    return int(n)


def _image(img: torch.Tensor, lut: Optional[torch.Tensor] = None, swap_rb: bool = False, who: str = "encode_png"):
    """The C description of one image: uint8 [H,W] or [H,W,C] (C in 1, 3, 4) on a CUDA device, any strides."""
    if not isinstance(img, torch.Tensor):
        raise ValueError("%s: the image must be a tensor, got %s" % (who, type(img).__name__))
    if img.dtype != torch.uint8:
        raise ValueError("%s: the image must be uint8, got %s" % (who, img.dtype))
    if img.dim() not in (2, 3):
        raise ValueError("%s: the image must be [H,W] or [H,W,C], got shape %s" % (who, tuple(img.shape)))
    H, W = int(img.shape[0]), int(img.shape[1])
    Cn = int(img.shape[2]) if img.dim() == 3 else 1
    if Cn not in (1, 3, 4):
        raise ValueError("%s: the image has %d channels (1, 3 or 4)" % (who, Cn))
    if H == 0 or W == 0:
        raise ValueError("%s: the image is empty (shape %s)" % (who, tuple(img.shape)))
    if not img.is_cuda:
        raise RuntimeError("autovfx_b200.%s: the image must be a CUDA tensor, got one on %s (there is no CPU path)" % (who, img.device))
    if lut is not None:
        if Cn != 1:
            raise ValueError("%s: a lookup table needs a 1-channel image, got %d channels" % (who, Cn))
        if not isinstance(lut, torch.Tensor) or lut.dtype != torch.uint8 or tuple(lut.shape) != (256, 3) or not lut.is_contiguous():
            raise ValueError("%s: lut must be a contiguous uint8 [256,3] tensor" % who)
        if lut.device != img.device:
            raise ValueError("%s: lut is on %s, the image on %s" % (who, lut.device, img.device))
    st = img.stride()
    d = _lib.gsr_png_image()
    d.data, d.stride_h, d.stride_w = img.data_ptr(), st[0], st[1]
    d.stride_c = st[2] if img.dim() == 3 else 1
    d.H, d.W, d.C = H, W, Cn
    d.flags = _lib.GSR_PNG_SWAP_RB if (swap_rb and Cn >= 3) else 0
    d.lut = lut.data_ptr() if lut is not None else None
    return d, (3 if lut is not None else Cn)


def _align(n: int) -> int:
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


def _encode_into(descs: List[_lib.gsr_png_image], outputs: List[int], sizes_ptr: int, device: torch.device) -> None:
    n = len(descs)
    arr = (_lib.gsr_png_image * n)(*descs)
    nbytes = int(_lib.lib.gsr_png_workspace_bytes(n, arr))
    with torch.cuda.device(device):
        ws = _lib.scratch_bytes(nbytes, device)
        outs = (C.c_void_p * n)(*outputs)
        _lib.check(_lib.lib.gsr_png_encode(arr, n, outs, sizes_ptr, ws.data_ptr(), nbytes, _lib.stream_ptr(device)), "gsr_png_encode")


def encode_pngs(items: Sequence, pinned: bool = False) -> Tuple[torch.Tensor, List[Tuple[int, int]], torch.Tensor]:
    """Encode a list of images in one call on the current stream.  Each item is an image tensor or ``(image, lut)`` or
    ``(image, lut, swap_rb)``.  Returns ``(buffer, spans, sizes)``: one uint8 buffer (device, or pinned host when ``pinned``) holding
    file i at ``spans[i] = (offset, capacity)``, and an int64 tensor (same memory kind) of the file sizes.  Nothing synchronises with
    the host; read the sizes after the stream has finished."""
    if len(items) == 0:
        raise ValueError("encode_pngs: no images")
    descs, spans, refs = [], [], []
    off = 0
    dev = None
    for it in items:
        img, lut, swap = (it, None, False) if isinstance(it, torch.Tensor) else (tuple(it) + (None, False))[:3]
        d, cf = _image(img, lut, bool(swap), "encode_pngs")
        if dev is not None and img.device != dev:
            raise ValueError("encode_pngs: images on %s and %s" % (dev, img.device))
        dev = img.device
        cap = png_bound(d.H, d.W, cf)
        descs.append(d)
        spans.append((off, cap))
        refs.append(img)
        off += _align(cap)
    if pinned:
        buf = torch.empty(off, dtype=torch.uint8, pin_memory=True)
        sizes = torch.zeros(len(items), dtype=torch.int64, pin_memory=True)
    else:
        buf = torch.empty(off, dtype=torch.uint8, device=dev)
        sizes = torch.empty(len(items), dtype=torch.int64, device=dev)
    _encode_into(descs, [buf.data_ptr() + o for o, _ in spans], sizes.data_ptr(), dev)
    return buf, spans, sizes


def encode_png(img: torch.Tensor, lut: Optional[torch.Tensor] = None, swap_rb: bool = False, pinned: bool = False
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """One PNG file: ``(buffer, size)`` with the file in ``buffer[:size]`` (a 0-dim int64 tensor), on the image's device or, with
    ``pinned``, in pinned host memory.  ``img`` is uint8 [H,W] (grey), [H,W,3] (RGB) or [H,W,4] (RGBA) on a CUDA device, any strides;
    ``swap_rb`` reads BGR / BGRA; ``lut`` (uint8 [256,3] RGB) turns a [H,W] index image into an RGB file.  Runs on the current stream
    without host synchronisation."""
    buf, _, sizes = encode_pngs([(img, lut, swap_rb)], pinned=pinned)
    return buf, sizes[0]


def _file_bytes(img, lut=None, swap_rb=False) -> bytes:
    buf, _, sizes = encode_pngs([(img, lut, swap_rb)], pinned=True)
    torch.cuda.current_stream(img.device).synchronize()
    return buf.numpy()[: int(sizes[0])].tobytes()


def _write(fp, data: bytes) -> None:
    if hasattr(fp, "write"):
        fp.write(data)
    else:
        with open(fp, "wb") as f:
            f.write(data)


def save_image(tensor: torch.Tensor, fp, format: Optional[str] = None, **kwargs) -> None:
    """Drop-in for ``torchvision.utils.save_image(tensor, fp)`` as the frame loop calls it: one float [C,H,W] image (C = 1, 3 or 4)
    on a CUDA device, rounded as torchvision does (``mul(255).add_(0.5).clamp_(0, 255)``, then uint8), 1 channel written as RGB
    (``make_grid``'s rule for one image).  Any ``make_grid`` argument, or a format other than PNG, raises ValueError."""
    if kwargs:
        raise ValueError("save_image: make_grid arguments are not supported (%s)" % ", ".join(sorted(kwargs)))
    if format is not None and format.lower() != "png":
        raise ValueError("save_image: only PNG is written, got format %r" % format)
    if not isinstance(tensor, torch.Tensor) or tensor.dim() != 3:
        raise ValueError("save_image: one [C,H,W] image is supported, got %s" % (tuple(tensor.shape) if isinstance(tensor, torch.Tensor) else type(tensor).__name__))
    if not tensor.is_floating_point():
        raise ValueError("save_image: the image must be floating point, got %s" % tensor.dtype)
    if tensor.shape[0] not in (1, 3, 4):
        raise ValueError("save_image: the image has %d channels (1, 3 or 4)" % tensor.shape[0])
    if not tensor.is_cuda:
        raise RuntimeError("autovfx_b200.save_image: the image must be a CUDA tensor, got one on %s (there is no CPU path)" % tensor.device)
    with torch.no_grad():
        t = tensor.detach()
        if t.shape[0] == 1:
            t = torch.cat((t, t, t), 0)
        u8 = t.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)
    _write(fp, _file_bytes(u8))


def _as_device_u8(img, who: str) -> torch.Tensor:
    if isinstance(img, np.ndarray):
        if img.dtype != np.uint8:
            raise ValueError("%s: the image must be uint8, got %s" % (who, img.dtype))
        img = torch.from_numpy(np.ascontiguousarray(img)).to(torch.device("cuda", torch.cuda.current_device()))
    if isinstance(img, torch.Tensor) and img.dim() == 3 and img.shape[2] == 1:
        img = img[:, :, 0]
    return img


def imwrite(path, img, params=None) -> bool:
    """Drop-in for ``cv2.imwrite(path, img)`` on ``.png`` paths: uint8 [H,W] grey, [H,W,3] BGR or [H,W,4] BGRA, as a CUDA tensor or a
    numpy array (uploaded to the current device).  The file holds the pixels cv2's file holds.  Returns True."""
    if params:
        raise ValueError("imwrite: encoder parameters are not supported")
    if not str(path).lower().endswith(".png"):
        raise ValueError("imwrite: only .png paths are written, got %r" % str(path))
    img = _as_device_u8(img, "imwrite")
    _write(path, _file_bytes(img, swap_rb=True))
    return True


_TURBO = {}


def turbo_lut_rgb(device) -> torch.Tensor:
    """``depth2img``'s TURBO colormap as an RGB [256,3] table on ``device``: a depth8 image through it is the colour image
    ``cv2.imwrite`` stores for ``cv2.applyColorMap(depth8, COLORMAP_TURBO)``."""
    device = torch.device(device)
    if device not in _TURBO:
        from .renderer import TURBO_LUT_BGR
        _TURBO[device] = TURBO_LUT_BGR.flip(1).contiguous().to(device)
    return _TURBO[device]


# ------------------------------------------------------------------------------------------------------------ the async writer
class _Slot:
    def __init__(self):
        self.buf: Optional[torch.Tensor] = None
        self.sizes: Optional[torch.Tensor] = None
        self.host: Dict[int, torch.Tensor] = {}  # pinned copies of .npy arrays, by item index


class PngWriter:
    """Asynchronous PNG (and ``.npy``) files from device images.

    ``submit(path, image, lut=None, swap_rb=False)`` (or ``submit_many``) enqueues the encode on the current stream into one of
    ``ring`` pinned host buffers and returns; ``threads`` host threads wait for each submission's event and write its files.  When
    every buffer is in flight, ``submit`` waits for a writer thread to free one (a host wait, not a device synchronisation).
    ``flush()`` waits for every file and re-raises the first I/O error as RuntimeError; ``close()`` flushes and stops the threads.
    The images may be reused by work queued later on the same stream."""

    def __init__(self, ring: int = 4, threads: int = 2):
        if ring < 1 or threads < 1:
            raise ValueError("PngWriter: ring and threads must be >= 1")
        self._slots = [_Slot() for _ in range(ring)]
        self._free: "queue.Queue[int]" = queue.Queue()
        for i in range(ring):
            self._free.put(i)
        self._jobs: "queue.Queue" = queue.Queue()
        self._errors: List[BaseException] = []
        self._lock = threading.Lock()
        self._threads = [threading.Thread(target=self._run, daemon=True) for _ in range(threads)]
        self._closed = False
        for t in self._threads:
            t.start()

    def submit(self, path, image: torch.Tensor, lut: Optional[torch.Tensor] = None, swap_rb: bool = False) -> None:
        self.submit_many([(path, image, lut, swap_rb)])

    def submit_many(self, pngs: Sequence, arrays: Sequence = ()) -> None:
        """One encode for several files: ``pngs`` holds ``(path, image[, lut[, swap_rb]])`` and ``arrays`` ``(path, tensor)`` pairs
        saved with ``np.save`` after a copy to pinned memory on the current stream."""
        if self._closed:
            raise RuntimeError("PngWriter: closed")
        if not pngs and not arrays:
            return
        descs, spans, refs, dev = [], [], [], None
        off = 0
        for it in pngs:
            path, img = it[0], it[1]
            lut = it[2] if len(it) > 2 else None
            swap = bool(it[3]) if len(it) > 3 else False
            d, cf = _image(img, lut, swap, "PngWriter.submit")
            if dev is not None and img.device != dev:
                raise ValueError("PngWriter.submit: images on %s and %s" % (dev, img.device))
            dev = img.device
            cap = png_bound(d.H, d.W, cf)
            descs.append(d)
            spans.append((str(path), off, cap))
            refs.append(img)
            off += _align(cap)
        for path, t in arrays:
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise RuntimeError("autovfx_b200.PngWriter: arrays must be CUDA tensors")
        slot_id = self._free.get()
        slot = self._slots[slot_id]
        try:
            if descs:
                if slot.buf is None or slot.buf.numel() < off:
                    slot.buf = torch.empty(off, dtype=torch.uint8, pin_memory=True)
                if slot.sizes is None or slot.sizes.numel() < len(descs):
                    slot.sizes = torch.zeros(len(descs), dtype=torch.int64, pin_memory=True)
                _encode_into(descs, [slot.buf.data_ptr() + o for _, o, _ in spans], slot.sizes.data_ptr(), dev)
            npys = []
            for k, (path, t) in enumerate(arrays):
                h = slot.host.get(k)
                if h is None or h.shape != t.shape or h.dtype != t.dtype:
                    h = slot.host[k] = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                h.copy_(t, non_blocking=True)
                npys.append((str(path), h))
                dev = t.device
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
        except BaseException:
            self._free.put(slot_id)
            raise
        self._jobs.put((slot_id, ev, spans, npys, refs))

    def _run(self):
        while True:
            job = self._jobs.get()
            if job is None:
                self._jobs.task_done()
                return
            slot_id, ev, spans, npys, refs = job
            try:
                ev.synchronize()
                slot = self._slots[slot_id]
                if spans:
                    host = slot.buf.numpy()
                    sizes = slot.sizes.numpy()
                    for i, (path, off, _) in enumerate(spans):
                        try:
                            with open(path, "wb") as f:
                                f.write(host[off: off + int(sizes[i])])
                        except OSError as ex:
                            with self._lock:
                                self._errors.append(ex)
                for path, h in npys:
                    try:
                        np.save(path, h.numpy())
                    except OSError as ex:
                        with self._lock:
                            self._errors.append(ex)
            except BaseException as ex:  # noqa: BLE001
                with self._lock:
                    self._errors.append(ex)
            finally:
                del refs
                self._free.put(slot_id)
                self._jobs.task_done()

    def flush(self) -> None:
        """Wait until every submitted file is written; raise the first error since the last flush as RuntimeError."""
        self._jobs.join()
        with self._lock:
            errs, self._errors = self._errors, []
        if errs:
            raise RuntimeError("PngWriter: %d file(s) failed, first: %s" % (len(errs), errs[0])) from errs[0]

    def close(self) -> None:
        if self._closed:
            return
        try:
            self.flush()
        finally:
            self._closed = True
            for _ in self._threads:
                self._jobs.put(None)
            for t in self._threads:
                t.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class FrameFiles:
    """``consume`` callback for ``FrameLoop(..., pack8=True, to_host=False)`` (with or without ``product=True``): the reference loop's
    files (scene_representation.py:424-438) under the same names, ``images/NAME.png`` (RGBA), ``depth/NAME.npy`` (``np.save`` of
    the float32 depth), ``depth/NAME.png`` (``depth2img``'s TURBO colormap) and, with ``product=True``, ``normal/NAME.png``.
    ``names[i]`` is frame i's ``view.image_name`` (default ``%05d``).  The three PNGs of a frame are one encode on the current stream,
    queued before the loop can reuse the frame's ring slot (FrameLoop with one stream).  ``flush()`` / ``close()`` as PngWriter."""

    def __init__(self, out_dir: str, names: Optional[Sequence[str]] = None, writer: Optional[PngWriter] = None):
        self.out_dir, self.names = out_dir, names
        self.writer = writer if writer is not None else PngWriter()
        self._own = writer is None
        for sub in ("images", "depth"):
            os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
        self._normal_dir = False

    def __call__(self, i: int, frame: Dict[str, torch.Tensor], stats=None) -> None:
        for k in ("rgba8", "depth", "depth8"):
            if k not in frame:
                raise ValueError("FrameFiles: the frame has no %r (FrameLoop needs pack8=True)" % k)
        if not frame["rgba8"].is_cuda:
            raise ValueError("FrameFiles: the frame is in host memory; run FrameLoop with to_host=False")
        name = self.names[i] if self.names is not None else "%05d" % i
        o = self.out_dir
        pngs = [(os.path.join(o, "images", name + ".png"), frame["rgba8"]),
                (os.path.join(o, "depth", name + ".png"), frame["depth8"], turbo_lut_rgb(frame["depth8"].device))]
        if "normal8" in frame:
            if not self._normal_dir:
                os.makedirs(os.path.join(o, "normal"), exist_ok=True)
                self._normal_dir = True
            pngs.append((os.path.join(o, "normal", name + ".png"), frame["normal8"]))
        self.writer.submit_many(pngs, arrays=[(os.path.join(o, "depth", name + ".npy"), frame["depth"])])

    consume = __call__

    def flush(self) -> None:
        self.writer.flush()

    def close(self) -> None:
        if self._own:
            self.writer.close()
        else:
            self.writer.flush()
