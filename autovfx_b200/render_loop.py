"""Per-frame render loop and its multi-GPU sharding.

Replaces the reference's frame loops (``scene_representation.py:355-438`` render_from_3DGS, ``sugar/gaussian_splatting/
render.py:53-64`` render_set, ``sugar/render.py:109-139``): those call the rasterizer once per camera from Python, block on
a device->host copy inside every forward (rasterizer_impl.cu:281-282) and then copy / encode four images per frame
synchronously.  ``FrameLoop`` keeps the Gaussian parameters resident, issues every frame without a host synchronisation
(``forward_raw(sync=False)``), renders straight into a ring of ``[5,H,W]`` device frames (rgb | depth | alpha), streams
finished frames to pinned host memory on a copy stream that overlaps the next frame's kernels, and validates each
frame's device-side counters before handing it to the consumer (a frame whose binning buffer overflowed is re-rendered).

Multi-GPU (SURVEY §8e): frames are independent given the parameters, so ranks shard the camera list; the only
collectives are the one-time parameter broadcast, the camera scatter and the gather of per-frame statistics.  The
rendered frames stay on the rank that produced them (the reference writes them to disk per frame anyway).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import torch

from .scene import Camera

CAM_FLOATS = 37  # view(16) | proj(16) | campos(3) | tanfovx | tanfovy


# ----------------------------------------------------------------------------- host placement
def bind_to_gpu_numa_node(index: int) -> str:
    """Pin the calling process to the CPUs NVML reports as closest to GPU ``index`` so that pinned host buffers (the D2H ring
    of ``FrameLoop``) are first-touched on that NUMA node.  With one process per GPU on an 8-GPU node this decides whether the
    eight frame streams share one socket's memory controllers.  Call it before creating the loop; returns a short description, never raises."""
    try:
        import os
        import pynvml
        pynvml.nvmlInit()
        pynvml.nvmlDeviceSetCpuAffinity(pynvml.nvmlDeviceGetHandleByIndex(index))
        return "cpus=%d" % len(os.sched_getaffinity(0))
    except Exception as ex:  # noqa: BLE001
        return "unchanged (%s)" % type(ex).__name__


# ----------------------------------------------------------------------------- sharding (pure host logic)
def shard_indices(n_frames: int, rank: int, world: int, mode: str = "roundrobin") -> List[int]:
    """Frames owned by ``rank``.  Round-robin balances the slowly varying per-frame cost (R changes smoothly along a
    trajectory); "block" keeps contiguous runs."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    if mode == "roundrobin":
        return list(range(rank, n_frames, world))
    if mode == "block":
        per = (n_frames + world - 1) // world
        return list(range(rank * per, min(n_frames, (rank + 1) * per)))
    raise ValueError("mode must be 'roundrobin' or 'block'")


def pack_cameras(cams: Sequence[Camera]) -> torch.Tensor:
    """[N,37] fp32 host tensor, the per-camera payload of the scatter."""
    if len(cams) == 0:
        return torch.zeros((0, CAM_FLOATS), dtype=torch.float32)
    return torch.stack([c.packed() for c in cams]).contiguous()


def scatter_cameras(packed: Optional[torch.Tensor], n_frames: int, device, mode: str = "roundrobin", group=None) -> torch.Tensor:
    """Rank 0 holds ``packed`` [N,37]; every rank receives the rows of its own frames via one ``dist.scatter`` (padded to
    equal length; NCCL on GPUs, gloo in the CPU tests).  Single-process: just moves the tensor."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return packed.to(device)
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    per = (n_frames + world - 1) // world
    recv = torch.zeros((per, CAM_FLOATS), dtype=torch.float32, device=device)
    chunks = None
    if rank == 0:
        chunks = []
        for r in range(world):
            idx = shard_indices(n_frames, r, world, mode)
            c = torch.zeros((per, CAM_FLOATS), dtype=torch.float32)
            if idx:
                c[:len(idx)] = packed[idx]
            chunks.append(c.to(device))
    dist.scatter(recv, chunks, src=0, group=group)
    return recv[:len(shard_indices(n_frames, rank, world, mode))]


def broadcast_gaussians(g: Optional[Dict[str, torch.Tensor]], device, group=None) -> Dict[str, torch.Tensor]:
    """One-time replication of the parameters from rank 0 (708 MB at 3M Gaussians / M=16)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return {k: v.to(device) for k, v in g.items()}
    rank = dist.get_rank(group)
    keys = ["means3D", "scales", "rotations", "opacities", "shs"]
    # shapes first, as one small tensor on the collective's own path (no pickling, no extra host round trips)
    is_cuda = torch.device(device).type == "cuda"
    meta = torch.zeros((len(keys), 4), dtype=torch.int64, device=device if is_cuda else "cpu")
    if rank == 0:
        for i, k in enumerate(keys):
            shp = tuple(g[k].shape)
            meta[i, 0] = len(shp)
            for j, n in enumerate(shp):
                meta[i, 1 + j] = n
    dist.broadcast(meta, src=0, group=group)
    meta = meta.cpu().tolist()
    out = {}
    for i, k in enumerate(keys):
        shape = tuple(int(n) for n in meta[i][1:1 + int(meta[i][0])])
        t = g[k].to(device).float().contiguous() if rank == 0 else torch.empty(shape, dtype=torch.float32, device=device)
        dist.broadcast(t, src=0, group=group)
        out[k] = t
    return out


def gather_stats(local: torch.Tensor, group=None) -> Optional[List[torch.Tensor]]:
    """Gather a small per-rank statistics tensor on rank 0."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return [local]
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bufs = [torch.zeros_like(local) for _ in range(world)] if rank == 0 else None
    dist.gather(local, bufs, dst=0, group=group)
    return bufs


# ----------------------------------------------------------------------------- the loop
class FrameLoop:
    """Renders a list of cameras for one resident set of Gaussians on one GPU.

    ``product=False``: one rasterizer forward per camera; the finished frame is ``[5,H,W]`` (rgb | depth | alpha).
    ``product=True`` : the reference's whole ``render()`` per camera (gaussian_renderer/__init__.py:83-218): SH image, normal
                       image and the normal / pseudo-normal maps, as gsr_axis_normals -> one 6-channel forward ->
                       gsr_normal_maps; the finished frame is a dict ``{"frame" [5,H,W], "normal" [H,W,3], "pseudo_normal"
                       [H,W,3]}``.
    ``pack8=True``   : hand the frame off as the bytes the reference's loop gives its encoders (scene_representation.py:424-438):
                       ``{"rgba8" [H,W,4], "depth" [H,W] f32, "depth8" [H,W]}`` (+ ``"normal8" [H,W,3]`` with ``product``) —
                       18.7 MB (24.9 MB) instead of 41.5 MB (66 MB) of fp32 over PCIe per 1080p frame.
    """

    def __init__(self, gaussians: Dict[str, torch.Tensor], sh_degree: int, width: int, height: int, bg=(0.0, 0.0, 0.0),
                 scale_modifier: float = 1.0, device=None, ring: int = 3, to_host: bool = True, tight_tiles: Optional[bool] = None,
                 product: bool = False, pack8: bool = False, depth_scale: float = 3.0, streams: int = 1):
        from . import rasterizer as R  # requires the CUDA library
        self._R = R
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.g = {k: v.to(self.device).float().contiguous() for k, v in gaussians.items()}
        self.sh_degree, self.W, self.H, self.scale_modifier = sh_degree, width, height, scale_modifier
        self.bg = torch.tensor(bg, dtype=torch.float32, device=self.device)
        # streams > 1: consecutive frames are issued on different CUDA streams (ring slot s always uses stream s % streams), so the
        # tail of one frame's kernels overlaps the head of the next frame's; the ring is rounded up to a multiple of `streams`.
        # Frames edited per frame through `before_frame` share one set of resident arrays and fall back to a single stream.
        self.nstreams = max(1, int(streams))
        if self.nstreams > 1:
            ring = ((max(ring, self.nstreams) + self.nstreams - 1) // self.nstreams) * self.nstreams
        self.ring = ring
        self.to_host = to_host
        self.tight_tiles = tight_tiles  # None: follow rasterizer.set_tight_tiles()
        self.product, self.pack8, self.depth_scale = product, pack8, depth_scale
        P = self.g["means3D"].shape[0]
        H, W = height, width
        dev = self.device
        self.frames = [torch.empty((5, H, W), dtype=torch.float32, device=dev) for _ in range(ring)]
        self.radii = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(ring)]
        self.outputs: List[Dict[str, torch.Tensor]] = []  # per slot: what a finished frame consists of (device side)
        if product:
            from . import renderer as RD
            self._RD = RD
            # per-Gaussian normal*0.5+0.5 of the frame in flight, one buffer per compute stream
            self.normals_s = [torch.empty((P, 3), dtype=torch.float32, device=dev) for _ in range(self.nstreams)]
            self.normals = self.normals_s[0]
            self.extra = [torch.empty((3, H, W), dtype=torch.float32, device=dev) for _ in range(ring)]
            self.nmaps = [(torch.empty((H, W, 3), dtype=torch.float32, device=dev), torch.empty((H, W, 3), dtype=torch.float32, device=dev))
                          for _ in range(ring)]
        for s in range(ring):
            if not product and not pack8:
                self.outputs.append({"frame": self.frames[s]})
            elif not product:
                self.outputs.append({"rgba8": torch.empty((H, W, 4), dtype=torch.uint8, device=dev), "depth": self.frames[s][3],
                                     "depth8": torch.empty((H, W), dtype=torch.uint8, device=dev)})
            elif not pack8:
                self.outputs.append({"frame": self.frames[s], "normal": self.nmaps[s][0], "pseudo_normal": self.nmaps[s][1]})
            else:
                self.outputs.append({"rgba8": torch.empty((H, W, 4), dtype=torch.uint8, device=dev), "depth": self.frames[s][3],
                                     "depth8": torch.empty((H, W), dtype=torch.uint8, device=dev),
                                     "normal8": torch.empty((H, W, 3), dtype=torch.uint8, device=dev)})
        self.host = [{k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in self.outputs[s].items()} for s in range(ring)] if to_host else None
        self.copy_stream = torch.cuda.Stream(self.device) if to_host else None
        self.compute_streams = [torch.cuda.Stream(self.device) for _ in range(self.nstreams)] if self.nstreams > 1 else None
        # per-frame host->device payload: the 37 camera floats, plus (product mode) the 4x4 inverse of the view matrix that the
        # pseudo-normal needs — inverted on the host in float64 (the reference calls torch.inverse on the GPU every frame)
        self._cam_floats = CAM_FLOATS + (16 if product else 0)
        self.cam_pinned = torch.empty((ring, self._cam_floats), dtype=torch.float32).pin_memory()
        self.cam_dev = torch.empty((ring, self._cam_floats), dtype=torch.float32, device=self.device)
        self.h2d_bytes_per_frame = self._cam_floats * 4
        self.d2h_bytes_per_frame = sum(v.numel() * v.element_size() for v in self.outputs[0].values()) if to_host else 0
        self.rerendered = 0
        self._prep = [None] * ring

    def _prepared(self, slot: int):
        """Per-slot resolved forward (and, in product mode, the resolved argument lists of the surrounding kernels): built on
        first use and whenever the parameter tensors change (``set_gaussians``)."""
        g = self.g
        key = tuple((g[k].data_ptr(), tuple(g[k].shape)) for k in ("means3D", "shs", "opacities", "scales", "rotations"))
        ent = self._prep[slot]
        if ent is not None and ent["key"] == key:
            return ent
        import ctypes as C
        from . import _lib
        R, f, P, cam = self._R, self.frames[slot], g["means3D"].shape[0], self.cam_dev[slot]
        out = (f[0:3], f[3:4], f[4:5], self.radii[slot][:P])
        ent = {"key": key}
        if not self.product:
            ent["fwd"] = R.PreparedForward(g["means3D"], g["shs"], g["opacities"], g["scales"], g["rotations"], cam, self.W, self.H, self.bg,
                                           self.sh_degree, self.scale_modifier, out, tight=self.tight_tiles)
            if self.pack8:
                o = self.outputs[slot]
                ent["pack"] = (self.W, self.H, f[0:3].data_ptr(), f[4].data_ptr(), f[3].data_ptr(), None, float(self.depth_scale),
                               o["rgba8"].data_ptr(), None, o["depth8"].data_ptr())
                ent["L"], ent["check"], ent["C"] = _lib.lib, _lib.check, C
        else:
            normals = self.normals_s[slot % self.nstreams][:P]
            ent["fwd"] = R.PreparedForward(g["means3D"], g["shs"], g["opacities"], g["scales"], g["rotations"], cam, self.W, self.H, self.bg,
                                           self.sh_degree, self.scale_modifier, out, extra=normals, extra_out=self.extra[slot], tight=self.tight_tiles)
            L = _lib.lib
            camp = cam.data_ptr()
            n_out, p_out = self.nmaps[slot]
            ptr = lambda t: t.data_ptr() if t.numel() else None  # noqa: E731
            ent["axis"] = (P, ptr(g["means3D"]), ptr(g["scales"]), ptr(g["rotations"]), camp + 32 * 4, 1, ptr(normals))
            ent["maps"] = (self.W, self.H, self.extra[slot].data_ptr(), f[3].data_ptr(), camp + CAM_FLOATS * 4)
            ent["maps_out"] = (n_out.data_ptr(), p_out.data_ptr())
            if self.pack8:
                o = self.outputs[slot]
                ent["pack"] = (self.W, self.H, f[0:3].data_ptr(), f[4].data_ptr(), f[3].data_ptr(), n_out.data_ptr(), float(self.depth_scale),
                               o["rgba8"].data_ptr(), o["normal8"].data_ptr(), o["depth8"].data_ptr())
            ent["L"], ent["check"], ent["C"] = L, _lib.check, C
        self._prep[slot] = ent
        return ent

    def _issue(self, slot: int, cam_row: torch.Tensor, sync: bool):
        """host camera row -> pinned -> device (H2D inside the frame), then the frame's kernels into ring slot ``slot``.
        Everything is launched through per-slot prepared argument lists: per frame the host only copies the camera, updates two
        scalars and makes the C calls."""
        self.cam_pinned[slot, :CAM_FLOATS].copy_(cam_row)
        if self.product:
            self.cam_pinned[slot, CAM_FLOATS:] = torch.linalg.inv(cam_row[0:16].view(4, 4).double()).float().reshape(16)
        self.cam_dev[slot].copy_(self.cam_pinned[slot], non_blocking=True)
        tfx, tfy = float(cam_row[35]), float(cam_row[36])
        ent = self._prepared(slot)
        fwd = ent["fwd"]
        if not self.product:
            ticket = fwd.launch(tfx, tfy)
            while sync and not ticket.ok():  # ok() waits for the counters and grows the capacity after an overflow
                ticket = fwd.launch(tfx, tfy)
            if self.pack8:
                with torch.cuda.device(self.device):
                    ent["check"](ent["L"].gsr_pack_frame(*ent["pack"], ent["C"].c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                                 "gsr_pack_frame")
            return ticket
        L, check, C = ent["L"], ent["check"], ent["C"]
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        with torch.cuda.device(self.device):
            check(L.gsr_axis_normals(*ent["axis"], stream), "gsr_axis_normals")
            ticket = fwd.launch(tfx, tfy)
            while sync and not ticket.ok():
                ticket = fwd.launch(tfx, tfy)
            W, H, extra_p, depth_p, c2w_p = ent["maps"]
            check(L.gsr_normal_maps(W, H, extra_p, depth_p, c2w_p, self.W / (2 * tfx), self.H / (2 * tfy), self.W / 2, self.H / 2,
                                    ent["maps_out"][0], ent["maps_out"][1], stream), "gsr_normal_maps")
            if self.pack8:
                check(L.gsr_pack_frame(*ent["pack"], stream), "gsr_pack_frame")
        return ticket

    def _copy_out(self, slot: int):
        for k, v in self.outputs[slot].items():
            self.host[slot][k].copy_(v, non_blocking=True)

    def _finished(self, slot: int):
        src = self.host[slot] if self.to_host else self.outputs[slot]
        return src["frame"] if not (self.product or self.pack8) else src

    def set_gaussians(self, gaussians: Dict[str, torch.Tensor]) -> None:
        """Swap the (activated) parameter tensors the next frames read — e.g. the views ``edit.ResidentScene.compose`` returns
        for this frame.  The tensors must live on this loop's device; kernels run in stream order, so frames already issued
        are not affected as long as the caller's edits are issued on the same stream (``compose`` is)."""
        P_old = self.g["means3D"].shape[0]
        self.g = {k: v for k, v in gaussians.items()}
        P = self.g["means3D"].shape[0]
        if P > self.radii[0].shape[0]:
            self.radii = [torch.empty((P,), dtype=torch.int32, device=self.device) for _ in range(self.ring)]
            if self.product:
                self.normals_s = [torch.empty((P, 3), dtype=torch.float32, device=self.device) for _ in range(self.nstreams)]
                self.normals = self.normals_s[0]
        del P_old

    def render(self, packed_cams: torch.Tensor, consume: Optional[Callable] = None,
               before_frame: Optional[Callable[[int], Optional[Dict[str, torch.Tensor]]]] = None) -> List[Dict[str, int]]:
        """Render every row of ``packed_cams`` ([N,37] host tensor).  ``consume(i, frame, stats)`` receives the finished
        frame (pinned host memory if ``to_host`` else the device ring slot; a ``[5,H,W]`` tensor, or the dict described in
        the class docstring when ``product``) — valid until ``ring-1`` further frames have been issued.
        ``before_frame(i)`` runs before frame ``i`` is issued and may return the Gaussians of that frame (per-frame object
        edits: ``lambda i: resident_scene.compose(transforms[i])``; reference scene_representation.py:357-371).  Returns the
        per-frame statistics."""
        n = packed_cams.shape[0]
        stats: List[Optional[Dict[str, int]]] = [None] * n
        inflight = []  # (frame index, slot, ticket, copy_done_event)
        cur = torch.cuda.current_stream(self.device)
        multi = self.compute_streams is not None and before_frame is None
        if multi:  # the compute streams start after whatever the caller queued on its stream (parameter uploads, edits)
            start = torch.cuda.Event()
            start.record(cur)
            for cs in self.compute_streams:
                cs.wait_event(start)

        def stream_of(slot):
            return self.compute_streams[slot % self.nstreams] if multi else cur

        def retire(entry):
            i, slot, ticket, ev = entry
            if not ticket.ok():  # binning overflow: re-render this frame synchronously with the grown capacity
                self.rerendered += 1
                if ev is not None:
                    ev.synchronize()  # the earlier (useless) async copy of this slot must not race the re-render / re-copy
                if before_frame is not None:  # later frames may have edited the resident arrays: restore frame i's scene first
                    g_i = before_frame(i)
                    if g_i is not None:
                        self.set_gaussians(g_i)
                with torch.cuda.stream(stream_of(slot)):
                    ticket = self._issue(slot, packed_cams[i], sync=True)
                    if self.to_host:
                        self._copy_out(slot)
                stream_of(slot).synchronize()
            elif ev is not None:
                ev.synchronize()
            stats[i] = ticket.stats()
            if consume is not None:
                consume(i, self._finished(slot), stats[i])

        for i in range(n):
            slot = i % self.ring
            if len(inflight) == self.ring:
                retire(inflight.pop(0))  # frees this slot (device frame + pinned frame)
            if before_frame is not None:
                g_i = before_frame(i)
                if g_i is not None:
                    self.set_gaussians(g_i)
            cs = stream_of(slot)
            with torch.cuda.stream(cs):
                ticket = self._issue(slot, packed_cams[i], sync=False)
                ev = None
                if self.to_host:
                    done = ticket.event
                    if self.product or self.pack8:  # the ticket's event was recorded after the forward; the post kernels come later on the stream
                        done = torch.cuda.Event()
                        done.record(cs)
                    self.copy_stream.wait_event(done)
                    with torch.cuda.stream(self.copy_stream):
                        self._copy_out(slot)
                        ev = torch.cuda.Event()
                        ev.record(self.copy_stream)
            inflight.append((i, slot, ticket, ev))
        while inflight:
            retire(inflight.pop(0))
        if multi:  # later work on the caller's stream is ordered after the frames
            for cs in self.compute_streams:
                e = torch.cuda.Event()
                e.record(cs)
                cur.wait_event(e)
        return stats  # type: ignore[return-value]
