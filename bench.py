#!/usr/bin/env python
"""bench.py — rendered frames/s at 1920x1080 with 3M Gaussians (BASELINE.json metric), plus HBM roofline.

    python bench.py --gpus N --steps K --warmup W [--impl reference]

A *step* is one pass of the rasterizer hot path (one ``GaussianRasterizer`` forward in SH mode: projection -> binning ->
per-tile sort -> blend) over one camera of the synthetic 300-frame trajectory (SURVEY §8d configs 3/4), per rank.  With N ranks
every rank renders its own round-robin shard of the trajectory (no data-path collective; weak scaling), so the job renders N*K
frames in the timed region and ``value`` = N*K / max-over-ranks time.

Keys of the JSON line (rank 0 prints exactly one line on stdout):
* ``value``        frames/s with the Gaussians and cameras resident in HBM (async issue, no host sync, no D2H).
* ``e2e``          the same metric through the public frame loop (``autovfx_b200.render_loop.FrameLoop``) with HOST buffers: every
                   step copies its camera payload pinned-host -> device and the finished frame device -> pinned-host inside the timed
                   region.  ``e2e`` hands the frame off as the reference's loop stores it (RGBA8 + fp32 depth + 8-bit depth index,
                   18.7 MB/frame); ``e2e_fp32`` hands off the five fp32 planes (41.5 MB/frame).
* ``dropin``       frames/s through the literal drop-in call of the reference's callers: ``GaussianRasterizer(settings)(means3D=..)``
                   with nn.Parameter inputs under torch.no_grad(), safe mode (one event sync per call), fresh output tensors.
* ``value_single_stream``  the same K frames issued on ONE stream (this pass also provides ``roofline.kernel_ms``); ``value`` alternates
                   consecutive frames between two CUDA streams so that the tail of one frame's kernels overlaps the next frame's.
* ``train_step``   forward + backward through the autograd module (config 3), iterations/s.
* ``strong``       the 300-frame trajectory as ONE job over the N ranks: parameter broadcast + camera scatter + 300/N frames per
                   rank with the 8-bit hand-off to host memory; wall time and frames/s (the driver derives the speed-up over N=1).
* ``product_frame``  what the reference's render() produces per camera (SH image + normal image + normal / pseudo-normal maps).
* ``config2`` / ``config5``  the other BASELINE configs (1M-Gaussian .ply stand-in, forward; 5M SuGaR-style scene + inserted object,
                   end to end), see DESIGN.md.
* ``roofline``     dominant kernel: algorithmic bytes per launch (DESIGN.md) / its CUDA-event duration, vs the measured HBM peak of
                   MEASURED_PEAKS.json; ``frame_*`` keys give the same for the whole frame (B_fwd of SURVEY §8d).
* ``cpu_baseline``  the CPU oracle (oracle/gsr_oracle.c, OpenMP) on one frame of the same workload (rank 0, N=1);
                   ``torch_cpu_baseline``: the pure-CPU PyTorch rasterize loop (oracle/torch_cpu_raster.py) on BASELINE config 1.
* ``--impl reference``  the UNMODIFIED reference CUDA rasterizer (oracle/_ref, compiled from the reference sources) on the same GPU and
                   workload; its line carries the same metric plus ``train_step``, ``product_frame`` (the reference's own render()
                   executed from oracle/_ref_py on its own rasterizer) and ``config2``.  The reference's implementation of this
                   path *is* CUDA (it has no CPU implementation), so the reference arm runs on the device; BASELINE.md names it as the
                   >=10x target.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from autovfx_b200 import scene  # noqa: E402

W_IMG, H_IMG = 1920, 1080
N_TRAJ = 300
METRIC = "rendered frames/sec at 1920x1080, 3M Gaussians"


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def measured_hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet 3.35 TB/s)"


class ClockSampler:
    """SM clock / throttle reasons / power sampled IN-PROCESS through NVML every 4 ms on a daemon thread (nvidia-smi -lms needs a few
    hundred ms to come up, longer than a short timed region).  ``mark()`` stamps the start / end of the timed region; ``report()``
    summarises the samples that fall inside it (and says so if fewer than two do and the whole loaded window is used instead)."""
    REASONS = ((0x0000000000000008, "hw_slowdown"), (0x0000000000000040, "hw_thermal_slowdown"), (0x0000000000000020, "sw_thermal_slowdown"),
               (0x0000000000000004, "sw_power_cap"))

    def __init__(self, index: int):
        self.samples = []
        self.stop_flag = False
        self.ok = False
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
            self.ok = True
            self.t = threading.Thread(target=self._run, daemon=True)
            self.t.start()
        except Exception as ex:  # noqa: BLE001
            self.err = str(ex)

    def _run(self):
        nv = self.nv
        while not self.stop_flag:
            try:
                mhz = float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                rs = int(nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h))
                pw = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
                self.samples.append((time.time(), mhz, rs, pw))
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.004)

    def report(self, t0: float, t1: float):
        if not self.ok:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"], "samples": 0}
        window = "timed region"
        sel = [s for s in self.samples if t0 <= s[0] <= t1]
        if len(sel) < 2:
            window = "warm-up + timed region (same kernels, back to back)"
            sel = [s for s in self.samples if s[0] <= t1]
        mhz = sorted(s[1] for s in sel)
        bits = 0
        for s in sel:
            bits |= s[2]
        return {"sm_mhz": mhz[len(mhz) // 2] if mhz else None, "sm_max_mhz": self.max_mhz, "reasons": [n for b, n in self.REASONS if bits & b],
                "samples": len(sel), "power_w_max": max((s[3] for s in sel), default=None), "window": window, "how": "NVML in-process, 4 ms period"}

    def stop(self):
        self.stop_flag = True


def dist_setup():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def algorithmic_bytes(P, P_vis, R, M_used=16):
    """SURVEY §8d / DESIGN.md: bytes that must move once per forward frame, split per stage (kernel)."""
    project = P * 44 + P * 4 + P_vis * 28           # means, scales, rotations, opacity read; radii + 2D geometry written
    color_emit = P_vis * (12 * M_used + 12) + R * 12  # SH + colour; key + value written once
    sort = R * 12                                    # key + value read once (one-pass lower bound of the sort)
    blend = R * 40 + W_IMG * H_IMG * 20
    return {"project": project, "tile_scan": 0, "color_emit": color_emit, "sort_tiles": sort, "blend": blend,
            "frame": project + color_emit + sort + blend}


_RESULT_FD = None


def emit_result(line) -> None:
    data = (json.dumps(line) + "\n").encode()
    sys.stdout.flush()
    os.write(1 if _RESULT_FD is None else _RESULT_FD, data)


def cuda_time(fn, n, sync):
    """ms per call of fn(i), i in range(n), between two events on the current stream."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync()
    e0.record()
    out = [fn(i) for i in range(n)]
    e1.record()
    sync()
    return e0.elapsed_time(e1) / max(n, 1), out


def config2_tensors(dev):
    """BASELINE config 2 stand-in through the .ply path: write, re-read, activate on the GPU."""
    import tempfile
    from autovfx_b200 import edit
    raw = scene.config2_raw()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "config2.ply")
        n = lambda t: t.numpy()  # noqa: E731
        scene.save_ply(p, n(raw["xyz"]), n(raw["f_dc"]), n(raw["f_rest"]), n(raw["opacity"]), n(raw["scaling"]), n(raw["rotation"]))
        ld = scene.load_ply(p)
    g = edit.activate({"xyz": torch.from_numpy(ld["xyz"]), "f_dc": torch.from_numpy(ld["f_dc"]), "f_rest": torch.from_numpy(ld["f_rest"]),
                       "opacity": torch.from_numpy(ld["opacity"]), "scaling": torch.from_numpy(ld["scale"]), "rotation": torch.from_numpy(ld["rot"])}, dev)
    return g, scene.config2_camera().to(dev)


DUMP_BYTES = 64 << 20


def dump_outputs(outdir, arrays):
    """DIR/<name>.npy as float32, at most DUMP_BYTES in all: each array whole while it fits (at 1080p the images and up to ~5.7M
    radii do), else a fixed seeded sample of its elements in the remaining budget, their sorted indices in <name>_index.npy (float64)."""
    import numpy as np
    os.makedirs(outdir, exist_ok=True)
    left = DUMP_BYTES
    for name, t in arrays.items():
        a = t.float().cpu().numpy()
        if a.nbytes > left:
            n = left // 12  # 4 bytes per value + 8 per index
            idx = np.sort(np.random.default_rng(0).choice(a.size, n, replace=False))
            a = a.reshape(-1)[idx]
            np.save(os.path.join(outdir, name + "_index.npy"), idx.astype(np.float64))
            left -= idx.size * 8
        np.save(os.path.join(outdir, name + ".npy"), a)
        left -= a.nbytes


# ===================================================================================================== reference arm
def reference_arm(args, K, Wm, dev, g, cams, my_cams, my_cams_host, workload, g_cpu):
    from oracle import ref_cuda
    cam_of_step = lambda s: s % my_cams.shape[0]  # noqa: E731
    if not ref_cuda.available():
        # no compiled reference on this box: fall back to the CPU oracle port on a bounded sample
        from tests import helpers as Hh
        a = Hh.resolve(dict(g=g_cpu, cam=cams[0], sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0))
        t = time.time()
        Hh.run_oracle(a)
        dt = time.time() - t
        fps = 1.0 / dt
        emit_result({"impl": "reference", "metric": METRIC, "value": fps, "unit": "frames/s", "n_gpus": 0, "steps": 1, "warmup": 0,
                     "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                     "config": {"workload": workload},
                     "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": os.cpu_count(), "kind": "port", "sample": "1 frame (camera 0), CPU oracle"},
                     "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}})
        return 0

    def ref_frame(s):
        ci = cam_of_step(s)
        c = my_cams[ci]
        return ref_cuda.forward(g["means3D"], g["opacities"], c[0:16], c[16:32], c[32:35], W_IMG, H_IMG, float(my_cams_host[ci, 35]),
                                float(my_cams_host[ci, 36]), shs=g["shs"], scales=g["scales"], rotations=g["rotations"], sh_degree=3)
    sampler = ClockSampler(dev.index)
    for s in range(Wm):
        ref_frame(s)
    torch.cuda.synchronize()
    t0 = time.time()
    ms, outs = cuda_time(lambda s: ref_frame(Wm + s)["num_rendered"], K, torch.cuda.synchronize)
    clocks = sampler.report(t0, time.time())
    fps = 1000.0 / ms
    # forward + backward (config 3) on the reference's own kernels
    gen = torch.Generator().manual_seed(7)
    dc, dd, da = (torch.randn(c, H_IMG, W_IMG, generator=gen).to(dev) for c in (3, 1, 1))
    n_tr = max(3, min(20, K))
    for s in range(2):
        ref_cuda.backward(ref_frame(s), dc, dd, da)
    ms_tr, _ = cuda_time(lambda s: ref_cuda.backward(ref_frame(Wm + s), dc, dd, da), n_tr, torch.cuda.synchronize)
    # product frame: the reference's own render() (two rasterizer passes + torch post-processing) on its own rasterizer
    product = None
    try:
        from oracle import ref_py
        if ref_py.available():
            ns = ref_py.load("ref")

            class _PC:  # the fields render() reads, already activated (what GaussianModel.get_* return)
                active_sh_degree, max_sh_degree = 3, 3
                get_xyz, get_opacity, get_scaling, get_rotation, get_features = g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"]

                @staticmethod
                def get_normal(dir_pp_normalized=None):
                    ax = ns.general_utils.get_minimum_axis(g["scales"], g["rotations"])
                    ax, _ = ns.general_utils.flip_align_view(ax, dir_pp_normalized)
                    return ax / ax.norm(dim=1, keepdim=True)
            bgz = torch.zeros(3, device=dev)

            def ref_product(s):
                c = my_cams[cam_of_step(s)]

                class _Cam:
                    FoVx, FoVy = 2 * math.atan(float(my_cams_host[cam_of_step(s), 35])), 2 * math.atan(float(my_cams_host[cam_of_step(s), 36]))
                    image_height, image_width = H_IMG, W_IMG
                    world_view_transform, full_proj_transform, camera_center = c[0:16].view(4, 4), c[16:32].view(4, 4), c[32:35]
                with torch.no_grad():
                    return ns.renderer.render(_Cam, _PC, ref_py.Pipe(), bgz)["render"]
            n_pr = max(3, min(30, K))
            for s in range(2):
                ref_product(s)
            ms_pr, _ = cuda_time(lambda s: ref_product(Wm + s), n_pr, torch.cuda.synchronize)
            product = {"value": 1000.0 / ms_pr, "unit": "product frames/s", "frames": n_pr,
                       "note": "the reference's own render() (gaussian_renderer/__init__.py:83-218, executed from oracle/_ref_py) on its own "
                               "Python front end + CUDA rasterizer: two passes + torch post-processing; fed already-activated parameters (the "
                               "per-frame exp / sigmoid / normalize of GaussianModel.get_* are not charged to it)"}
    except Exception as ex:  # noqa: BLE001
        product = {"value": None, "error": "%s: %s" % (type(ex).__name__, ex)}
    # config 2 (1M .ply stand-in, forward) on the reference rasterizer
    cfg2 = None
    try:
        g2, cam2 = config2_tensors(dev)

        def ref_c2(_):
            return ref_cuda.forward(g2["means3D"], g2["opacities"], cam2.world_view_transform, cam2.full_proj_transform, cam2.camera_center, W_IMG, H_IMG,
                                    cam2.tanfovx, cam2.tanfovy, shs=g2["shs"], scales=g2["scales"], rotations=g2["rotations"], sh_degree=3)
        for s in range(3):
            ref_c2(s)
        ms_c2, o2 = cuda_time(ref_c2, 30, torch.cuda.synchronize)
        cfg2 = {"value": 1000.0 / ms_c2, "unit": "frames/s", "num_rendered": o2[-1]["num_rendered"],
                "workload": "config 2 stand-in: 1M Gaussians (seed 1) through the .ply path, one 1920x1080 camera, forward"}
        del g2
    except Exception as ex:  # noqa: BLE001
        cfg2 = {"value": None, "error": str(ex)}
    knn = None
    try:
        ref_cuda.dist2(g["means3D"][:100000])
        torch.cuda.synchronize()
        ms_knn, _ = cuda_time(lambda i: ref_cuda.dist2(g["means3D"]).shape[0], 1, torch.cuda.synchronize)
        knn = {"value": ms_knn, "unit": "ms", "points": int(g["means3D"].shape[0]), "higher_is_better": False, "what": "SimpleKNN::knn (KNN/simple_knn.cu:185-220) on the 3M means, 1 call"}
    except Exception as ex:  # noqa: BLE001
        knn = {"value": None, "error": str(ex)}
    emit_result({"impl": "reference", "metric": METRIC, "value": fps, "unit": "frames/s", "n_gpus": 1, "steps": K, "warmup": Wm, "ms_per_step": ms,
                 "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                 "config": {"workload": workload, "reference": "unmodified diff-gaussian-rasterization CUDA (oracle/_ref) on the same GPU",
                            "avg_num_rendered": sum(outs) / len(outs), "l2": "inputs larger than L2 (708 MB of SH per frame)"},
                 "clocks": clocks,
                 "train_step": {"value": 1000.0 / ms_tr, "unit": "iterations/s", "ms": ms_tr, "iterations": n_tr,
                                "what": "Rasterizer::forward + Rasterizer::backward, dL/dimage ~ N(0,1) seed 7"},
                 "product_frame": product, "config2": cfg2, "dist2": knn,
                 "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": 1, "kind": "reference",
                                  "sample": "%d frames; the reference path is CUDA, driven by 1 host thread incl. its per-frame blocking D2H" % K},
                 "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}})
    return 0


# ===================================================================================================== main
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--gaussians", type=int, default=3_000_000, help="override only for debugging; the metric is quoted at 3M")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--quick", action="store_true", help="headline + e2e only (skip the secondary measurements)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed headline frame (color, depth, alpha, radii) as DIR/<name>.npy")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes the outputs of this implementation's timed path: use it with --impl ours")
    # stdout carries exactly ONE line, the JSON result: everything else that writes to file descriptor 1 (NCCL's version
    # banner, library chatter) is sent to stderr for the duration of the run
    sys.stdout.flush()
    global _RESULT_FD
    _RESULT_FD = os.dup(1)
    os.dup2(2, 1)
    K, Wm = args.steps, max(args.warmup, 3)
    rank, world, local = dist_setup()
    if os.environ.get("BENCH_DEBUG_DUMP"):
        import faulthandler
        faulthandler.dump_traceback_later(float(os.environ["BENCH_DEBUG_DUMP"]), repeat=True, file=sys.stderr)
    if args.impl == "reference" and rank != 0:
        return 0  # only rank 0 runs the reference arm

    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    use_dist = world > 1 and args.impl == "ours"
    from autovfx_b200.render_loop import bind_to_gpu_numa_node
    affinity = bind_to_gpu_numa_node(local)
    log("[bench] rank %d: cpu affinity %s" % (rank, affinity))
    if use_dist:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        dist.barrier()

    def barrier():
        if use_dist:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def reduce_ranks(x: float, op: str) -> float:
        if not use_dist:
            return x
        import torch.distributed as dist
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX if op == "max" else dist.ReduceOp.SUM)
        return float(t.item())

    # ---- workload: synthetic 3M-Gaussian scene + 300-camera trajectory (generated on rank 0, broadcast over NCCL) ----
    t0 = time.time()
    traj = scene.trajectory_dict(radius=4.0, num_views=N_TRAJ, theta=30.0, w=W_IMG, h=H_IMG, fov_x_deg=60.0)
    cams = scene.cameras_from_trajectory(traj)
    g_cpu = scene.config3_scene(P=args.gaussians) if rank == 0 else None
    from autovfx_b200 import render_loop as RL
    g0 = {k: v.to(dev) for k, v in g_cpu.items()} if rank == 0 else None  # the scene starts resident on rank 0's GPU (loading it is not the job)
    packed_all = RL.pack_cameras(cams) if rank == 0 else None
    if use_dist:  # NCCL connects its channels lazily on the first use of each pattern (broadcast tree, point-to-point for scatter):
        import torch.distributed as dist  # that one-time communicator set-up happens here, before the timed distribution of the job
        warm = torch.zeros(8 << 20, device=dev)
        dist.broadcast(warm, src=0)
        del warm
        RL.scatter_cameras(torch.zeros((world, RL.CAM_FLOATS)) if rank == 0 else None, world, dev)
        if rank != 0:  # the receive buffers of the job come out of the process's caching allocator, as in a long-running render worker:
            _reserve = torch.empty(int(args.gaussians * 236 * 1.1) + (64 << 20), dtype=torch.uint8, device=dev)  # a first cudaMalloc of
            del _reserve  # 0.7 GB in a process with peer mappings costs ~20 ms; the memory stays in torch's pool, unallocated
    torch.zeros((N_TRAJ, RL.CAM_FLOATS)).to(dev)  # first small pageable host -> device copy of the process (driver-side staging set-up), untimed
    barrier()
    t_b0 = time.perf_counter()
    g = RL.broadcast_gaussians(g0, dev) if use_dist else g0
    my_cams = RL.scatter_cameras(packed_all, N_TRAJ, dev) if use_dist else packed_all.to(dev)
    barrier()
    t_distribute = reduce_ranks(time.perf_counter() - t_b0, "max")  # NCCL broadcast of the parameters from rank 0's GPU + camera scatter
    my_cams_host = my_cams.cpu()
    P = g["means3D"].shape[0]
    log("[bench] rank %d: scene P=%d, %d local cameras, setup %.1fs" % (rank, P, my_cams.shape[0], time.time() - t0))
    workload = "synthetic %.1fM Gaussians SH-deg 3 (M=16), %dx%d, 300-frame half-sphere trajectory, forward" % (P / 1e6, W_IMG, H_IMG)
    peak, peak_src = measured_hbm_peak()
    cam_of_step = lambda s: s % my_cams.shape[0]  # noqa: E731

    if args.impl == "reference":
        return reference_arm(args, K, Wm, dev, g, cams, my_cams, my_cams_host, workload, g_cpu)

    # =================================================================================== our arm
    from autovfx_b200 import rasterizer as R
    from autovfx_b200 import _lib
    import ctypes as C
    bg = torch.zeros(3, device=dev)

    def settings_for(s):
        ci = cam_of_step(s)
        c = my_cams[ci]
        return R.GaussianRasterizationSettings(image_height=H_IMG, image_width=W_IMG, tanfovx=float(my_cams_host[ci, 35]), tanfovy=float(my_cams_host[ci, 36]),
                                               bg=bg, scale_modifier=1.0, viewmatrix=c[0:16], projmatrix=c[16:32], sh_degree=3, campos=c[32:35],
                                               prefiltered=False, debug=False)

    all_settings = [settings_for(s) for s in range(Wm + K)]
    out_ring = [(torch.empty((3, H_IMG, W_IMG), device=dev), torch.empty((1, H_IMG, W_IMG), device=dev), torch.empty((1, H_IMG, W_IMG), device=dev),
                 torch.empty((P,), dtype=torch.int32, device=dev)) for _ in range(2)]

    def frame(s, sync, tight=False, exact=False):
        return R.forward_raw(g["means3D"], g["shs"], None, g["opacities"], g["scales"], g["rotations"], None, all_settings[s], sync=sync, out=out_ring[s % 2],
                             tight=tight, exact=exact)

    # The timed loops issue each frame through rasterizer.PreparedForward (what FrameLoop uses): arguments resolved once per
    # (camera, output slot), camera rows resident on the device; issuing a frame is one C call + the 32-byte counters copy, a few
    # microseconds of host time, so N ranks sharing the host's cores do not slow each other's launch thread down.
    prepared = {}

    def frame_fast(s):
        ci, slot = cam_of_step(s), s % 2
        pf = prepared.get((ci, slot))
        if pf is None:
            pf = prepared[(ci, slot)] = R.PreparedForward(g["means3D"], g["shs"], g["opacities"], g["scales"], g["rotations"], my_cams[ci], W_IMG, H_IMG,
                                                          bg, 3, 1.0, out_ring[slot])
        return pf.launch(float(my_cams_host[ci, 35]), float(my_cams_host[ci, 36]))

    # pre-pass (untimed, synchronous): every camera of the run is rendered once, which sizes the binning capacity — the timed loop is the
    # steady state of a render loop over a known trajectory (no frame of it meets an undersized buffer; overflows would be re-rendered)
    sampler = ClockSampler(local)
    for s in range(Wm + K):
        frame(s, True)
    attempts = 0
    while True:
        attempts += 1
        for s in range(Wm + K):  # untimed: builds and binds the prepared call of every step, then the warm-up proper
            frame_fast(s)
        for s in range(Wm):
            frame_fast(s)
        barrier()
        _lib.check(_lib.lib.gsr_profile_begin_strided(K, 4), "gsr_profile_begin")  # per-kernel events on every 4th frame of the timed region
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t_w0 = time.time()
        e0.record()
        tickets = [frame_fast(Wm + s) for s in range(K)]
        e1.record()
        barrier()
        t_w1 = time.time()
        ms_k = (C.c_float * 5)()
        nfr = C.c_int(0)
        _lib.check(_lib.lib.gsr_profile_end(ms_k, C.byref(nfr)), "gsr_profile_end")
        clocks = sampler.report(t_w0, t_w1)
        ms_local = e0.elapsed_time(e1)
        st = [t.stats() for t in tickets]
        bad = [x for x in st if x["overflow"]]
        throttled = any(r in clocks["reasons"] for r in ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"))
        if (not bad and not throttled) or attempts >= 2:
            break
        log("[bench] re-measuring (overflow=%d throttled=%s)" % (len(bad), throttled))
    ms_single = reduce_ranks(ms_local, "max")
    frames_total = K * world
    value_single = frames_total / (ms_single * 1e-3)

    # ---- headline: the same K frames alternating between two CUDA streams (separate workspaces per stream): the tail of one frame's
    #      kernels overlaps the head of the next frame's.  The single-stream pass above provides the per-kernel breakdown. ----
    streams = [torch.cuda.Stream(dev) for _ in range(2)]

    def frame_on(s):
        with torch.cuda.stream(streams[s % 2]):
            return frame_fast(s)
    for s in range(Wm + 2):
        with torch.cuda.stream(streams[s % 2]):
            frame(s, True)
    prepared.clear()  # the prepared calls are bound to the workspaces of the stream they run on
    for s in range(Wm + K):
        frame_on(s)
    for s in range(Wm):
        frame_on(s)
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_v0 = time.time()
    e0.record()
    for st_ in streams:
        st_.wait_event(e0)
    tk2 = [frame_on(Wm + s) for s in range(K)]
    for st_ in streams:
        ev = torch.cuda.Event()
        ev.record(st_)
        torch.cuda.current_stream(dev).wait_event(ev)
    e1.record()
    barrier()
    clocks2 = sampler.report(t_v0, time.time())
    ms = reduce_ranks(e0.elapsed_time(e1), "max")
    ovf2 = sum(t.stats()["overflow"] for t in tk2)
    if ovf2 or any(r in clocks2["reasons"] for r in ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown")):
        log("[bench] two-stream loop rejected (overflow=%d, reasons=%s): reporting the single-stream loop" % (ovf2, clocks2["reasons"]))
        ms, clocks2 = ms_single, clocks
    value = frames_total / (ms * 1e-3)
    clocks = clocks2
    if args.dump_outputs and rank == 0:  # the frame the last timed step rendered, before later measurements reuse its output slot
        dump_outputs(args.dump_outputs, dict(zip(("color", "depth", "alpha", "radii"), out_ring[(Wm + K - 1) % 2])))
    avg_R = sum(x["num_rendered"] for x in st) / len(st)
    avg_vis = sum(x["num_visible"] for x in st) / len(st)
    avg_redo = sum(x["exact_redos"] for x in st) / len(st)
    kernels = ["project", "tile_scan", "color_emit", "sort_tiles", "blend"]
    kms = {k: float(ms_k[i]) for i, k in enumerate(kernels)}
    ab = algorithmic_bytes(P, avg_vis, avg_R)
    dom = max(kms, key=kms.get)
    dom_bytes = ab[dom]
    dom_gbs = dom_bytes / (kms[dom] * 1e-3) / 1e9 if kms[dom] > 0 else 0.0
    traffic = None
    tp = os.path.join(ROOT, "profiles", "traffic.json")
    if os.path.exists(tp):
        try:
            with open(tp) as f:
                traffic = json.load(f).get(dom)
        except Exception:  # noqa: BLE001
            traffic = None
    frame_gbs = ab["frame"] / (ms / K * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "k_" + dom, "achieved": dom_gbs, "peak": peak, "unit": "GB/s", "frac": dom_gbs / peak, "traffic": traffic,
                "peak_source": peak_src, "algorithmic_bytes_per_launch": dom_bytes, "kernel_ms": kms,
                "kernel_share": {k: (v / sum(kms.values()) if sum(kms.values()) else 0) for k, v in kms.items()},
                "per_kernel_gbs": {k: (ab[k] / (v * 1e-3) / 1e9 if v > 0 else 0) for k, v in kms.items()},
                "frame_algorithmic_bytes": ab["frame"], "frame_achieved": frame_gbs, "frame_frac": frame_gbs / peak,
                "note": "k_blend_lists reads the 40 bytes of every splat it evaluates from shared memory in every lane of a warp, so its HBM "
                        "fraction is low by design; it is reported because the metric names the HBM roofline. The HBM-streaming kernels are "
                        "k_project and k_color_emit (per_kernel_gbs)"}

    line = {"metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wm,
            "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload, "gaussians": P, "avg_visible": avg_vis, "avg_num_rendered": avg_R, "frames_per_rank": K,
                       "parallelism": "frame-sharded x%d (round-robin cameras, NCCL only for parameter broadcast + camera scatter)" % world,
                       "l2": "inputs larger than L2 (708 MB of SH read per frame; 50 MB L2 on H100)",
                       "streams": "frames alternate between 2 CUDA streams (value); value_single_stream and roofline.kernel_ms come from the same K frames "
                                  "on one stream",
                       "api": "rasterizer.PreparedForward.launch per frame (the call FrameLoop makes), device-resident camera rows",
                       "sync": "async issue, counters validated after the timed region; an untimed pre-pass rendered every camera of the run once (steady "
                               "state of a loop over a known trajectory: binning capacity already sized)",
                       "image_mode": "default: alpha = ex2.approx(power*log2e + log2 opacity), decisions inside the error band re-blended exactly "
                                     "(avg %.0f of 65,280 warps per frame); GSR_FLAG_EXACT_IMAGES gives bit-identical images (exact_images key)" % avg_redo},
            "clocks": clocks, "gpu_launches": 5 * K * world, "value_single_stream": value_single, "roofline": roofline}

    def timed_loop(fn, n=K):
        for s in range(Wm):
            fn(s)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        tk = [fn(Wm + s) for s in range(n)]
        e1.record()
        barrier()
        return reduce_ranks(e0.elapsed_time(e1), "max"), tk

    log("[bench] headline done: %.1f frames/s" % value)
    if not args.quick:
        # ---- bit-identical image mode and opt-in tight tiles, reported separately ----
        for s in range(Wm):
            frame(s, True, exact=True)
        ms_ex, _ = timed_loop(lambda s: frame(s, False, exact=True)[5])
        line["exact_images"] = {"value": frames_total / (ms_ex * 1e-3), "unit": "frames/s",
                                "note": "GSR_FLAG_EXACT_IMAGES: the reference's fp32 instruction sequence in the blend, images bit-identical to its CUDA"}
        for s in range(Wm):
            frame(s, True, tight=True)
        ms_tight, tt = timed_loop(lambda s: frame(s, False, tight=True)[5])
        st_t = [t.stats() for t in tt]
        line["tight_tiles"] = {"value": frames_total / (ms_tight * 1e-3), "unit": "frames/s", "avg_num_rendered": sum(x["num_rendered"] for x in st_t) / len(st_t),
                               "note": "opt-in GSR_FLAG_TIGHT_TILES: per-tile lists are sub-sequences of the reference's; images / radii unchanged. "
                                       "This loop records no per-kernel events (the headline loop records six per 4th frame)"}

        log("[bench] exact/tight done (%.0f s)" % (time.time() - t0))
        # ---- the literal drop-in call of the reference's callers: module call, Parameters under no_grad, safe mode ----
        params = {k: torch.nn.Parameter(g[k]) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
        m2 = torch.zeros_like(g["means3D"])

        def dropin(s):
            with torch.no_grad():
                out = R.GaussianRasterizer(all_settings[s])(means3D=params["means3D"], means2D=m2, opacities=params["opacities"], shs=params["shs"],
                                                            scales=params["scales"], rotations=params["rotations"])
            return out[3].shape[0]  # the four fresh output tensors of the call are dropped, like the reference's callers do per frame
        ms_di, _ = timed_loop(dropin)
        line["dropin"] = {"value": frames_total / (ms_di * 1e-3), "unit": "frames/s",
                          "api": "diff_gaussian_rasterization.GaussianRasterizer(raster_settings)(means3D=..., shs=..., ...) with nn.Parameter inputs under "
                                 "torch.no_grad(), safe mode (one event sync per call), fresh output tensors per call"}
        del params

        log("[bench] dropin done (%.0f s)" % (time.time() - t0))
        # ---- forward + backward (config 3) through the autograd module ----
        leaves = {k: g[k].detach().clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        gen = torch.Generator().manual_seed(7)
        dc, dd, da = (torch.randn(c, H_IMG, W_IMG, generator=gen).to(dev) for c in (3, 1, 1))

        def train_step(s):
            mm = torch.zeros_like(leaves["means3D"], requires_grad=True)
            color, depth, alpha, _ = R.GaussianRasterizer(all_settings[s])(leaves["means3D"], mm, leaves["opacities"], shs=leaves["shs"],
                                                                            scales=leaves["scales"], rotations=leaves["rotations"])
            ((color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()).backward()
            for v in leaves.values():
                v.grad = None
            return 0
        n_tr = max(3, min(20, K))
        ms_tr, _ = timed_loop(train_step, n_tr)
        line["train_step"] = {"value": n_tr * world / (ms_tr * 1e-3), "unit": "iterations/s", "ms": ms_tr / n_tr, "iterations": n_tr,
                              "what": "GaussianRasterizer forward + backward through torch.autograd (incl. the three image-loss reductions), dL/dimage ~ N(0,1) seed 7"}
        del leaves, dc, dd, da

        log("[bench] train_step done (%.0f s)" % (time.time() - t0))
        # ---- product frame (SURVEY §8 a19 / f-1): what the reference's render() does per camera ----
        from autovfx_b200 import renderer as RD
        normals_buf = torch.empty((P, 3), dtype=torch.float32, device=dev)
        extra_img = torch.empty((3, H_IMG, W_IMG), dtype=torch.float32, device=dev)
        c2w_dev = [torch.linalg.inv_ex(s_.viewmatrix.view(4, 4))[0].contiguous() for s_ in all_settings]
        fx_, fy_ = W_IMG / (2 * all_settings[0].tanfovx), H_IMG / (2 * all_settings[0].tanfovy)

        def product_fused(s):
            st_ = all_settings[s]
            RD.axis_normals(g["means3D"], g["scales"], g["rotations"], st_.campos, remap01=True, out=normals_buf)
            res = R.forward_multi(g["means3D"], g["shs"], None, normals_buf, g["opacities"], g["scales"], g["rotations"], None, st_, sync=False,
                                  out=out_ring[0], extra_out=extra_img)
            RD.normal_maps(extra_img, out_ring[0][1][0], c2w_dev[s], fx_, fy_, W_IMG / 2, H_IMG / 2)
            return res[5]

        def product_two_pass(s):
            st_ = all_settings[s]
            RD.axis_normals(g["means3D"], g["scales"], g["rotations"], st_.campos, remap01=True, out=normals_buf)
            R.forward_raw(g["means3D"], g["shs"], None, g["opacities"], g["scales"], g["rotations"], None, st_, sync=False, out=out_ring[0])
            t_ = R.forward_raw(g["means3D"], None, normals_buf, g["opacities"], g["scales"], g["rotations"], None, st_, sync=False, out=out_ring[1])[5]
            RD.normal_maps(out_ring[1][0], out_ring[0][1][0], c2w_dev[s], fx_, fy_, W_IMG / 2, H_IMG / 2)
            return t_
        ms_prod, tkp = timed_loop(product_fused)
        ms_prod2, _ = timed_loop(product_two_pass)
        product_info = {"value": frames_total / (ms_prod * 1e-3), "unit": "product frames/s", "overflowed": sum(t.stats()["overflow"] for t in tkp),
                        "two_pass_value": frames_total / (ms_prod2 * 1e-3),
                        "note": "one product frame = the reference's render(): SH image + normal image + normal/pseudo-normal maps. value: "
                                "axis_normals + one 6-channel forward (gsr_forward_multi) + normal_maps; two_pass_value: two forwards, the "
                                "second re-blending on the first one's geometry (GSR_FLAG_REUSE_GEOMETRY). The reference arm measures the reference's "
                                "own render() beside it (product_frame in its line)"}
        line["product_frame"] = product_info
        del normals_buf, extra_img

    log("[bench] product done (%.0f s)" % (time.time() - t0))
    # ---- e2e: public frame loop, host camera payload in, finished frame out to pinned host memory, every step ----
    e2e_cams = torch.stack([my_cams_host[cam_of_step(Wm + s)] for s in range(K)])

    def run_loop(loop, cams_host, touch):
        loop.render(cams_host[:min(cams_host.shape[0], 6)])  # warm-up (pinned buffers, copy stream)
        barrier()
        t_start = time.perf_counter()
        acc = [0.0]
        loop.render(cams_host, lambda i, fr, stt: acc.__setitem__(0, acc[0] + touch(fr)))  # the consumer touches the host copy of every frame
        torch.cuda.synchronize()
        return reduce_ranks(time.perf_counter() - t_start, "max")

    loop = RL.FrameLoop(g, 3, W_IMG, H_IMG, device=dev, ring=4, to_host=True, streams=2)
    e2e_s = run_loop(loop, e2e_cams, lambda fr: float(fr[4, H_IMG // 2, W_IMG // 2]))
    line["e2e_fp32"] = {"value": frames_total / e2e_s, "unit": "frames/s", "h2d_bytes_per_step": loop.h2d_bytes_per_frame, "d2h_bytes_per_step": loop.d2h_bytes_per_frame,
                        "api": "FrameLoop.render, five fp32 planes [5,H,W] per frame to pinned host memory (41.5 MB/frame: the PCIe link / host memory is the limit at N=8)",
                        "rerendered": loop.rerendered, "d2h_gbs_per_gpu": loop.d2h_bytes_per_frame * K / e2e_s / 1e9}
    del loop
    loop8 = RL.FrameLoop(g, 3, W_IMG, H_IMG, device=dev, ring=4, to_host=True, pack8=True, streams=2)
    e2e8_s = run_loop(loop8, e2e_cams, lambda fr: int(fr["rgba8"][H_IMG // 2, W_IMG // 2, 0]) + float(fr["depth"][H_IMG // 2, W_IMG // 2]))
    line["e2e"] = {"value": frames_total / e2e8_s, "unit": "frames/s", "h2d_bytes_per_step": loop8.h2d_bytes_per_frame,
                   "d2h_bytes_per_step": loop8.d2h_bytes_per_frame, "rerendered": loop8.rerendered,
                   "api": "autovfx_b200.render_loop.FrameLoop(pack8=True, streams=2).render: per frame the camera payload host -> device, one rasterizer forward, and the "
                          "frame as the reference's loop stores it (scene_representation.py:424-433: RGBA as 8-bit PNG pixels, depth as float32 .npy + its 8-bit colormap "
                          "index) device -> pinned host memory",
                   "d2h_gbs_per_gpu": loop8.d2h_bytes_per_frame * K / e2e8_s / 1e9}

    # ---- strong scaling: the whole 300-frame trajectory as ONE job over the N ranks (8-bit hand-off) ----
    if not args.quick:
        t_job = run_loop(loop8, my_cams_host, lambda fr: int(fr["rgba8"][H_IMG // 2, W_IMG // 2, 0]))
        line["strong"] = {"frames": N_TRAJ, "wall_s": t_distribute + t_job, "render_s": t_job, "distribute_s": t_distribute,
                          "value": N_TRAJ / (t_distribute + t_job), "unit": "frames/s", "frames_per_rank": int(my_cams_host.shape[0]),
                          "what": "NCCL broadcast of the 708 MB of parameters from rank 0's GPU + camera scatter (distribute_s; the communicator's channels were "
                                  "connected by a warm-up broadcast / scatter and the receivers' allocator pool was reserved before) + every rank rendering its 300/N "
                                  "round-robin frames with the RGBA8 + depth hand-off to pinned host memory (render_s, max over ranks); fixed total work"}
    del loop8

    if not args.quick:
        log("[bench] strong done (%.0f s)" % (time.time() - t0))
        # ---- product e2e: FrameLoop(product=True, pack8=True) — render() per camera + 8-bit hand-off to pinned host memory ----
        try:
            ploop = RL.FrameLoop(g, 3, W_IMG, H_IMG, device=dev, ring=4, to_host=True, product=True, pack8=True, streams=2)
            pe2e_s = run_loop(ploop, e2e_cams, lambda fr: int(fr["rgba8"][H_IMG // 2, W_IMG // 2, 0]))
            line["product_frame"]["e2e"] = {"value": frames_total / pe2e_s, "unit": "product frames/s", "h2d_bytes_per_step": ploop.h2d_bytes_per_frame,
                                            "d2h_bytes_per_step": ploop.d2h_bytes_per_frame, "rerendered": ploop.rerendered,
                                            "api": "FrameLoop(product=True, pack8=True): render() per camera, RGBA8 + depth f32 + depth8 + normal8 to pinned host memory"}
            del ploop
        except Exception as ex:  # noqa: BLE001
            line["product_frame"]["e2e"] = {"value": None, "error": str(ex)}

        log("[bench] product e2e done (%.0f s)" % (time.time() - t0))
        # ---- config 2: 1M-Gaussian stand-in through the .ply path, one camera, forward ----
        try:
            g2, cam2 = config2_tensors(dev)
            s2 = R.GaussianRasterizationSettings(H_IMG, W_IMG, cam2.tanfovx, cam2.tanfovy, bg, 1.0, cam2.world_view_transform, cam2.full_proj_transform, 3,
                                                 cam2.camera_center, False, False)
            out2 = (out_ring[0][0], out_ring[0][1], out_ring[0][2], torch.empty((g2["means3D"].shape[0],), dtype=torch.int32, device=dev))

            def f2(_, sync=False):
                return R.forward_raw(g2["means3D"], g2["shs"], None, g2["opacities"], g2["scales"], g2["rotations"], None, s2, sync=sync, out=out2)[5]
            f2(0, True)
            ms_c2, tk = timed_loop(f2, 60)
            line["config2"] = {"value": 60 * world / (ms_c2 * 1e-3), "unit": "frames/s", "num_rendered": tk[-1].stats()["num_rendered"],
                               "workload": "config 2 stand-in: 1M Gaussians (seed 1) written to and re-read from the 3DGS .ply layout, activated on the GPU, "
                                           "one 1920x1080 camera, forward (every rank renders the same camera)"}
            del g2, out2
        except Exception as ex:  # noqa: BLE001
            line["config2"] = {"value": None, "error": str(ex)}

        log("[bench] config2 done (%.0f s)" % (time.time() - t0))
        # ---- config 5 stand-in: 5M SuGaR-style Gaussians (M=25) + a 200k-Gaussian object edited every frame, product frames, 8-bit hand-off ----
        try:
            line["config5"] = config5(dev, rank, world, barrier, reduce_ranks, frames_per_rank=40)
        except Exception as ex:  # noqa: BLE001
            line["config5"] = {"value": None, "error": "%s: %s" % (type(ex).__name__, ex)}

    log("[bench] config5 done (%.0f s)" % (time.time() - t0))
    if not args.quick and rank == 0:
        # ---- distCUDA2 (simple_knn) on the scene's 3M points: init-time call of GaussianModel.create_from_pcd ----
        try:
            from simple_knn._C import distCUDA2
            distCUDA2(g["means3D"])
            torch.cuda.synchronize()
            ms_knn, _ = cuda_time(lambda i: distCUDA2(g["means3D"]).shape[0], 3, torch.cuda.synchronize)
            line["dist2"] = {"value": ms_knn, "unit": "ms", "points": P, "higher_is_better": False,
                             "what": "simple_knn._C.distCUDA2 on the 3M means (exact 3-NN mean squared distance); the reference arm times SimpleKNN::knn on the same points"}
        except Exception as ex:  # noqa: BLE001
            line["dist2"] = {"value": None, "error": str(ex)}

    # ---- CPU baselines (rank 0, N=1 only) ----
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        try:
            from tests import helpers as Hh
            a = Hh.resolve(dict(g=g_cpu, cam=cams[0], sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0))
            t = time.time()
            Hh.run_oracle(a)
            dt = time.time() - t
            line["cpu_baseline"] = {"value": 1.0 / dt, "unit": "frames/s", "cores": os.cpu_count(), "kind": "port",
                                    "sample": "1 full frame (trajectory camera 0) of the same 3M/1080p workload, oracle/gsr_oracle.c with OpenMP, %.1f s" % dt}
        except Exception as ex:  # noqa: BLE001
            line["cpu_baseline"] = {"value": None, "unit": "frames/s", "cores": os.cpu_count(), "kind": "port", "sample": "failed: %s" % ex}
        try:
            from oracle import torch_cpu_raster as TR
            from tests import helpers as Hh
            n_thr = min(8, os.cpu_count() or 1)  # per-tile [256 x n] ops: more threads only add synchronisation (64 threads: minutes per frame)
            torch.set_num_threads(n_thr)
            a = Hh.resolve(Hh.case_inputs("config1"))
            args_t = (a["means3D"], a["scales"], a["rotations"], a["opacities"], a["shs"], a["view"], a["proj"], a["campos"], a["W"], a["H"], a["tanfovx"],
                      a["tanfovy"], 3, 1.0)
            TR.rasterize(*args_t)
            t = time.time()
            nfr = 0
            while nfr < 5 and time.time() - t < 20.0:
                TR.rasterize(*args_t)
                nfr += 1
            dt = (time.time() - t) / nfr
            line["torch_cpu_baseline"] = {"value": 1.0 / dt, "unit": "frames/s", "cores": n_thr, "host_cores": os.cpu_count(),
                                          "workload": "BASELINE config 1: 10k Gaussians, 256x256, pure-CPU PyTorch rasterize loop "
                                                      "(oracle/torch_cpu_raster.py), %d frames, torch.set_num_threads(%d)" % (nfr, n_thr)}
        except Exception as ex:  # noqa: BLE001
            line["torch_cpu_baseline"] = {"value": None, "error": str(ex)}

    sampler.stop()
    if rank == 0:
        emit_result(line)
    if use_dist:
        import torch.distributed as dist
        dist.destroy_process_group()
    return 0


def config5(dev, rank, world, barrier, reduce_ranks, frames_per_rank=40):
    """SURVEY §8d config 5 stand-in (the SuGaR checkpoint is not available offline): see tools/bench_config5.py for the stand-alone form."""
    from autovfx_b200 import edit
    from autovfx_b200 import render_loop as RL
    from tools.bench_config5 import to_raw
    n_scene, n_obj = 5_000_000, 200_000
    g_scene = scene.synthetic_gaussians(n_scene, seed=1234, extent=(4, 4, 1), log_scale_mean=math.log(0.006), log_scale_std=0.5, opacity_mean=0.0,
                                        opacity_std=2.0, sh_degree=4)
    g_obj = scene.synthetic_gaussians(n_obj, seed=77, extent=(0.4, 0.4, 0.4), log_scale_mean=math.log(0.004), log_scale_std=0.4, opacity_mean=1.0,
                                      opacity_std=1.0, sh_degree=4)
    raw_scene, M = to_raw(g_scene)
    raw_obj, _ = to_raw(g_obj)
    rs = edit.ResidentScene(raw_scene, {"obj": raw_obj}, dev)
    del g_scene, raw_scene
    cams_all = scene.cameras_from_trajectory(scene.trajectory_dict(num_views=300))
    idx = RL.shard_indices(min(300, frames_per_rank * world), rank, world)
    cams = RL.pack_cameras([cams_all[i] for i in idx])

    def transform(i):  # the object circles the origin, spinning about z, growing slightly
        a = 2 * math.pi * idx[i] / 300.0
        c, s = math.cos(3 * a), math.sin(3 * a)
        Rm = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        return {"obj": (torch.tensor([1.5 * math.cos(a), 1.5 * math.sin(a), 0.2]), Rm, 1.0 + 0.3 * math.sin(a), torch.zeros(3))}
    loop = RL.FrameLoop(rs.compose(transform(0)), 0, W_IMG, H_IMG, device=dev, ring=3, to_host=True, product=True, pack8=True)
    loop.render(cams[:4], before_frame=lambda i: rs.compose(transform(i)))
    barrier()
    chk = [0]
    t0 = time.perf_counter()
    stats = loop.render(cams, lambda i, fr, st: chk.__setitem__(0, chk[0] + int(fr["rgba8"][H_IMG // 2, W_IMG // 2, 0])),
                        before_frame=lambda i: rs.compose(transform(i)))
    torch.cuda.synchronize()
    dt = reduce_ranks(time.perf_counter() - t0, "max")
    return {"value": len(idx) * world / dt, "unit": "product frames/s", "frames_per_rank": len(idx), "rerendered": loop.rerendered,
            "avg_num_rendered": sum(s["num_rendered"] for s in stats) / len(stats), "d2h_bytes_per_step": loop.d2h_bytes_per_frame,
            "workload": "config 5 stand-in: 5M Gaussians stored SuGaR-style (M=25) + one 200k-Gaussian object moved rigidly every frame, 1920x1080, rendered at "
                        "SH degree 0 like the reference's merged model (gaussians_utils.py:75); per frame: edit + merge (ResidentScene.compose), render() "
                        "(6-channel forward + normal maps), 8-bit conversions, hand-off to pinned host memory; frames sharded over the ranks"}


if __name__ == "__main__":
    sys.exit(main())
