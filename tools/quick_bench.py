"""Developer A/B harness: per-kernel times of the forward on the bench workload (3M Gaussians, 1080p, trajectory cameras).

    python tools/quick_bench.py --frames 60 [--exact] [--tight] [--tag name]

Prints one JSON line (and appends it to gpurun_out/quick_bench.jsonl).  Kernel-selection knobs are environment variables read
once per process, so every variant is its own process.  Not the bench of record (that is bench.py)."""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from autovfx_b200 import scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--exact", action="store_true")
    ap.add_argument("--tight", action="store_true")
    ap.add_argument("--backward", action="store_true", help="also time forward+backward through autograd (20 iterations)")
    ap.add_argument("--streams", type=int, default=1, help="issue consecutive frames round-robin on this many CUDA streams")
    ap.add_argument("--prepared", action="store_true", help="issue frames through PreparedForward (a few microseconds of host time per frame)")
    ap.add_argument("--depth", type=int, default=0, help="with --prepared: wait for the ticket of frame i - depth before issuing frame i (0: never wait)")
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    from autovfx_b200 import rasterizer as R, _lib
    dev = torch.device("cuda:0")
    g = {k: v.to(dev) for k, v in scene.config3_scene(P=args.gaussians).items()}
    cams = scene.cameras_from_trajectory(scene.trajectory_dict(num_views=300))
    from autovfx_b200 import render_loop as RL
    packed = RL.pack_cameras(cams).to(dev)
    host = packed.cpu()
    bg = torch.zeros(3, device=dev)
    P = g["means3D"].shape[0]
    K = args.frames

    def settings(i):
        c = packed[i]
        return R.GaussianRasterizationSettings(1080, 1920, float(host[i, 35]), float(host[i, 36]), bg, 1.0, c[0:16], c[16:32], 3, c[32:35], False, False)
    S = [settings(i % 300) for i in range(K + 5)]
    NS = max(1, args.streams)
    outs = [(torch.empty((3, 1080, 1920), device=dev), torch.empty((1, 1080, 1920), device=dev), torch.empty((1, 1080, 1920), device=dev),
             torch.empty((P,), dtype=torch.int32, device=dev)) for _ in range(NS)]
    streams = [torch.cuda.current_stream(dev)] if NS == 1 else [torch.cuda.Stream(dev) for _ in range(NS)]

    prepared = {}
    issued = []

    def frame(i, sync):
        if args.prepared and not sync:
            ci = i % 300
            with torch.cuda.stream(streams[i % NS]):
                pf = prepared.get((ci, i % NS))
                if pf is None:
                    pf = prepared[(ci, i % NS)] = R.PreparedForward(g["means3D"], g["shs"], g["opacities"], g["scales"], g["rotations"], packed[ci], 1920, 1080, bg,
                                                                    3, 1.0, outs[i % NS], tight=args.tight, exact=args.exact)
                if args.depth > 0 and len(issued) >= args.depth:
                    issued[-args.depth].event.synchronize()
                t = pf.launch(float(host[ci, 35]), float(host[ci, 36]))
                issued.append(t)
                return (None,) * 5 + (t,)
        with torch.cuda.stream(streams[i % NS]):
            return R.forward_raw(g["means3D"], g["shs"], None, g["opacities"], g["scales"], g["rotations"], None, S[i], sync=sync, out=outs[i % NS],
                                 tight=args.tight, exact=args.exact)
    torch.cuda.synchronize()
    for i in range(K + 5):
        frame(i, True)
    if args.prepared:
        for i in range(K + 5):
            frame(i, False)
    for i in range(5):
        frame(i, False)
    torch.cuda.synchronize()
    del issued[:]
    _lib.check(_lib.lib.gsr_profile_begin_strided(K, 2), "profile")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if NS > 1:
        _lib.lib.gsr_profile_end((C.c_float * 5)(), None)  # per-kernel events assume one stream
    e0.record()
    if NS > 1:
        for st_ in streams:
            st_.wait_event(e0)
    tk = [frame(5 + i, False)[5] for i in range(K)]
    if NS > 1:
        for st_ in streams:
            ev = torch.cuda.Event()
            ev.record(st_)
            torch.cuda.current_stream(dev).wait_event(ev)
    e1.record()
    torch.cuda.synchronize()
    ms_k = (C.c_float * 5)()
    n = C.c_int(0)
    if NS == 1:
        _lib.check(_lib.lib.gsr_profile_end(ms_k, C.byref(n)), "profile_end")
    st = [t.stats() for t in tk]
    ms = e0.elapsed_time(e1) / K
    res = {"tag": args.tag, "exact": args.exact, "tight": args.tight, "streams": NS, "ms_per_frame": round(ms, 4), "fps": round(1000.0 / ms, 1),
           "kernel_ms": {k: round(float(ms_k[i]), 4) for i, k in enumerate(["project", "tile_scan", "emit", "sort_tiles", "blend"])},
           "avg_R": sum(s["num_rendered"] for s in st) / K, "avg_foot": sum(s["foot_total"] for s in st) / K,
           "avg_redos": sum(s["exact_redos"] for s in st) / K, "overflow": sum(s["overflow"] for s in st)}
    if args.backward:
        from tests import helpers as Hh  # noqa: F401
        leaves = {k: g[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        gen = torch.Generator().manual_seed(7)
        dc, dd, da = (torch.randn(c, 1080, 1920, generator=gen).to(dev) for c in (3, 1, 1))
        R.set_exact_images(args.exact)

        def step(i):
            rast = R.GaussianRasterizer(S[i])
            m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
            color, depth, alpha, _ = rast(leaves["means3D"], m2, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"])
            ((color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()).backward()
            for v in leaves.values():
                v.grad = None
        for i in range(3):
            step(i)
        torch.cuda.synchronize()
        e0.record()
        for i in range(20):
            step(3 + i)
        e1.record()
        torch.cuda.synchronize()
        res["fwd_bwd_ms"] = round(e0.elapsed_time(e1) / 20, 3)
    line = json.dumps(res)
    print(line, flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "quick_bench.jsonl"), "a") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
