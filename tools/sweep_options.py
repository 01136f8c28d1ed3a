"""Developer A/B harness for the gsr_set_option knobs: one process, one scene, many configurations.

    python tools/sweep_options.py --frames 120 --configs "sort_single_pass=0;sort_single_pass=1;blend_persist=5" --streams 1,2

One scene (3M Gaussians, 1080p trajectory); for every configuration (';'-separated, each a ','-separated list of name=value; options
not named are reset to their defaults) and stream count the frames of the trajectory are issued through PreparedForward round-robin
over the streams and timed with CUDA events (async issue, the same loop as bench.py's headline); with one stream the per-kernel
times come from the events inside gsr_forward.  The first configuration's images are the reference for a bit-equality check of every
other one.  Appends one JSON line per (configuration, streams) to gpurun_out/sweep_options.jsonl.  (The co-residency experiment of
profiles/r02_experiments.md was: --configs "blend_persist=0;blend_persist=7;...;blend_persist=3" --streams 1,2,3.)"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from autovfx_b200 import scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--configs", default="blend_persist=0;blend_persist=5")
    ap.add_argument("--streams", default="1,2")
    ap.add_argument("--repeat", type=int, default=2)
    args = ap.parse_args()
    from autovfx_b200 import rasterizer as R, _lib, render_loop as RL
    dev = torch.device("cuda:0")
    g = {k: v.to(dev) for k, v in scene.config3_scene(P=args.gaussians).items()}
    cams = scene.cameras_from_trajectory(scene.trajectory_dict(num_views=300))
    packed = RL.pack_cameras(cams).to(dev)
    host = packed.cpu()
    bg = torch.zeros(3, device=dev)
    P = g["means3D"].shape[0]
    K = args.frames
    DEFAULTS = {"blend_persist": 0, "sort_single_pass": 1}
    configs = []
    for c in args.configs.split(";"):
        d = dict(DEFAULTS)
        for kv in c.split(","):
            if kv.strip():
                k_, v_ = kv.split("=")
                d[k_.strip()] = int(v_)
        configs.append((c, d))
    nstreams = [int(x) for x in args.streams.split(",")]
    NSMAX = max(nstreams)
    outs = [(torch.empty((3, 1080, 1920), device=dev), torch.empty((1, 1080, 1920), device=dev), torch.empty((1, 1080, 1920), device=dev),
             torch.empty((P,), dtype=torch.int32, device=dev)) for _ in range(NSMAX)]
    streams = [torch.cuda.Stream(dev) for _ in range(NSMAX)]
    prepared = {}

    def launch(i, NS):
        ci, si = i % 300, i % NS
        with torch.cuda.stream(streams[si]):
            pf = prepared.get((ci, si))
            if pf is None:
                pf = prepared[(ci, si)] = R.PreparedForward(g["means3D"], g["shs"], g["opacities"], g["scales"], g["rotations"], packed[ci], 1920, 1080,
                                                            bg, 3, 1.0, outs[si])
            return pf.launch(float(host[ci, 35]), float(host[ci, 36]))

    # size the binning capacity: one synchronous pass over the cameras that will be timed
    R.set_sync_mode("safe")
    for i in range(K + 8):
        with torch.cuda.stream(streams[0]):
            s = R.GaussianRasterizationSettings(1080, 1920, float(host[i % 300, 35]), float(host[i % 300, 36]), bg, 1.0, packed[i % 300][0:16],
                                                packed[i % 300][16:32], 3, packed[i % 300][32:35], False, False)
            R.forward_raw(g["means3D"], g["shs"], None, g["opacities"], g["scales"], g["rotations"], None, s, sync=True, out=outs[0])
    torch.cuda.synchronize()

    ref_img = None
    results = []
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    import ctypes as C
    for cname, cfg in configs:
        for k_, v_ in cfg.items():
            rc = _lib.lib.gsr_set_option(k_.encode(), v_)
            if rc != 0 and k_ in cname:
                raise RuntimeError("unknown option %s" % k_)
        # correctness: frame 7 on stream 0 against the first configuration's frame
        t = launch(7, 1)
        torch.cuda.synchronize()
        img = torch.cat([outs[0][0], outs[0][1], outs[0][2]]).clone()
        st7 = t.stats()
        if ref_img is None:
            ref_img = img
        same = bool(torch.equal(img, ref_img))
        for NS in nstreams:
            best = None
            kms = None
            for rep in range(args.repeat):
                if NS == 1:
                    _lib.check(_lib.lib.gsr_profile_begin_strided(K, 2), "profile")
                for i in range(8):
                    launch(i, NS)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                cur = torch.cuda.current_stream(dev)
                e0.record(cur)
                for s_ in streams[:NS]:
                    s_.wait_event(e0)
                tk = [launch(8 + i, NS) for i in range(K)]
                for s_ in streams[:NS]:
                    ev = torch.cuda.Event()
                    ev.record(s_)
                    cur.wait_event(ev)
                e1.record(cur)
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / K
                if NS == 1:
                    ms_k, nfr = (C.c_float * 5)(), C.c_int(0)
                    _lib.check(_lib.lib.gsr_profile_end(ms_k, C.byref(nfr)), "profile_end")
                    if best is None or ms < best:
                        kms = {k_: round(float(ms_k[i_]), 4) for i_, k_ in enumerate(["project", "tile_scan", "emit", "sort_tiles", "blend"])}
                ovf = sum(t_.stats()["overflow"] for t_ in tk)
                best = ms if best is None else min(best, ms)
            res = {"config": cname, "streams": NS, "kernel_ms": kms, "ms_per_frame": round(best, 4), "fps": round(1000.0 / best, 1), "bit_equal": same,
                   "overflow": ovf, "redos7": st7["exact_redos"]}
            results.append(res)
            line = json.dumps(res)
            print(line, flush=True)
            with open(os.path.join(ROOT, "gpurun_out", "sweep_options.jsonl"), "a") as f:
                f.write(line + "\n")
    for k_, v_ in DEFAULTS.items():
        _lib.lib.gsr_set_option(k_.encode(), v_)


if __name__ == "__main__":
    main()
