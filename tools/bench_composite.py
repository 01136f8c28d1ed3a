"""Frame compositing (autovfx_b200.composite) against the reference's blend_frames (blender/blend_all.py).

Prints the card, its power limit and the host's core count, then median / p10 / p90 of:
  gpu_kernel   composite_frame at 1080p with every layer (3DGS object, smoke, fire), device time by CUDA events per call;
  cpu_body     the loop body :206-342 in numpy (tests/composite_ref.composite_np, the restatement pinned op for op against the
               reference) on the same decoded arrays, one frame;
  e2e_ref      the reference's blend_frames per frame on a synthetic 1080p directory (decode + composite + PNG write), when
               build() staged it under oracle/_ref_py: one sample per run over the directory (run time / frames);
  e2e_ours     the drop-in composite.blend_frames per frame on the same directory, runs alternated with the reference's.
The end-to-end gain is the ratio of the two medians as measured.  The floor from bytes (each layer read once, the smoke depth five times by
the percentile, the frame written once, at 3.35 TB/s) is printed as a bound, not a measurement.

    python tools/bench_composite.py [--frames 4] [--reps 5] [--iters 200] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests import composite_ref as CR  # noqa: E402


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)), "n": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5, help="timed runs of each blend_frames over the directory, after one warm-up run")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_composite measures on a GPU"
    from autovfx_b200.composite import composite_frame
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "cpu_cores": os.cpu_count()}
    H, W = 1080, 1920
    case = CR.make_case(1, H, W, True, True, True)
    want = CR.composite_np(**case)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in case.items()}
    args = dict(rgba8=t["bg_c"], depth=None, obj=t["o_c"], obj_depth=t["o_d"], shadow=t["s_c"], shadow_depth=t["s_d"], all_=t["o_s_c"],
                obj3dgs=t["o_gs_c"], obj3dgs_depth=t["o_gs_d"], smoke=t["s_f_c"], smoke_depth=t["s_f_d"], fire=t["s_f_c_pre"])
    out = composite_frame(**args)
    assert np.array_equal(out.cpu().numpy(), want), "composite_frame differs from the restatement"
    for _ in range(20):
        composite_frame(**args, out=out)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.iters)]
    for e0, e1 in ev:
        e0.record()
        composite_frame(**args, out=out)
        e1.record()
    torch.cuda.synchronize()
    res["gpu_kernel"] = stats([e0.elapsed_time(e1) for e0, e1 in ev])
    cpu = []
    for _ in range(5):
        t0 = time.perf_counter()
        CR.composite_np(**case)
        cpu.append((time.perf_counter() - t0) * 1e3)
    res["cpu_body"] = stats(cpu)
    px = H * W
    floor_bytes = px * (7 * 4 + 4 * 4 + 5 * 4 + 4)  # seven RGBA8 layers, four depths, five percentile passes over smoke, the frame
    res["floor_from_bytes_not_measured_ms"] = floor_bytes / 3.35e12 * 1e3

    ref = CR.load_reference()
    from autovfx_b200 import composite
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, _ = CR.write_dir(tmp, a.frames, 600, H, W)
        mods = []
        if ref is not None:
            ref.generate_video_from_frames = lambda frames, path, fps=30: None
            mods.append(("e2e_ref", ref))
        ours = CR.load_reference("_ours_blend_all") if ref is not None else None
        if ours is None:  # the loaders of BA/:56-75, for machines without the staged reference
            from tests.test_gpu_composite import _loaders_module
            ours = _loaders_module()
        ours.blend_frames = composite.blend_frames
        ours.generate_video_from_frames = lambda frames, path, fps=30: None
        mods.append(("e2e_ours", ours))
        per_frame = {name: [] for name, _ in mods}
        for rep in range(a.reps + 1):  # the first run warms the file cache and the decoders
            for name, m in mods:
                t0 = time.perf_counter()
                m.blend_frames(results, cfg)
                torch.cuda.synchronize()
                if rep:
                    per_frame[name].append((time.perf_counter() - t0) * 1e3 / a.frames)
        for name, v in per_frame.items():
            res[name] = dict(stats(v), frames=a.frames)
    if "e2e_ref" in res:
        res["e2e_gain_measured"] = res["e2e_ref"]["median_ms"] / res["e2e_ours"]["median_ms"]
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
