"""Shared helpers for the parity tests and tools: run the same seeded inputs through (a) the product CUDA path
(autovfx_b200, via the C ABI), (b) the compiled reference (oracle/_ref, GPU) and (c) the CPU oracle."""
from __future__ import annotations

import math
import os
import sys
from typing import Dict, Optional

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from autovfx_b200 import scene  # noqa: E402


def case_inputs(name: str) -> Dict:
    """Named deterministic cases.  Returns dict(g=gaussians (cpu tensors), cam=Camera, kw=extra settings)."""
    if name == "config1":  # BASELINE configs[0]: 10k Gaussians, 256x256
        g, cam = scene.config1_scene()
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "small_sh":  # tiny, non-multiple-of-16 image, coloured background
        g = scene.synthetic_gaussians(600, seed=3, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.6)
        cam = scene.lookat_camera((0.3, -3.0, 0.4), (0, 0, 0), 100, 75, 55.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.2, 0.5, 0.9), scale_modifier=1.0)
    if name == "small_deg1_m25":  # SuGaR-style storage: M=25 (stride 300 B), active degree 1, scale modifier
        g = scene.synthetic_gaussians(500, seed=5, extent=(1, 1, 1), log_scale_mean=math.log(0.06), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((-2.0, -2.0, 1.0), (0, 0, 0), 96, 64, 70.0)
        return dict(g=g, cam=cam, sh_degree=1, bg=(1.0, 1.0, 1.0), scale_modifier=0.8)
    if name == "deg3_m25":  # SuGaR storage (M=25, 300-byte rows: only 4-byte aligned) rendered at degree 3 and 2: windowed SH staging
        g = scene.synthetic_gaussians(3000, seed=23, extent=(1, 1, 1), log_scale_mean=math.log(0.04), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((1.5, -2.5, 0.8), (0, 0, 0), 144, 96, 65.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.3, 0.3, 0.3), scale_modifier=1.0)
    if name == "deg2_m25":
        g = scene.synthetic_gaussians(2000, seed=29, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((-1.0, -2.8, 0.5), (0, 0, 0), 112, 80, 65.0)
        return dict(g=g, cam=cam, sh_degree=2, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "small_precomp":  # colors_precomp + cov3D_precomp mode
        g = scene.synthetic_gaussians(700, seed=7, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.5)
        cam = scene.lookat_camera((0.0, -2.5, 1.5), (0, 0, 0), 80, 80, 60.0)
        return dict(g=g, cam=cam, sh_degree=0, bg=(0.0, 0.0, 0.0), scale_modifier=1.0, precomp=True)
    if name == "big_splats":  # few huge splats (warp-cooperative tile walk) + a camera inside the cloud (near culling)
        g = scene.synthetic_gaussians(300, seed=11, extent=(1.5, 1.5, 1.5), log_scale_mean=math.log(0.4), log_scale_std=0.7)
        cam = scene.lookat_camera((0.2, -0.6, 0.1), (0, 0.5, 0), 128, 112, 80.0)
        return dict(g=g, cam=cam, sh_degree=2, bg=(0.1, 0.1, 0.1), scale_modifier=1.0)
    if name == "dense_tile":  # > 4096 splats on single tiles: exercises the large-bucket sort path
        g = scene.synthetic_gaussians(30000, seed=13, extent=(0.05, 0.05, 1.0), log_scale_mean=math.log(0.004), log_scale_std=0.3,
                                      opacity_mean=-3.0, opacity_std=1.0)
        cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 64, 64, 40.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "coplanar":  # thousands of exactly equal depths: sort ties resolve by Gaussian id; degenerate depth range
        g = scene.synthetic_gaussians(6000, seed=17, extent=(0.6, 0.0, 0.6), log_scale_mean=math.log(0.02), log_scale_std=0.3,
                                      opacity_mean=-2.0, opacity_std=1.0)
        cam = scene.lookat_camera((0.0, -2.0, 0.0), (0, 0, 0), 96, 96, 50.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.2, 0.0), scale_modifier=1.0)
    raise KeyError(name)


def load_golden(path: str) -> Dict:
    """A golden case; the gradients of the larger cases are stored beside it under golden/grads/ (same file name)."""
    gold = dict(np.load(path))
    grads = os.path.join(os.path.dirname(path), "grads", os.path.basename(path))
    if os.path.exists(grads):
        gold.update(np.load(grads))
    return gold


def cov3d_from(scales: torch.Tensor, rotations: torch.Tensor, mod: float) -> torch.Tensor:
    """Python-side precomputed covariance (what gaussian_model.get_covariance builds, gaussian_model.py:47-52,117-118)."""
    r, x, y, z = rotations.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).view(-1, 3, 3)
    L = R * (scales * mod).unsqueeze(1)  # R @ diag(s)
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=-1).contiguous()


def resolve(case: Dict, device=None) -> Dict:
    """Flatten a case into the exact argument set of one rasterizer call."""
    g, cam = case["g"], case["cam"]
    a = dict(means3D=g["means3D"], opacities=g["opacities"], view=cam.world_view_transform, proj=cam.full_proj_transform,
             campos=cam.camera_center, W=cam.image_width, H=cam.image_height, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
             sh_degree=case["sh_degree"], scale_modifier=case["scale_modifier"], bg=torch.tensor(case["bg"], dtype=torch.float32),
             shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None)
    if case.get("precomp"):
        gen = torch.Generator().manual_seed(99)
        a["colors_precomp"] = torch.rand(g["means3D"].shape[0], 3, generator=gen)
        a["cov3D_precomp"] = cov3d_from(g["scales"], g["rotations"], case["scale_modifier"])
    else:
        a["shs"], a["scales"], a["rotations"] = g["shs"], g["scales"], g["rotations"]
    if device is not None:
        a = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in a.items()}
    return a


def settings_from(a: Dict, debug=False, prefiltered=False):
    from autovfx_b200.rasterizer import GaussianRasterizationSettings
    return GaussianRasterizationSettings(image_height=a["H"], image_width=a["W"], tanfovx=a["tanfovx"], tanfovy=a["tanfovy"], bg=a["bg"],
                                         scale_modifier=a["scale_modifier"], viewmatrix=a["view"], projmatrix=a["proj"],
                                         sh_degree=a["sh_degree"], campos=a["campos"], prefiltered=prefiltered, debug=debug)


def run_ours(a: Dict, for_backward=False, sorted_keys=False, debug=True, tight=None, exact=None):
    from autovfx_b200 import rasterizer as R
    s = settings_from(a, debug=debug)
    color, depth, alpha, radii, ws, ticket, keep = R.forward_raw(a["means3D"], a["shs"], a["colors_precomp"], a["opacities"], a["scales"],
                                                                 a["rotations"], a["cov3D_precomp"], s, for_backward=for_backward,
                                                                 sorted_keys=sorted_keys, sync=True, tight=tight, exact=exact)
    views = R.debug_views(ws, a["means3D"].shape[0], a["W"], a["H"])
    return dict(color=color, depth=depth, alpha=alpha, radii=radii, views=views, stats=ticket.stats(), ws=ws, keep=keep)


def run_ref(a: Dict):
    """The compiled reference's forward on the same tensors, or None where it is not built: comparisons against its outputs
    go through the ref_* helpers below, which replay stored digests of them in that case."""
    from oracle import ref_cuda
    if not ref_cuda.available():
        return None
    fw = ref_cuda.forward(a["means3D"], a["opacities"], a["view"], a["proj"], a["campos"], a["W"], a["H"], a["tanfovx"], a["tanfovy"],
                          shs=a["shs"], colors_precomp=a["colors_precomp"], scales=a["scales"], rotations=a["rotations"],
                          cov3D_precomp=a["cov3D_precomp"], sh_degree=a["sh_degree"], scale_modifier=a["scale_modifier"], bg=a["bg"])
    return fw


def ref_state(device):
    """ref_cuda.state() after run_ref, or None where the reference is not built."""
    from oracle import ref_cuda
    return ref_cuda.state(device) if ref_cuda.available() else None


def ref_backward(a: Dict, dc, dd, da):
    """The reference's gradients for run_ref(a), or None where the reference is not built."""
    from oracle import ref_cuda
    return ref_cuda.backward(run_ref(a), dc, dd, da) if ref_cuda.available() else None


def run_oracle(a: Dict, stop_after="render"):
    from oracle import gsr_oracle as O
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    return O.forward(n(a["means3D"]), n(a["opacities"]), n(a["view"]), n(a["proj"]), n(a["campos"]), a["W"], a["H"], a["tanfovx"],
                     a["tanfovy"], shs=n(a["shs"]), colors_precomp=n(a["colors_precomp"]), scales=n(a["scales"]), rotations=n(a["rotations"]),
                     cov3D_precomp=n(a["cov3D_precomp"]), sh_degree=a["sh_degree"], scale_modifier=a["scale_modifier"],
                     bg=tuple(float(v) for v in a["bg"].cpu()), stop_after=stop_after)


def oracle_backward(a: Dict, fw, dc, dd, da):
    from oracle import gsr_oracle as O
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    return O.backward(fw, n(a["means3D"]), n(a["view"]), n(a["proj"]), n(a["campos"]), a["W"], a["H"], a["tanfovx"], a["tanfovy"],
                      n(dc), n(dd), n(da), shs=n(a["shs"]), colors_precomp=n(a["colors_precomp"]), scales=n(a["scales"]),
                      rotations=n(a["rotations"]), cov3D_precomp=n(a["cov3D_precomp"]), sh_degree=a["sh_degree"],
                      scale_modifier=a["scale_modifier"], bg=tuple(float(v) for v in a["bg"].cpu()))


def image_grads(a: Dict, seed=7, device=None):
    """dL/dcolor, dL/ddepth, dL/dalpha ~ N(0,1), seed 7 (SURVEY §8d config 3)."""
    g = torch.Generator().manual_seed(seed)
    H, W = a["H"], a["W"]
    dc, dd, da = torch.randn(3, H, W, generator=g), torch.randn(1, H, W, generator=g), torch.randn(1, H, W, generator=g)
    if device is not None:
        dc, dd, da = dc.to(device), dd.to(device), da.to(device)
    return dc, dd, da


def ours_backward(a: Dict, dc, dd, da):
    """Forward+backward through the public GaussianRasterizer API; returns (outputs, grads dict)."""
    from autovfx_b200.rasterizer import GaussianRasterizer
    leaves = {}
    for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"):
        leaves[k] = None if a[k] is None else a[k].detach().clone().requires_grad_(True)
    means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
    rast = GaussianRasterizer(settings_from(a))
    color, depth, alpha, radii = rast(leaves["means3D"], means2D, leaves["opacities"], shs=leaves["shs"], colors_precomp=leaves["colors_precomp"],
                                      scales=leaves["scales"], rotations=leaves["rotations"], cov3D_precomp=leaves["cov3D_precomp"])
    loss = (color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()
    loss.backward()
    grads = {k: (None if v is None else v.grad) for k, v in leaves.items()}
    grads["means2D"] = means2D.grad
    return (color, depth, alpha, radii), grads


# default (fast-alpha) blend against exact images: the measured differences are ~1e-6 of the value; BASELINE allows 1e-4
FAST_TOL = {"color": 1e-5, "alpha": 1e-5, "depth": 5e-5}


def assert_images_close(got: Dict, want: Dict, tol=None):
    for k in ("color", "depth", "alpha"):
        t = FAST_TOL[k] if tol is None else tol
        e = maxabs(got[k], want[k])
        assert e <= t, "%s: max abs %.3g > %.3g" % (k, e, t)


def maxabs(a, b) -> float:
    a = torch.as_tensor(a).float().cpu()
    b = torch.as_tensor(b).float().cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max())


def relerr(a, b) -> float:
    """max |a-b| / (max|b| + tiny): scale-aware error for gradient tensors."""
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ---- comparisons against the compiled reference (oracle/_ref), live or replayed ---------------------------------------------
# Each ref_* call compares one of our tensors with a value of the reference, passed as a function that computes it.  Where the
# reference library is built the function runs and the comparison is exact, and with GSR_REF_RECORD=<dir> every value is also
# stored, in call order, as <dir>/<test id>.npz: a SHA-256 of its bytes for bit-identity checks, a seeded sample of REF_SAMPLE
# elements (plus its max |value|) for tolerance checks: one per block of the flattened tensor.  Where
# an exact-mode image is shown bit-identical to the reference, tests also compare the default-mode image with it in full.  Where the library is absent the functions are never called and the same
# comparisons run against tests/golden/ref/<test id>.npz, recorded by the reference on an H100.
REF_GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")
REF_SAMPLE = 2048
_ref_log: Dict = {"test": None, "i": 0, "rec": {}}


def _test_id() -> str:
    tid = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    return "".join(c if c.isalnum() or c in "-_." else "_" for c in tid.replace("tests/", "", 1))


def use_ref_python():
    """Declares that the running test's reference values come from the reference's Python code (oracle/ref_py): its comparisons
    run live only where that code is staged (not merely the compiled library) and replay the stored values elsewhere."""
    _ref_log["py_test"] = _test_id()


def ref_live() -> bool:
    """Whether the running test's reference values are computed here (else they are replayed)."""
    from oracle import ref_cuda, ref_py
    return ref_py.available() if _ref_log.get("py_test") == _test_id() else ref_cuda.available()


def have_ref() -> bool:
    """The reference is built here, or its values are stored for the running test."""
    return ref_live() or os.path.exists(os.path.join(REF_GOLDEN, _test_id() + ".npz"))


def _canon(t) -> torch.Tensor:
    t = torch.as_tensor(t).detach()
    t = t.float() if t.is_floating_point() else t.long()
    return t.contiguous().cpu()


def _digest(t: torch.Tensor) -> str:
    import hashlib
    return hashlib.sha256(str(tuple(t.shape)).encode() + t.numpy().tobytes()).hexdigest()


def _sample_idx(n: int) -> np.ndarray:
    """Stratified: one seeded element from each of REF_SAMPLE equal blocks of the flattened tensor, so every region is covered."""
    if n <= REF_SAMPLE:
        return np.arange(n)
    edges = (np.arange(REF_SAMPLE + 1, dtype=np.int64) * n) // REF_SAMPLE
    return edges[:-1] + np.random.default_rng(n).integers(0, edges[1:] - edges[:-1])


def _ref_entry(kind: str, fn):
    """The reference's record for the next comparison of the running test: computed by fn (and stored when recording) or replayed."""
    tid = _test_id()
    if _ref_log["test"] != tid:
        _ref_log.update(test=tid, i=0, rec={})
    i = _ref_log["i"]
    _ref_log["i"] += 1
    if not ref_live():
        path = os.path.join(REF_GOLDEN, tid + ".npz")
        if tid not in _ref_log["rec"]:
            assert os.path.exists(path), "no compiled reference and no stored reference values (%s)" % path
            _ref_log["rec"][tid] = dict(np.load(path))
        rec = _ref_log["rec"][tid]
        assert "%d_kind" % i in rec and str(rec["%d_kind" % i]) == kind, "stored reference values do not match comparison %d" % i
        return None, {k.split("_", 1)[1]: v for k, v in rec.items() if k.split("_", 1)[0] == str(i)}
    v = fn()
    out = os.environ.get("GSR_REF_RECORD")
    if out:
        e = {"kind": np.str_(kind)}
        if kind == "value":
            e["value"] = np.asarray(v)
        else:
            c = _canon(v)
            e["shape"] = np.asarray(c.shape, dtype=np.int64)
            if kind == "same":
                e["sha"] = np.str_(_digest(c))
            else:
                flat = c.double().reshape(-1)
                e["sample"] = flat[torch.from_numpy(_sample_idx(flat.numel()))].float().numpy()
                e["absmax"] = np.asarray(float(flat.abs().max()) if flat.numel() else 0.0)
        rec = _ref_log["rec"].setdefault(tid, {})
        rec.update({"%d_%s" % (i, k): x for k, x in e.items()})
        os.makedirs(out, exist_ok=True)
        np.savez_compressed(os.path.join(out, tid + ".npz"), **rec)
    return v, None


def ref_value(fn):
    """A scalar of the reference (e.g. num_rendered)."""
    v, rec = _ref_entry("value", fn)
    return v if rec is None else rec["value"].item()


def ref_same(x, fn) -> bool:
    """Bit identity with a tensor of the reference (integers compared as int64, floats as float32)."""
    v, rec = _ref_entry("same", fn)
    if rec is None:
        a, b = _canon(x), _canon(v)
        return a.shape == b.shape and torch.equal(a, b)
    c = _canon(x)
    return list(c.shape) == rec["shape"].tolist() and _digest(c) == str(rec["sha"])


def _ref_pair(x, fn):
    v, rec = _ref_entry("sample", fn)
    a = _canon(x).double().reshape(-1)
    if rec is None:
        return a, _canon(v).double().reshape(-1), None
    assert a.numel() == int(np.prod(rec["shape"])), "shape differs from the stored reference values"
    return a[torch.from_numpy(_sample_idx(a.numel()))], torch.from_numpy(rec["sample"]).double(), float(rec["absmax"])


def ref_maxabs(x, fn) -> float:
    a, b, _ = _ref_pair(x, fn)
    return float((a - b).abs().max()) if a.numel() else 0.0


def ref_meanabs(x, fn) -> float:
    a, b, _ = _ref_pair(x, fn)
    return float((a - b).abs().mean()) if a.numel() else 0.0


def ref_allclose(x, fn, rtol: float) -> bool:
    a, b, _ = _ref_pair(x, fn)
    return bool(((a - b).abs() <= rtol * b.abs()).all())


def ref_relerr(x, fn) -> float:
    a, b, bmax = _ref_pair(x, fn)
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / ((float(b.abs().max()) if bmax is None else bmax) + 1e-30))


def ref_images_close(got: Dict, ref, tol=None):
    """assert_images_close against the reference's forward (run_ref's result, None where replayed)."""
    for k in ("color", "depth", "alpha"):
        t = FAST_TOL[k] if tol is None else tol
        e = ref_maxabs(got[k], lambda: ref[k])
        assert e <= t, "%s: max abs %.3g > %.3g" % (k, e, t)
