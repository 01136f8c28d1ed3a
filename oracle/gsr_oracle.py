"""TEST INFRASTRUCTURE — numpy/ctypes front end of the CPU oracle (oracle/gsr_oracle.c).

Only tests/, bench.py's cpu_baseline / reference legs and __graft_entry__.smoke() may import this
module; the product package (autovfx_b200) never does.  Parity status: pinned against golden vectors
produced by the reference's own CUDA code (tests/golden/, see tests/golden/make_golden.py).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Dict, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgsr_oracle.so")
_lib = None

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "gsr_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "cpu"], stdout=subprocess.DEVNULL)
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.gsro_preprocess.restype = C.c_int64
        _lib.gsro_binning.restype = C.c_int
    return _lib


def _opt(a: Optional[np.ndarray]):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def forward(means3D, opacities, view, proj, campos, W, H, tanfovx, tanfovy, *, shs=None, colors_precomp=None,
            scales=None, rotations=None, cov3D_precomp=None, sh_degree=3, scale_modifier=1.0, bg=(0, 0, 0),
            prefiltered=False, stop_after: str = "render") -> Dict[str, np.ndarray]:
    """Full forward (Rasterizer::forward, rasterizer_impl.cu:197-339).  Returns every stage buffer."""
    L = lib()
    means3D = _opt(means3D)
    P = means3D.shape[0]
    opacities = _opt(opacities).reshape(-1)
    shs, colors_precomp = _opt(shs), _opt(colors_precomp)
    scales, rotations, cov3D_precomp = _opt(scales), _opt(rotations), _opt(cov3D_precomp)
    view, proj, campos = _opt(view).reshape(-1), _opt(proj).reshape(-1), _opt(campos).reshape(-1)
    bg = np.asarray(bg, dtype=np.float32)
    M = 0 if shs is None else shs.shape[1]
    out = {
        "radii": np.zeros(P, np.int32), "means2D": np.zeros((P, 2), np.float32), "depths": np.zeros(P, np.float32),
        "cov3D": np.zeros((P, 6), np.float32), "rgb": np.zeros((P, 3), np.float32),
        "conic_opacity": np.zeros((P, 4), np.float32), "clamped": np.zeros((P, 3), np.uint8),
        "tiles_touched": np.zeros(P, np.uint32),
    }
    R = L.gsro_preprocess(C.c_int(P), C.c_int(sh_degree), C.c_int(M), _p(means3D), _p(scales), C.c_float(scale_modifier),
                          _p(rotations), _p(opacities), _p(shs), _p(cov3D_precomp), _p(colors_precomp), _p(view), _p(proj),
                          _p(campos), C.c_int(W), C.c_int(H), C.c_float(tanfovx), C.c_float(tanfovy), C.c_int(int(prefiltered)),
                          _p(out["radii"]), _p(out["means2D"]), _p(out["depths"]), _p(out["cov3D"]), _p(out["rgb"]),
                          _p(out["conic_opacity"]), _p(out["clamped"]), _p(out["tiles_touched"]))
    if R < 0:
        raise RuntimeError("oracle: point culled although prefiltered is set (reference traps, auxiliary.h:156-160)")
    out["num_rendered"] = int(R)
    if stop_after == "preprocess":
        return out
    gx, gy = (W + 15) // 16, (H + 15) // 16
    out["keys"] = np.zeros(R, np.uint64)
    out["point_list"] = np.zeros(R, np.uint32)
    out["ranges"] = np.zeros((gx * gy, 2), np.uint32)
    rc = L.gsro_binning(C.c_int(P), C.c_int(W), C.c_int(H), _p(out["means2D"]), _p(out["depths"]), _p(out["radii"]),
                        _p(out["tiles_touched"]), C.c_int64(R), _p(out["keys"]), _p(out["point_list"]), _p(out["ranges"]))
    if rc != 0:
        raise RuntimeError("oracle binning failed: %d" % rc)
    if stop_after == "binning":
        return out
    out["color"] = np.zeros((3, H, W), np.float32)
    out["depth"] = np.zeros((1, H, W), np.float32)
    out["alpha"] = np.zeros((1, H, W), np.float32)
    out["n_contrib"] = np.zeros((H, W), np.uint32)
    feats = colors_precomp if colors_precomp is not None else out["rgb"]
    L.gsro_render(C.c_int(W), C.c_int(H), _p(out["ranges"]), _p(out["point_list"]), _p(out["means2D"]), _p(feats),
                  _p(out["depths"]), _p(out["conic_opacity"]), _p(bg), _p(out["color"]), _p(out["depth"]), _p(out["alpha"]),
                  _p(out["n_contrib"]))
    return out


def backward(fw: Dict[str, np.ndarray], means3D, view, proj, campos, W, H, tanfovx, tanfovy, dL_dcolor, dL_ddepth,
             dL_dalpha, *, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None, sh_degree=3,
             scale_modifier=1.0, bg=(0, 0, 0)) -> Dict[str, np.ndarray]:
    """Rasterizer::backward (rasterizer_impl.cu:343-446) on the buffers of a previous ``forward``."""
    L = lib()
    means3D = _opt(means3D)
    P = means3D.shape[0]
    shs, colors_precomp = _opt(shs), _opt(colors_precomp)
    scales, rotations, cov3D_precomp = _opt(scales), _opt(rotations), _opt(cov3D_precomp)
    view, proj, campos = _opt(view).reshape(-1), _opt(proj).reshape(-1), _opt(campos).reshape(-1)
    bg = np.asarray(bg, dtype=np.float32)
    M = 0 if shs is None else shs.shape[1]
    dL_dcolor, dL_ddepth, dL_dalpha = _opt(dL_dcolor), _opt(dL_ddepth), _opt(dL_dalpha)
    g = {
        "dL_dmeans2D": np.zeros((P, 3), np.float32), "dL_dconic": np.zeros((P, 4), np.float32),
        "dL_dopacity": np.zeros((P, 1), np.float32), "dL_dcolors": np.zeros((P, 3), np.float32),
        "dL_ddepths": np.zeros((P, 1), np.float32), "dL_dmeans3D": np.zeros((P, 3), np.float32),
        "dL_dcov3D": np.zeros((P, 6), np.float32), "dL_dsh": np.zeros((P, M, 3), np.float32),
        "dL_dscales": np.zeros((P, 3), np.float32), "dL_drotations": np.zeros((P, 4), np.float32),
    }
    feats = colors_precomp if colors_precomp is not None else fw["rgb"]
    L.gsro_render_backward(C.c_int(W), C.c_int(H), _p(fw["ranges"]), _p(fw["point_list"]), _p(bg), _p(fw["means2D"]),
                           _p(fw["conic_opacity"]), _p(feats), _p(fw["depths"]), _p(fw["alpha"]), _p(fw["n_contrib"]),
                           _p(dL_dcolor), _p(dL_ddepth), _p(dL_dalpha), _p(g["dL_dmeans2D"]), _p(g["dL_dconic"]),
                           _p(g["dL_dopacity"]), _p(g["dL_dcolors"]), _p(g["dL_ddepths"]))
    cov3Ds = cov3D_precomp if cov3D_precomp is not None else fw["cov3D"]
    L.gsro_preprocess_backward(C.c_int(P), C.c_int(sh_degree), C.c_int(M), _p(means3D), _p(fw["radii"]), _p(shs),
                               _p(fw["clamped"]), _p(scales), _p(rotations), C.c_float(scale_modifier), _p(cov3Ds), _p(view),
                               _p(proj), C.c_int(W), C.c_int(H), C.c_float(tanfovx), C.c_float(tanfovy), _p(campos),
                               _p(g["dL_dmeans2D"]), _p(g["dL_dconic"]), _p(g["dL_dmeans3D"]), _p(g["dL_dcolors"]),
                               _p(g["dL_ddepths"]), _p(g["dL_dcov3D"]), _p(g["dL_dsh"]), _p(g["dL_dscales"]),
                               _p(g["dL_drotations"]))
    return g


def mark_visible(means3D, view, proj) -> np.ndarray:
    means3D = _opt(means3D)
    out = np.zeros(means3D.shape[0], np.uint8)
    lib().gsro_mark_visible(C.c_int(means3D.shape[0]), _p(means3D), _p(_opt(view).reshape(-1)), _p(_opt(proj).reshape(-1)), _p(out))
    return out.astype(bool)


def dist2(points, brute: bool = False) -> np.ndarray:
    points = _opt(points)
    out = np.zeros(points.shape[0], np.float32)
    fn = lib().gsro_dist2_brute if brute else lib().gsro_dist2
    fn(C.c_int(points.shape[0]), _p(points), _p(out))
    return out
