"""TEST INFRASTRUCTURE — runs the reference's OWN Python callers of the hot path on the GPU box.

`make -C oracle refpy` stages a handful of unmodified reference .py files into the git-ignored ``oracle/_ref_py/`` (they
travel to the GPU box like ``oracle/_ref``): ``render()`` (sugar/gaussian_splatting/gaussian_renderer/__init__.py:83-218),
``GaussianModel`` (scene/gaussian_model.py), ``Camera`` (scene/cameras.py), the utils they import, ``transform_gaussians`` /
``merge_two_gaussians`` (gaussians_utils.py), rotation_utils.py, and the reference's Python autograd front end of the
rasterizer (diff_gaussian_rasterization/__init__.py, staged as ``ref_dgr``).

This module
  * provides stand-ins for the third-party imports those files make but never exercise on this path and that are not installed
    here (``kornia.create_meshgrid``, ``plyfile``, ``trimesh``, ``e3nn``) — written from their documented behaviour;
  * binds ``ref_dgr._C`` (the pybind module of the reference) to the compiled reference CUDA (``oracle/_ref`` via
    ``oracle.ref_cuda``), so ``ref_dgr.GaussianRasterizer`` is the reference's Python on the reference's kernels;
  * loads the reference modules against a chosen rasterizer / kNN backend: ``load("ours")`` resolves
    ``diff_gaussian_rasterization`` and ``simple_knn._C`` to this repository's drop-in packages, ``load("ref")`` to the
    reference's own code.  The same reference ``render()`` can therefore be executed on both and compared output by output.

Only tests/ and tools/ import this file; the product package never does.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types
from typing import Dict

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
STAGE = os.path.join(_HERE, "_ref_py")
GS = os.path.join(STAGE, "sugar", "gaussian_splatting")


# every staged file load() imports (oracle/Makefile: refpy); a partly staged tree counts as absent
STAGED = [os.path.join(GS, "gaussian_renderer", "__init__.py"), os.path.join(GS, "scene", "gaussian_model.py"),
          os.path.join(GS, "scene", "cameras.py"), os.path.join(GS, "utils", "general_utils.py"), os.path.join(GS, "utils", "graphics_utils.py"),
          os.path.join(GS, "utils", "sh_utils.py"), os.path.join(GS, "utils", "system_utils.py"), os.path.join(STAGE, "gaussians_utils.py"),
          os.path.join(STAGE, "rotation_utils.py"), os.path.join(STAGE, "ref_dgr", "__init__.py")]


def available() -> bool:
    from . import ref_cuda
    return all(os.path.exists(p) for p in STAGED) and ref_cuda.available()


# ------------------------------------------------------------------------------------------------ third-party stand-ins
def _create_meshgrid(height, width, normalized_coordinates=True, device=None, dtype=torch.float32):
    """kornia.utils.create_meshgrid: [1, H, W, 2] grid, last dim = (x, y); pixel coordinates when not normalised."""
    xs = torch.linspace(0, width - 1, width, device=device, dtype=dtype)
    ys = torch.linspace(0, height - 1, height, device=device, dtype=dtype)
    if normalized_coordinates:
        xs = (xs / (width - 1) - 0.5) * 2
        ys = (ys / (height - 1) - 0.5) * 2
    base = torch.stack(torch.meshgrid([xs, ys], indexing="ij"), dim=-1)  # [W, H, 2]
    return base.permute(1, 0, 2).unsqueeze(0)


class _PlyProperty:
    def __init__(self, name):
        self.name = name


class PlyElement:
    """The subset of plyfile.PlyElement the reference touches: describe(), [] by property name, .properties."""

    def __init__(self, data: np.ndarray, name: str):
        self.data, self.name = data, name
        self.properties = [_PlyProperty(n) for n in data.dtype.names]

    @staticmethod
    def describe(data, name):
        return PlyElement(np.asarray(data), name)

    def __getitem__(self, key):
        return self.data[key]


class PlyData:
    """plyfile.PlyData for single-element binary little-endian files of float properties (what save_ply / load_ply use)."""
    _TYPES = {"f4": "float", "f8": "double", "i4": "int", "u1": "uchar"}

    def __init__(self, elements):
        self.elements = list(elements)

    def write(self, path):
        el = self.elements[0]
        hdr = ["ply", "format binary_little_endian 1.0", "element %s %d" % (el.name, el.data.shape[0])]
        for n in el.data.dtype.names:
            hdr.append("property %s %s" % (self._TYPES[el.data.dtype[n].str[1:]], n))
        hdr.append("end_header")
        with open(path, "wb") as f:
            f.write(("\n".join(hdr) + "\n").encode("ascii"))
            f.write(np.ascontiguousarray(el.data).astype(el.data.dtype.newbyteorder("<"), copy=False).tobytes())

    @staticmethod
    def read(path):
        inv = {v: k for k, v in PlyData._TYPES.items()}
        with open(path, "rb") as f:
            assert f.readline().strip() == b"ply"
            name, count, props = None, 0, []
            while True:
                line = f.readline().decode("ascii").strip()
                if line == "end_header":
                    break
                tok = line.split()
                if tok[0] == "format":
                    assert tok[1] == "binary_little_endian", "stand-in reads binary little-endian PLY only"
                elif tok[0] == "element":
                    name, count = tok[1], int(tok[2])
                elif tok[0] == "property":
                    props.append((tok[2], "<" + inv[tok[1]]))
            data = np.frombuffer(f.read(), dtype=np.dtype(props), count=count)
        return PlyData([PlyElement(data, name)])


def _install_stubs() -> None:
    if "kornia" not in sys.modules:
        k = types.ModuleType("kornia")
        k.create_meshgrid = _create_meshgrid
        sys.modules["kornia"] = k
    if "plyfile" not in sys.modules:
        p = types.ModuleType("plyfile")
        p.PlyData, p.PlyElement = PlyData, PlyElement
        sys.modules["plyfile"] = p
    for name in ("trimesh",):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    if "e3nn" not in sys.modules:
        e = types.ModuleType("e3nn")
        e.o3 = types.ModuleType("e3nn.o3")
        sys.modules["e3nn"], sys.modules["e3nn.o3"] = e, e.o3


# ------------------------------------------------------------------------- ref_dgr._C: the reference's pybind surface on oracle/_ref
def _none_if_empty(t):
    return None if (t is None or t.numel() == 0) else t


class _RefC(types.ModuleType):
    """rasterize_gaussians / rasterize_gaussians_backward / mark_visible with the signatures of DGR/rasterize_points.h, executed
    by the compiled reference (oracle/_ref/libref_dgr.so).  The C wrapper keeps ONE set of internal buffers, so the backward
    re-runs its forward first (deterministic) when another forward has happened in between."""

    def __init__(self):
        super().__init__("ref_dgr._C")
        self._calls: Dict[int, tuple] = {}
        self._last = -1

    def rasterize_gaussians(self, bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D, view, proj, tanfovx, tanfovy,
                            H, W, sh, degree, campos, prefiltered, debug):
        from . import ref_cuda
        fw = ref_cuda.forward(means3D, opacity, view, proj, campos, int(W), int(H), float(tanfovx), float(tanfovy), shs=_none_if_empty(sh),
                              colors_precomp=_none_if_empty(colors), scales=_none_if_empty(scales), rotations=_none_if_empty(rotations),
                              cov3D_precomp=_none_if_empty(cov3D), sh_degree=int(degree), scale_modifier=float(scale_modifier), bg=bg,
                              prefiltered=bool(prefiltered), debug=bool(debug))
        token = len(self._calls)
        self._calls[token] = fw
        self._last = token
        dev = means3D.device
        handle = torch.tensor([token], dtype=torch.int64)
        return fw["num_rendered"], fw["color"], fw["depth"], fw["alpha"], fw["radii"], handle, torch.empty(0, device=dev), torch.empty(0, device=dev)

    def rasterize_gaussians_backward(self, bg, means3D, radii, colors, scales, rotations, scale_modifier, cov3D, view, proj, tanfovx, tanfovy,
                                     dL_dcolor, dL_ddepth, dL_dalpha, sh, degree, campos, geomBuffer, R, binningBuffer, imgBuffer, alpha, debug):
        from . import ref_cuda
        token = int(geomBuffer[0])
        fw = self._calls.pop(token)
        if token != self._last:  # another forward overwrote the wrapper's buffers: replay this one
            k, (P, D, M, Wd, Hd, tanx, tany, mod) = fw["_keep"], fw["_cfg"]
            fw = ref_cuda.forward(k["means3D"], k["opacities"], k["view"], k["proj"], k["campos"], Wd, Hd, tanx, tany, shs=k["shs"],
                                  colors_precomp=k["colors_precomp"], scales=k["scales"], rotations=k["rotations"],
                                  cov3D_precomp=k["cov3D_precomp"], sh_degree=D, scale_modifier=mod, bg=k["bg"])
            self._last = -1
        g = ref_cuda.backward(fw, dL_dcolor, dL_ddepth, dL_dalpha, debug=bool(debug))
        return (g["dL_dmeans2D"], g["dL_dcolors"], g["dL_dopacity"], g["dL_dmeans3D"], g["dL_dcov3D"], g["dL_dsh"], g["dL_dscales"],
                g["dL_drotations"])

    def mark_visible(self, means3D, view, proj):
        from . import ref_cuda
        return ref_cuda.mark_visible(means3D, view, proj)


def _ref_knn_module():
    from . import ref_cuda
    m = types.ModuleType("simple_knn._C")
    m.distCUDA2 = lambda pts: ref_cuda.dist2(pts.float().contiguous())
    return m


_REF_DGR = None


def ref_rasterizer_package():
    """The reference's diff_gaussian_rasterization Python package (staged as ref_dgr) on the reference's CUDA."""
    global _REF_DGR
    if _REF_DGR is None:
        _install_stubs()
        if STAGE not in sys.path:
            sys.path.insert(0, STAGE)
        sys.modules["ref_dgr._C"] = _RefC()
        _REF_DGR = importlib.import_module("ref_dgr")
    return _REF_DGR


def _load_file(name: str, path: str):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


_LOADED: Dict[str, types.SimpleNamespace] = {}


def load(backend: str) -> types.SimpleNamespace:
    """Reference modules bound to a backend: "ours" (this repo's drop-in diff_gaussian_rasterization / simple_knn) or "ref"
    (the reference's Python + CUDA).  Returns a namespace: renderer (gaussian_renderer), gaussian_model, cameras, graphics_utils,
    sh_utils, general_utils, gaussians_utils, rotation_utils, rasterizer (the diff_gaussian_rasterization package in use)."""
    if backend in _LOADED:
        return _LOADED[backend]
    assert backend in ("ours", "ref")
    _install_stubs()
    for p in (ROOT, STAGE, GS):
        if p not in sys.path:
            sys.path.insert(0, p)
    if backend == "ours":
        dgr = importlib.import_module("diff_gaussian_rasterization")
        knn_c = importlib.import_module("simple_knn._C")
        assert os.path.dirname(os.path.abspath(dgr.__file__)).startswith(ROOT), "the repo's drop-in package must be the one imported"
    else:
        dgr = ref_rasterizer_package()
        knn_c = _ref_knn_module()
    # the reference files import `diff_gaussian_rasterization`, `simple_knn._C`, `utils.*`, `scene.*` by those names at import time
    saved = {k: sys.modules.get(k) for k in ("diff_gaussian_rasterization", "simple_knn", "simple_knn._C", "utils", "scene",
                                             "scene.gaussian_model", "utils.general_utils", "utils.graphics_utils", "utils.sh_utils",
                                             "utils.system_utils", "rotation_utils")}
    try:
        sys.modules["diff_gaussian_rasterization"] = dgr
        knn_pkg = types.ModuleType("simple_knn")
        knn_pkg._C = knn_c
        sys.modules["simple_knn"], sys.modules["simple_knn._C"] = knn_pkg, knn_c
        tag = "_refpy_%s" % backend
        utils_pkg = types.ModuleType("utils")
        utils_pkg.__path__ = [os.path.join(GS, "utils")]
        sys.modules["utils"] = utils_pkg
        for n in ("system_utils", "general_utils", "graphics_utils", "sh_utils"):
            m = _load_file("utils." + n, os.path.join(GS, "utils", n + ".py"))
            setattr(utils_pkg, n, m)
        scene_pkg = types.ModuleType("scene")
        scene_pkg.__path__ = [os.path.join(GS, "scene")]
        sys.modules["scene"] = scene_pkg
        gm = _load_file("scene.gaussian_model", os.path.join(GS, "scene", "gaussian_model.py"))
        scene_pkg.gaussian_model = gm
        cams = _load_file(tag + ".cameras", os.path.join(GS, "scene", "cameras.py"))
        renderer = _load_file(tag + ".gaussian_renderer", os.path.join(GS, "gaussian_renderer", "__init__.py"))
        rot = _load_file("rotation_utils", os.path.join(STAGE, "rotation_utils.py"))
        # gaussians_utils imports `sugar.gaussian_splatting.scene.gaussian_model`: give it the module loaded above
        sgs = sys.modules.get("sugar.gaussian_splatting.scene.gaussian_model")
        sys.modules["sugar.gaussian_splatting.scene.gaussian_model"] = gm
        for pkg in ("sugar", "sugar.gaussian_splatting", "sugar.gaussian_splatting.scene"):
            if pkg not in sys.modules:
                sys.modules[pkg] = types.ModuleType(pkg)
        gu = _load_file(tag + ".gaussians_utils", os.path.join(STAGE, "gaussians_utils.py"))
        if sgs is not None:
            sys.modules["sugar.gaussian_splatting.scene.gaussian_model"] = sgs
        ns = types.SimpleNamespace(renderer=renderer, gaussian_model=gm, cameras=cams, graphics_utils=sys.modules["utils.graphics_utils"],
                                   sh_utils=sys.modules["utils.sh_utils"], general_utils=sys.modules["utils.general_utils"],
                                   gaussians_utils=gu, rotation_utils=rot, rasterizer=dgr, backend=backend)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    _LOADED[backend] = ns
    return ns


# ------------------------------------------------------------------------------------------------ small helpers for the tests
def make_model(ns, raw: Dict[str, torch.Tensor], max_sh_degree: int, active_sh_degree: int):
    """A reference GaussianModel holding the raw parameter tensors of ``raw`` (xyz, f_dc [N,1,3], f_rest [N,M-1,3], opacity [N,1],
    scaling [N,3], rotation [N,4]) on cuda, as nn.Parameters like load_ply / create_from_pcd leave them."""
    from torch import nn
    m = ns.gaussian_model.GaussianModel(max_sh_degree)
    dev = torch.device("cuda")
    par = lambda t: nn.Parameter(t.detach().clone().to(dev).float().contiguous().requires_grad_(True))  # noqa: E731
    m._xyz, m._features_dc, m._features_rest = par(raw["xyz"]), par(raw["f_dc"]), par(raw["f_rest"])
    m._opacity, m._scaling, m._rotation = par(raw["opacity"]), par(raw["scaling"]), par(raw["rotation"])
    m.active_sh_degree = active_sh_degree
    return m


def make_camera(ns, R: np.ndarray, T: np.ndarray, fovx: float, fovy: float, W: int, H: int):
    """The reference Camera (scene/cameras.py:17-58) for a pinhole view; image is only used for its size."""
    img = torch.zeros(3, H, W)
    return ns.cameras.Camera(colmap_id=0, R=R, T=T, FoVx=fovx, FoVy=fovy, image=img, gt_alpha_mask=None, image_name="t", uid=0,
                             data_device="cuda")


class Pipe:
    """pipeline parameters render() reads (arguments/__init__.py PipelineParams)."""
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
