"""CPU tests of the host side: the C-ABI library loads and exports every declared symbol, size queries, the drop-in
Python surface, argument validation (reference error behaviour), caller-contract helpers.  No compute calls: there is
no GPU here and the library has no CPU path."""
import inspect
import math
import os
import re

import numpy as np
import pytest
import torch

from autovfx_b200 import scene
from autovfx_b200 import render_loop as RL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gsr_[a-z0-9_]+)\s*\(", src)))


def test_library_loads_and_exports_every_declared_symbol():
    from autovfx_b200 import _lib
    names = _declared_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(_lib.lib, n), n
    assert set(names) == set(_lib.EXPORTS)
    assert _lib.lib.gsr_abi_version() == _lib.ABI_VERSION == 4


def test_workspace_size_queries():
    from autovfx_b200._lib import lib
    assert lib.gsr_geom_bytes(0) > 0
    assert 3_000_000 * (48 + 32 + 24 + 1) <= lib.gsr_geom_bytes(3_000_000) < 3_000_000 * 110
    # 8 (pair) + 4 (list) + 1 (footprint ballot matrix) bytes per instance + a fixed 4 MiB of ballot rows (reference: 24 B + sort temp)
    per = (lib.gsr_binning_bytes(2_000_000) - lib.gsr_binning_bytes(1_000_000)) / 1_000_000
    assert 12.9 < per < 13.1 and lib.gsr_binning_bytes(1000) < 5 * 2 ** 20
    for c in (1, 1000, 12345, 7_000_000):
        assert lib.gsr_binning_capacity(lib.gsr_binning_bytes(c)) == c
    a, b = lib.gsr_image_bytes(1920, 1080), lib.gsr_image_bytes(256, 256)
    assert a > b > 256 * 256 * 4
    assert lib.gsr_dist2_bytes(100000) > 4 * 4 * 100000


def test_ctypes_structs_match_header_layout():
    from autovfx_b200 import _lib
    import ctypes as C
    assert C.sizeof(_lib.gsr_frame) == 10 * 4 + 11 * 8
    assert C.sizeof(_lib.gsr_workspace) == 6 * 8
    assert C.sizeof(_lib.gsr_counters) == 32
    assert C.sizeof(_lib.gsr_grads) == 10 * 8


def test_dropin_surface_matches_reference_names():
    import diff_gaussian_rasterization as dgr
    from simple_knn._C import distCUDA2
    S = dgr.GaussianRasterizationSettings
    assert S._fields == ("image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
                         "sh_degree", "campos", "prefiltered", "debug")
    sig = inspect.signature(dgr.GaussianRasterizer.forward)
    assert list(sig.parameters) == ["self", "means3D", "means2D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"]
    assert all(sig.parameters[p].default is None for p in ["shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"])
    assert list(inspect.signature(dgr.rasterize_gaussians).parameters) == ["means3D", "means2D", "sh", "colors_precomp", "opacities", "scales",
                                                                          "rotations", "cov3Ds_precomp", "raster_settings"]
    assert hasattr(dgr.GaussianRasterizer, "markVisible") and callable(distCUDA2)
    assert issubclass(dgr._RasterizeGaussians, torch.autograd.Function)


def _settings():
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    cam = scene.lookat_camera((0, -3, 0), (0, 0, 0), 32, 32)
    return GaussianRasterizationSettings(32, 32, cam.tanfovx, cam.tanfovy, torch.zeros(3), 1.0, cam.world_view_transform, cam.full_proj_transform, 3,
                                         cam.camera_center, False, False)


def test_argument_validation_matches_reference_messages():
    from diff_gaussian_rasterization import GaussianRasterizer
    r = GaussianRasterizer(_settings())
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="Please provide excatly one of either SHs or precomputed colors!"):
        r(m, m, torch.zeros(4, 1), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(Exception, match="Please provide excatly one of either SHs or precomputed colors!"):
        r(m, m, torch.zeros(4, 1), shs=torch.zeros(4, 16, 3), colors_precomp=torch.zeros(4, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(m, m, torch.zeros(4, 1), shs=torch.zeros(4, 16, 3), scales=torch.ones(4, 3))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(m, m, torch.zeros(4, 1), shs=torch.zeros(4, 16, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4), cov3D_precomp=torch.zeros(4, 6))


def test_no_cpu_fallback():
    """CPU tensors must fail loudly (the product has no CPU path), and a malformed means3D gives the reference's error."""
    from diff_gaussian_rasterization import GaussianRasterizer
    from autovfx_b200.knn import distCUDA2
    r = GaussianRasterizer(_settings())
    m = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        r(m, m, torch.zeros(4, 1), shs=torch.zeros(4, 16, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(RuntimeError, match=r"means3D must have dimensions \(num_points, 3\)"):
        r(torch.zeros(4, 2), m, torch.zeros(4, 1), shs=torch.zeros(4, 16, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(RuntimeError, match="no CPU path"):
        distCUDA2(torch.zeros(10, 3))
    with pytest.raises(RuntimeError):
        r.markVisible(m)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "autovfx_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                for ln in txt.splitlines():
                    if re.search(r"^\s*(from|import)\s+oracle", ln):
                        raise AssertionError("product file imports the oracle: %s: %s" % (f, ln))


# ----------------------------------------------------------------------------- caller contracts
def test_camera_contract():
    c2w = np.eye(4)
    c2w[:3, 3] = [0.5, -3.0, 0.25]
    cam = scene.camera_from_c2w(c2w, 500.0, 480.0, 640, 480)
    assert math.isclose(cam.FoVx, 2 * math.atan(640 / (2 * 500.0)))
    assert math.isclose(cam.tanfovy, 480 / (2 * 480.0), rel_tol=1e-6)
    w2c = np.linalg.inv(c2w)
    assert np.allclose(cam.world_view_transform.numpy(), w2c.T.astype(np.float32))
    P = cam.world_view_transform.inverse() @ cam.full_proj_transform  # = proj^T
    assert math.isclose(float(P[0, 0]), 1.0 / cam.tanfovx, rel_tol=1e-5) and math.isclose(float(P[1, 1]), 1.0 / cam.tanfovy, rel_tol=1e-5)
    assert math.isclose(float(P[2, 3]), 1.0, rel_tol=1e-5)  # z_sign = +1 (graphics_utils.py:67)
    assert np.allclose(cam.camera_center.numpy(), [0.5, -3.0, 0.25], atol=1e-6)
    packed = cam.packed()
    assert packed.shape == (37,) and torch.equal(packed[:16], cam.world_view_transform.reshape(-1))


def test_trajectory_json_roundtrip(tmp_path):
    traj = scene.trajectory_dict(radius=4.0, num_views=30, theta=30.0, w=1920, h=1080)
    assert set(traj) >= {"fl_x", "fl_y", "cx", "cy", "w", "h", "frames"} and len(traj["frames"]) == 30
    assert math.isclose(traj["fl_x"], 1662.77, rel_tol=1e-4)
    p = tmp_path / "traj.json"
    scene.save_trajectory(str(p), traj)
    cams = scene.cameras_from_trajectory(scene.load_trajectory(str(p)))
    assert len(cams) == 30
    for c in cams[:5]:
        assert math.isclose(float(c.camera_center.norm()), 4.0, rel_tol=1e-5)
        assert math.isclose(float(c.camera_center[2]), 4.0 * math.sin(math.radians(30)), rel_tol=1e-5)
        # looks at the origin: the origin projects to the image centre
        o = torch.tensor([0.0, 0.0, 0.0, 1.0]) @ c.full_proj_transform
        assert abs(float(o[0] / o[3])) < 1e-5 and abs(float(o[1] / o[3])) < 1e-5
    half = scene.cameras_from_trajectory(traj, downscale=2.0)
    assert half[0].image_width == 960 and half[0].image_height == 540


def test_ply_roundtrip(tmp_path):
    rng = np.random.default_rng(0)
    P, M = 37, 16
    raw = dict(xyz=rng.normal(size=(P, 3)).astype(np.float32), f_dc=rng.normal(size=(P, 1, 3)).astype(np.float32),
               f_rest=rng.normal(size=(P, M - 1, 3)).astype(np.float32), opacity=rng.normal(size=(P, 1)).astype(np.float32),
               scale=rng.normal(size=(P, 3)).astype(np.float32), rot=rng.normal(size=(P, 4)).astype(np.float32))
    p = str(tmp_path / "pc.ply")
    scene.save_ply(p, raw["xyz"], raw["f_dc"], raw["f_rest"], raw["opacity"], raw["scale"], raw["rot"])
    back = scene.load_ply(p)
    for k in raw:
        assert np.array_equal(back[k], raw[k]), k
    act = scene.activate(back)
    assert act["shs"].shape == (P, M, 3) and act["opacities"].shape == (P, 1)
    assert torch.allclose(act["rotations"].norm(dim=1), torch.ones(P), atol=1e-6)
    assert (act["scales"] > 0).all() and ((act["opacities"] > 0) & (act["opacities"] < 1)).all()
    # header layout of gaussian_model.py:187-199
    head = open(p, "rb").read(2000).decode("latin1")
    names = re.findall(r"property float (\S+)", head)
    assert names[:9] == ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] and names[-4:] == ["rot_0", "rot_1", "rot_2", "rot_3"]
    assert len(names) == 6 + 3 + 3 * (M - 1) + 1 + 3 + 4


def test_synthetic_scene_is_deterministic_and_activated():
    a, b = scene.synthetic_gaussians(1000, seed=5), scene.synthetic_gaussians(1000, seed=5)
    for k in a:
        assert torch.equal(a[k], b[k])
    assert a["shs"].shape == (1000, 16, 3) and a["opacities"].shape == (1000, 1)
    assert torch.allclose(a["rotations"].norm(dim=1), torch.ones(1000), atol=1e-6)


@pytest.mark.parametrize("n,world", [(300, 1), (300, 2), (300, 8), (7, 4), (3, 8), (0, 2)])
@pytest.mark.parametrize("mode", ["roundrobin", "block"])
def test_frame_sharding_is_a_partition(n, world, mode):
    parts = [RL.shard_indices(n, r, world, mode) for r in range(world)]
    flat = sorted(i for p in parts for i in p)
    assert flat == list(range(n))
    assert max(len(p) for p in parts) - min(len(p) for p in parts) <= (1 if mode == "roundrobin" else (n + world - 1) // world)


def test_bench_clock_sampler_windows():
    """bench.ClockSampler.report(t0, t1): samples inside the timed region when there are at least two, otherwise the loaded window so far."""
    import importlib
    import sys
    import time
    argv = sys.argv
    sys.argv = ["bench.py"]
    try:
        bench = importlib.import_module("bench")
    finally:
        sys.argv = argv
    now = time.time()
    s = bench.ClockSampler.__new__(bench.ClockSampler)  # no NVML on the CPU box: fill the sample list by hand
    s.ok, s.max_mhz, s.stop_flag = True, 1965.0, True
    s.samples = [(now - 1.0, 1965.0, 0x4, 700.0), (now - 0.5, 1950.0, 0, 710.0), (now - 0.45, 1965.0, 0, 710.0)]
    r = s.report(now - 0.6, now - 0.4)
    assert r["window"] == "timed region" and r["samples"] == 2 and r["reasons"] == [] and r["sm_max_mhz"] == 1965.0 and r["sm_mhz"] == 1965.0
    r = s.report(now - 0.1, now)
    assert r["samples"] == 3 and r["reasons"] == ["sw_power_cap"] and r["window"].startswith("warm-up")
    s.ok = False
    assert s.report(0, 1)["reasons"] == ["unavailable"]
