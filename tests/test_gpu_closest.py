"""RayMesh.closest / compute_closest_points and the melting-mesh frame (gsr_mesh_closest, gsr_mesh_isin_rows).  Run with -m gpu.

  1. tri and the bits of d2 equal the numpy brute force (tests/closest_ref.py) over every (point, triangle) pair on the ray-cast
     tests' meshes (icospheres, a height field, the mixed scene with duplicates, coplanar overlaps, degenerate and non-finite
     triangles), for near-surface, far, vertex, edge-midpoint, face and bisector-plane points, float32 and float64;
  2. N = 0, F = 0 and an all-invalid mesh; 4,096 of 3M near-surface points on the 2.41M-triangle bench scene against the torch
     mirror; bitwise repeats across runs, streams and a rebuild; ray casts unchanged after closest calls;
  3. the device isin line equals np.isin and gives MaskScorer.count the same integer;
  4. ResidentScene.compose(melting=...) equals activate() of the scene and of orig[np.isin(ids, melt_ids)] in the reference's
     order, with one device-to-host copy per frame.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import closest_ref as R  # noqa: E402
from tests.test_gpu_raycast import MESHES, heightfield, icosphere, scene_mixed  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import raycast  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


def normals(v, f):
    t = R.triangles(v, f)
    with np.errstate(all="ignore"):
        n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
        n /= np.linalg.norm(n, axis=1, keepdims=True)
    return np.nan_to_num(n)


def points_for(v, f, n, seed):
    """Points of every kind the tests name: near the surface (like Gaussians, offset along the normals), far away, on vertices,
    on edge midpoints, on faces, on the bisector plane of two adjacent triangles, and non-finite ones."""
    rng = np.random.default_rng(seed)
    t = R.triangles(v, f)
    ok = np.isfinite(t).all(axis=(1, 2))
    ti = np.nonzero(ok)[0]
    nm = normals(v, f)
    fin = v[np.isfinite(v).all(1)]
    lo, hi = fin.min(0), fin.max(0)
    ext = (hi - lo).max()
    k = n // 6
    out = []
    pick = ti[rng.integers(0, len(ti), k)]
    w = rng.dirichlet([1, 1, 1], k)
    out.append((t[pick] * w[:, :, None]).sum(1) + nm[pick] * (0.02 * ext * rng.standard_normal((k, 1))))  # near the surface
    out.append((lo + hi) / 2 + ext * 3 * rng.standard_normal((k, 3)))                                         # far
    out.append(t[ti[rng.integers(0, len(ti), k)], rng.integers(0, 3, k)])                                     # vertices
    pe = ti[rng.integers(0, len(ti), k)]
    e = rng.integers(0, 3, k)
    out.append(0.5 * (t[pe, e] + t[pe, (e + 1) % 3]))                                                       # edge midpoints
    pf = ti[rng.integers(0, len(ti), k)]
    out.append((t[pf] * rng.dirichlet([2, 2, 2], k)[:, :, None]).sum(1))                                     # on faces
    # the bisector plane of two triangles sharing an edge: the edge midpoint moved along the sum of their normals
    m = n - 5 * k
    shared = {}
    fv = np.asarray(f)
    for i in ti[: min(len(ti), 4000)]:
        for a in range(3):
            key = tuple(sorted((fv[i, a], fv[i, (a + 1) % 3])))
            shared.setdefault(key, []).append(i)
    pairs = [(key, fs[:2]) for key, fs in shared.items() if len(fs) >= 2][:m]
    bis = [0.5 * (v[a] + v[b]) + 0.05 * ext * rng.standard_normal() * (nm[i] + nm[j]) for (a, b), (i, j) in pairs]
    out.append(np.array(bis).reshape(-1, 3))
    p = np.concatenate(out)
    p[:3] = [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]]
    return p


def assert_same(tri, d2, rtri, rd2):
    tri, d2 = tri.cpu().numpy(), d2.cpu().numpy()
    bad = np.nonzero((tri != rtri) | (d2.view(np.int64) != rd2.view(np.int64)))[0]
    assert len(bad) == 0, "%d of %d points differ, first %s: ours (%s, %r), oracle (%s, %r)" % (
        len(bad), len(tri), bad[:5], tri[bad[:5]], d2[bad[:5]], rtri[bad[:5]], rd2[bad[:5]])


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_closest_equals_brute_force(dev, name, dtype):
    from autovfx_b200.raycast import RayMesh
    v, f = MESHES[name]()
    p = points_for(v, f, 1500, seed=sorted(MESHES).index(name)).astype(dtype)
    rm = RayMesh(v.astype(dtype) if name != "mixed" else v, f.astype(np.int32) if dtype == "float32" else f)
    tri, d2 = rm.closest(p)
    assert tri.dtype == torch.int64 and d2.dtype == torch.float64 and tri.device == dev
    vr = v.astype(dtype).astype(np.float64) if name != "mixed" else v
    rtri, rd2 = R.closest(p, vr, f)
    assert (rtri >= 0).sum() == len(p) - 3 and (rtri[:3] == -1).all()
    if dtype == "float64" or name != "mixed":
        assert (rd2 == 0).sum() > 0  # the vertex, edge and face points lie on the mesh (the mixed mesh stays float64)
    assert_same(tri, d2, rtri, rd2)
    assert torch.equal(rm.compute_closest_points(torch.from_numpy(p).to(dev))["primitive_ids"], tri)


def test_empty_and_invalid(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = icosphere(2)
    rm = RayMesh(v, f)
    tri, d2 = rm.closest(np.zeros((0, 3)))
    assert tri.shape == (0,) and d2.shape == (0,)
    empty = RayMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    tri, d2 = empty.closest(np.ones((5, 3), np.float32))
    assert tri.tolist() == [-1] * 5 and torch.isinf(d2).all()
    bad_v = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2], [np.nan, 0, 0], [0, 1, 0]], np.float64)
    invalid = RayMesh(bad_v, np.array([[0, 1, 2], [0, 3, 4], [0, 0, 4], [1, 1, 1]]))
    tri, d2 = invalid.closest(np.array([[0, 0, 0], [0.5, 0.5, 0.5], [9, 9, 9.]]))
    assert tri.tolist() == [-1] * 3 and torch.isinf(d2).all()


def test_bench_scene_sample(dev):
    """3M near-surface points against the 2.41M-triangle bench scene; 4,096 of them against the torch float64 mirror."""
    from autovfx_b200.raycast import RayMesh
    from tools.bench_closest import near_surface_points, scene
    v, f = scene(1000)
    assert len(f) == 2_409_600
    rm = RayMesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
    pts = near_surface_points(v, f, 3_000_000, seed=1, device=dev)
    tri, d2 = rm.closest(pts)
    assert int((tri < 0).sum()) == 0
    sel = torch.randperm(len(pts), generator=torch.Generator().manual_seed(2))[:4096].to(dev)
    tris = torch.from_numpy(R.triangles(v, f)).to(dev)
    ok = torch.from_numpy(R.valid(R.triangles(v, f))).to(dev)
    rtri, rd2 = R.closest_torch(pts[sel].cpu().numpy(), tris, ok)
    assert_same(tri[sel], d2[sel], rtri.cpu().numpy(), rd2.cpu().numpy())
    # the torch mirror is the numpy restatement: check it on a slice where numpy is affordable
    sub = slice(0, 20000)
    q = pts[sel[:32]].cpu().numpy()
    ntri, nd2 = R.closest(q, v, f[sub])
    ttri, td2 = R.closest_torch(q, tris[sub], ok[sub])
    assert np.array_equal(ttri.cpu().numpy(), ntri) and np.array_equal(td2.cpu().numpy().view(np.int64), nd2.view(np.int64))


def test_deterministic_and_ray_casts_unchanged(dev):
    from autovfx_b200.raycast import RayMesh
    from tests.test_gpu_raycast import rays_for
    v, f = scene_mixed()
    rm = RayMesh(v, f)
    o, d = rays_for(v, f, 20000, seed=4)
    hits = rm.first_hit(o, d)
    p = torch.from_numpy(points_for(v, f, 200000, seed=12)).to(dev)
    a = rm.closest(p)
    b = rm.closest(p)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        c = rm.closest(p)
        rm2 = RayMesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
        e = rm2.closest(p.float())
        e64 = rm2.closest(p)
    torch.cuda.synchronize(dev)
    for x in (b, c, e64):
        assert torch.equal(a[0], x[0]) and torch.equal(a[1].view(torch.int64), x[1].view(torch.int64))
    assert torch.equal(e[0], rm.closest(p.float())[0])
    after = rm.first_hit(o, d)
    assert torch.equal(hits[0], after[0]) and torch.equal(hits[1].view(torch.int64), after[1].view(torch.int64))


def test_isin_line_and_mask_scorer(dev):
    """extract_object.py:105-110 and :191-192 on the device: compute_closest_points, then mask_triangles[triangle_ids] equals
    np.isin(triangle_ids, mask_triangles_idx) and gives MaskScorer.count the same integer."""
    from autovfx_b200.extract import MaskScorer
    from autovfx_b200.raycast import RayMesh
    from tests import extract_ref as X
    from tests.test_gpu_extract import _masks, _scene
    from autovfx_b200 import rasterizer as Rz
    pc, cam = _scene("config1", dev)
    views = X.orbit_views(cam, 4, dev)
    xyz = pc._xyz.detach()
    lo, hi = xyz.min(0).values.cpu().numpy().astype(np.float64), xyz.max(0).values.cpu().numpy().astype(np.float64)
    hv, hf = heightfield(40, 40, seed=9, size=1.0)
    v = lo + hv * np.r_[hi[:2] - lo[:2], (hi[2] - lo[2]) * 2]
    rm = RayMesh(v.astype(np.float32), hf)
    triangle_ids = rm.compute_closest_points(xyz)["primitive_ids"]
    assert int((triangle_ids < 0).sum()) == 0
    ids_h = triangle_ids.cpu().numpy()
    assert np.array_equal(ids_h, R.closest(xyz.cpu().numpy(), v.astype(np.float32), hf)[0])
    Rz.set_exact_images(True)
    try:
        masks = _masks(pc, views, dev)
        scorer = MaskScorer(pc, views, masks, X.PIPE)
        rng = np.random.default_rng(3)
        for frac in (0.0, 0.1, 0.5, 1.0):
            mask_triangles = rng.random(len(hf)) < frac
            mask3d = torch.from_numpy(mask_triangles).cuda()[triangle_ids]
            ref = np.isin(ids_h, np.where(mask_triangles)[0])
            assert np.array_equal(mask3d.cpu().numpy(), ref)
            assert int(scorer.count(mask3d)) == int(scorer.count(ref))
    finally:
        Rz.set_exact_images(False)


def _obj_raw(n, M, center, seed):
    rng = np.random.default_rng(seed)
    u = rng.standard_normal((n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    xyz = center + u * (1.0 + 0.02 * rng.standard_normal((n, 1)))
    return {"xyz": torch.from_numpy(xyz.astype(np.float32)), "f_dc": torch.from_numpy(rng.standard_normal((n, 1, 3)).astype(np.float32)),
            "f_rest": torch.from_numpy(0.1 * rng.standard_normal((n, M - 1, 3)).astype(np.float32)),
            "opacity": torch.from_numpy(rng.standard_normal((n, 1)).astype(np.float32)),
            "scaling": torch.from_numpy((rng.standard_normal((n, 3)) - 4).astype(np.float32)),
            "rotation": torch.from_numpy(rng.standard_normal((n, 4)).astype(np.float32))}


def test_melting_frames(dev):
    from autovfx_b200 import edit
    from autovfx_b200.raycast import RayMesh
    from torch.profiler import ProfilerActivity, profile
    M = 16
    scene = _obj_raw(30000, M, np.zeros(3), 0)
    meshes = {"a_obj": icosphere(3, center=(3, 0, 0)), "b_obj": icosphere(2, center=(-3, 0, 0), radius=1.2)}
    raws = {"a_obj": _obj_raw(8000, M, np.array([3.0, 0, 0]), 1), "b_obj": _obj_raw(5000, M, np.array([-3.0, 0, 0]), 2)}
    melting = {k: (raws[k], RayMesh(meshes[k][0].astype(np.float32), meshes[k][1])) for k in meshes}
    rs = edit.ResidentScene(scene, device=dev, melting=melting)
    ids = {k: R.closest(raws[k]["xyz"].numpy(), meshes[k][0].astype(np.float32), meshes[k][1])[0] for k in meshes}
    assert all((ids[k] >= 0).all() for k in ids)
    rng = np.random.default_rng(5)

    def centres(k, kind):
        v, f = meshes[k]
        t = R.triangles(v, f).mean(axis=1)
        if kind == "empty":
            return np.zeros((0, 3), np.float32)
        if kind == "whole":
            return t.astype(np.float32)
        sel = rng.random(len(t)) < 0.3
        return (t[sel] + 0.05 * rng.standard_normal((int(sel.sum()), 3))).astype(np.float32)  # a melted copy, displaced

    frames = [{"a_obj": [centres("a_obj", "part"), centres("a_obj", "part")], "b_obj": [centres("b_obj", "whole")]},
              {"b_obj": [centres("b_obj", "empty"), centres("b_obj", "part")], "a_obj": [centres("a_obj", "whole")]},
              {"a_obj": [centres("a_obj", "empty")]},
              {}]
    want_scene = edit.activate(scene, dev)
    for fr in frames:
        torch.cuda.synchronize(dev)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            got = rs.compose(melting=fr)
            torch.cuda.synchronize(dev)
        d2h = [e for e in prof.events() if e.device_type.name == "CUDA" and "DtoH" in e.name]
        assert len(d2h) == (1 if any(len(c) for c in fr.values()) else 0), [e.name for e in d2h]
        parts = [want_scene]
        for k in sorted(fr):
            for c in fr[k]:
                melt_ids = R.closest(c, meshes[k][0].astype(np.float32), meshes[k][1])[0]
                keep = torch.from_numpy(np.isin(ids[k], melt_ids))
                if int(keep.sum()):
                    parts.append(edit.activate({kk: vv[keep] for kk, vv in raws[k].items()}, dev))
        for key in got:
            want = torch.cat([p[key] for p in parts])
            assert got[key].shape == want.shape, key
            assert torch.equal(got[key].view(torch.int32), want.view(torch.int32)), key
    with pytest.raises(ValueError, match="exclusive"):
        rs.compose({"x": (np.zeros(3), np.eye(3), 1.0, np.zeros(3))}, melting={})
    with pytest.raises(KeyError):
        rs.compose(melting={"c_obj": [np.zeros((1, 3))]})
