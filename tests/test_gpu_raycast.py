"""RayMesh and its kernels (gsr_mesh_build, gsr_mesh_first_hit, gsr_mesh_inpaint_mask).  Run with -m gpu on an H100.

  1. tri and the bits of t equal the numpy brute force (tests/raycast_ref.py) over every (ray, triangle) pair on meshes of about
     20k triangles: icospheres, a height field, duplicated and coplanar-overlapping triangles, degenerate and non-finite ones;
     rays through shared vertices, along edges, axis-aligned, from the surface, zero, NaN and infinite; N = 0 and F = 0;
  2. every ray aimed strictly inside a closed icosphere's silhouette hits it;
  3. at about 2M triangles, 256 rays (grazing ones included) equal a torch float64 mirror of the brute force;
  4. repeats and a second stream give the same bits; intersects_location, the vote loop's counters and the inpainting masks
     equal their restatements on the oracle's hits.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import raycast_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import raycast  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


def icosphere(level, center=(0, 0, 0), radius=1.0):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(level):
        cache, nf = {}, []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in cache:
                m = v[a] + v[b]
                v.append(m / np.linalg.norm(m))
                cache[k] = len(v) - 1
            return cache[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return np.array(v) * radius + np.asarray(center, np.float64), np.array(f, np.int64)


def heightfield(nx, ny, seed=0, size=10.0):
    rng = np.random.default_rng(seed)
    xs, ys = np.linspace(0, size, nx + 1), np.linspace(0, size, ny + 1)
    X, Y = np.meshgrid(xs, ys, indexing="xy")
    Z = 0.3 * np.sin(X) * np.cos(0.7 * Y) + 0.05 * rng.standard_normal(X.shape)
    v = np.stack([X, Y, Z], -1).reshape(-1, 3)
    i = np.arange(ny)[:, None] * (nx + 1) + np.arange(nx)[None, :]
    a, b, c, d = i, i + 1, i + nx + 1, i + nx + 2
    f = np.concatenate([np.stack([a, b, d], -1).reshape(-1, 3), np.stack([a, d, c], -1).reshape(-1, 3)])
    return v, f


def scene_mixed():
    """A height field, an icosphere on it, duplicates and coplanar overlaps, degenerate and non-finite triangles."""
    hv, hf = heightfield(70, 70, seed=1)
    sv, sf = icosphere(4, center=(5, 5, 1.5), radius=1.0)
    v = np.concatenate([hv, sv])
    f = np.concatenate([hf, sf + len(hv)])
    rng = np.random.default_rng(2)
    dup = f[rng.choice(len(f), 300, replace=False)]
    # coplanar overlaps: a flat plate at z = 2.9 and the same plate shifted by half a cell
    pv, pf = heightfield(10, 10, size=2.0)
    pv[:, 2] = 2.9
    pv[:, :2] += 3.0
    base = len(v)
    v = np.concatenate([v, pv, pv + [0.1, 0, 0]])
    f = np.concatenate([f, dup, pf + base, pf + base + len(pv)])
    # degenerate and non-finite triangles
    bad_v = np.array([[1, 1, 5], [2, 2, 5], [3, 3, 5], [np.nan, 1, 1], [np.inf, 2, 2], [4, 4, 4]], np.float64)
    base = len(v)
    v = np.concatenate([v, bad_v])
    f = np.concatenate([f, [[base, base + 1, base + 2], [base, base, base + 5], [base + 3, base + 1, base + 5], [base + 4, base + 5, base]]])
    return v, f


def rays_for(v, f, n, seed):
    """Rays of every kind the tests name: towards random surface points, through vertices, along edges, axis-aligned, from the
    surface, zero, NaN and infinite."""
    rng = np.random.default_rng(seed)
    fin = np.isfinite(v[f]).all(axis=(1, 2))
    ff = f[fin]
    lo, hi = v[np.isfinite(v).all(1)].min(0), v[np.isfinite(v).all(1)].max(0)
    c = (lo + hi) / 2
    ext = (hi - lo).max()
    o, d = [], []
    k = n // 6
    # towards random points of random triangles from outside
    tri = ff[rng.integers(0, len(ff), k)]
    w = rng.dirichlet([1, 1, 1], k)
    p = (v[tri] * w[:, :, None]).sum(1)
    src = c + ext * rng.standard_normal((k, 3))
    o.append(src); d.append(p - src)
    # through shared vertices
    vid = ff[rng.integers(0, len(ff), k), rng.integers(0, 3, k)]
    src = c + ext * rng.standard_normal((k, 3))
    o.append(src); d.append(v[vid] - src)
    # along edges (from a vertex, in the direction of the next one) and through edge midpoints
    e = ff[rng.integers(0, len(ff), k)]
    o.append(v[e[:, 0]] - 0.5 * (v[e[:, 1]] - v[e[:, 0]])); d.append(v[e[:, 1]] - v[e[:, 0]])
    src = c + ext * rng.standard_normal((k, 3))
    o.append(src); d.append(0.5 * (v[e[:, 1]] + v[e[:, 2]]) - src)
    # axis-aligned rays with zero components, above vertices of the height field and through the scene
    ax = np.zeros((k, 3))
    ax[np.arange(k), rng.integers(0, 3, k)] = rng.choice([-1.0, 1.0], k) * rng.choice([1.0, 0.5, 3.0], k)
    vv = v[ff[rng.integers(0, len(ff), k), 0]]
    o.append(vv - 4 * ax); d.append(ax)
    # origins on the surface (vertices and interior points), random directions
    m = n - 5 * k
    tri = ff[rng.integers(0, len(ff), m)]
    w = rng.dirichlet([1, 1, 1], m)
    w[: m // 2] = np.eye(3)[rng.integers(0, 3, m // 2)]
    o.append((v[tri] * w[:, :, None]).sum(1)); d.append(rng.standard_normal((m, 3)))
    o, d = np.concatenate(o), np.concatenate(d)
    # zero, NaN and infinite rays
    o[:3], d[:3] = c, [[0, 0, 0], [np.nan, 0, -1], [0, np.inf, -1]]
    o[3] = [np.nan, 0, 0]
    o[4] = [np.inf, 0, 0]
    return o, d


def assert_same(tri, t, rtri, rt):
    tri, t = tri.cpu().numpy(), t.cpu().numpy()
    bad = np.nonzero((tri != rtri) | (t.view(np.int64) != rt.view(np.int64)))[0]
    assert len(bad) == 0, "%d of %d rays differ, first %s: ours (%s, %r), oracle (%s, %r)" % (
        len(bad), len(tri), bad[:5], tri[bad[:5]], t[bad[:5]], rtri[bad[:5]], rt[bad[:5]])


MESHES = {
    "icosphere": lambda: icosphere(5),
    "heightfield": lambda: heightfield(100, 100, seed=0),
    "mixed": scene_mixed,
}


@pytest.mark.parametrize("name", list(MESHES))
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_first_hit_equals_brute_force(dev, name, dtype):
    from autovfx_b200.raycast import RayMesh
    v, f = MESHES[name]()
    assert 15000 <= len(f) <= 25000
    o, d = rays_for(v, f, 1500, seed=sorted(MESHES).index(name))
    o, d = o.astype(dtype), d.astype(dtype)
    faces = f.astype(np.int32) if dtype == "float32" else f
    rm = RayMesh(v.astype(dtype) if name != "mixed" else v, faces)
    tri, t = rm.first_hit(o, d)
    vr = v.astype(dtype).astype(np.float64) if name != "mixed" else v
    rtri, rt = R.first_hit(o, d, vr, f)
    assert (rtri >= 0).sum() > len(o) // 3  # most rays hit
    assert_same(tri, t, rtri, rt)
    # intersects_first is the same call's index
    assert torch.equal(rm.intersects_first(torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)), tri)


def test_empty_inputs(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = icosphere(2)
    rm = RayMesh(v, f)
    tri, t = rm.first_hit(np.zeros((0, 3)), np.zeros((0, 3)))
    assert tri.shape == (0,) and t.shape == (0,)
    loc, ir, it = rm.intersects_location(np.zeros((0, 3)), np.zeros((0, 3)))
    assert loc.shape == (0, 3) and ir.shape == (0,) and it.shape == (0,)
    empty = RayMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    tri, t = empty.first_hit(np.zeros((5, 3)), np.ones((5, 3)))
    assert tri.tolist() == [-1] * 5 and torch.isinf(t).all()
    one = RayMesh(np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.]]), np.array([[0, 1, 2]]))
    tri, t = one.first_hit(np.array([[0.25, 0.25, 1.0], [2, 2, 1]]), np.array([[0, 0, -1.0], [0, 0, -1]]))
    assert tri.tolist() == [0, -1] and t.tolist()[0] == 1.0


def test_watertight_icosphere(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = icosphere(5, center=(0.3, -0.2, 0.1), radius=2.0)
    rm = RayMesh(v, f)
    rng = np.random.default_rng(5)
    n = 1 << 20
    u = rng.standard_normal((n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = np.array([0.3, -0.2, 0.1]) + 5.0 * u
    # aim at points in the plane through the centre perpendicular to the ray, strictly inside the inscribed radius of the
    # polyhedron (every face's distance from the centre is > 0.99 radius at level 5)
    p = rng.standard_normal((n, 3))
    p -= (p * u).sum(1, keepdims=True) * u
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    p *= 2.0 * 0.98 * np.sqrt(rng.random((n, 1)))
    tri = rm.intersects_first(o, (np.array([0.3, -0.2, 0.1]) + p) - o)
    assert int((tri < 0).sum()) == 0


def test_two_million_triangles_sample(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = heightfield(1000, 1000, seed=3, size=100.0)
    assert len(f) == 2_000_000
    rm = RayMesh(v, f)
    rng = np.random.default_rng(7)
    n = 256
    # 128 camera-like rays from above, 64 grazing rays nearly parallel to the terrain (they skim many boxes' faces), 64 rays
    # along grid lines at a cell boundary height (origins on box faces)
    o1 = np.concatenate([rng.uniform(0, 100, (128, 2)), np.full((128, 1), 20.0)], 1)
    d1 = np.concatenate([rng.uniform(-0.5, 0.5, (128, 2)), -np.ones((128, 1))], 1)
    o2 = np.concatenate([np.zeros((64, 1)), rng.uniform(0, 100, (64, 1)), rng.uniform(-0.3, 0.4, (64, 1))], 1)
    d2 = np.concatenate([np.ones((64, 1)), rng.uniform(-0.01, 0.01, (64, 1)), rng.uniform(-1e-3, 1e-3, (64, 1))], 1)
    gx = rng.integers(0, 1001, 64) * 0.1
    o3 = np.stack([gx, np.full(64, -1.0), np.full(64, 0.0)], 1)
    d3 = np.stack([np.zeros(64), np.ones(64), rng.uniform(-1e-4, 1e-4, 64)], 1)
    o, d = np.concatenate([o1, o2, o3]), np.concatenate([d1, d2, d3])
    assert len(o) == n
    tri, t = rm.first_hit(o, d)
    tris = torch.from_numpy(R.triangles(v, f)).to(dev)
    ok = torch.from_numpy(R.valid(R.triangles(v, f))).to(dev)
    rtri, rt = R.first_hit_torch(o, d, tris, ok)
    assert_same(tri, t, rtri.cpu().numpy(), rt.cpu().numpy())
    # the torch mirror is the numpy restatement: check it on a slice where numpy is affordable
    sub = slice(0, 20000)
    ntri, nt = R.first_hit(o[:16], d[:16], v, f[sub])
    ttri, tt = R.first_hit_torch(o[:16], d[:16], tris[sub], ok[sub])
    assert np.array_equal(ttri.cpu().numpy(), ntri) and np.array_equal(tt.cpu().numpy().view(np.int64), nt.view(np.int64))


def test_deterministic_across_runs_and_streams(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = scene_mixed()
    rm = RayMesh(v, f)
    o, d = rays_for(v, f, 200000, seed=11)
    o, d = torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)
    a = rm.first_hit(o, d)
    b = rm.first_hit(o, d)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        c = rm.first_hit(o, d)
        rm2 = RayMesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
        e = rm2.first_hit(o, d)
    torch.cuda.synchronize(dev)
    for x in (b, c, e):
        assert torch.equal(a[0], x[0]) and torch.equal(a[1].view(torch.int64), x[1].view(torch.int64))
    assert torch.equal(rm.bvh, rm2.bvh)


def test_intersects_location(dev):
    from autovfx_b200.raycast import RayMesh
    v, f = icosphere(5)
    o, d = rays_for(v, f, 1500, seed=3)
    o32, d32 = o.astype(np.float32), d.astype(np.float32)
    rm = RayMesh(v, f)
    loc, ir, it = rm.intersects_location(o32, d32)
    rtri, rt = R.first_hit(o32, d32, v, f)
    rloc, rir, rit = R.locations(o32, d32, rtri, rt)
    assert ir.dtype == torch.int64 and it.dtype == torch.int64 and loc.dtype == torch.float64
    assert np.array_equal(ir.cpu().numpy(), rir) and np.array_equal(it.cpu().numpy(), rit)
    assert np.array_equal(loc.cpu().numpy().view(np.int64), rloc.view(np.int64))
    with pytest.raises(ValueError, match="multiple_hits"):
        rm.intersects_location(o, d, multiple_hits=True)


def _camera(eye, target, H, W, focal):
    """c2w (float32, OpenCV axes as get_ray_directions) looking from eye at target, K, and the view's rays as the reference makes
    them: directions @ c2w[:3, :3].T, origins c2w[:3, 3]."""
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0, 0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, :3] = np.stack([right, down, fwd], 1)
    c2w[:3, 3] = eye
    K = np.array([[focal, 0, W / 2], [0, focal, H / 2], [0, 0, 1]], np.float32)
    j, i = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    dirs = np.stack([(i - K[0, 2]) / K[0, 0], (j - K[1, 2]) / K[1, 1], np.ones_like(i)], -1)
    c2w_t = torch.from_numpy(c2w).cuda()
    rays_d = torch.from_numpy(dirs).cuda() @ c2w_t[:3, :3].T
    rays_o = c2w_t[:3, 3].expand_as(rays_d)
    return c2w_t, K, rays_o, rays_d


def test_vote_loop_counters(dev):
    """extract_object.py:137-159 on device tensors with index_tri from intersects_first, against the same lines on the oracle's
    index_tri, as the same integers."""
    from autovfx_b200.raycast import RayMesh
    hv, hf = heightfield(60, 60, seed=4)
    sv, sf = icosphere(3, center=(5, 5, 1.0), radius=0.8)
    v, f = np.concatenate([hv, sv]), np.concatenate([hf, sf + len(hv)])
    rm = RayMesh(v, f)
    centers = torch.Tensor(R.triangles(v, f).mean(axis=1)).to(dev)  # trimesh's triangles_center
    H, W = 48, 64

    def loop(cast):
        counter = torch.zeros(len(f), dtype=torch.int32, device=dev)
        naive = torch.zeros(len(f), dtype=torch.int32, device=dev)
        for k in range(6):
            ang = k * np.pi / 3
            eye = np.array([5 + 4 * np.cos(ang), 5 + 4 * np.sin(ang), 3.5])
            c2w, K, rays_o, rays_d = _camera(eye, (5, 5, 1.0), H, W, 60.0)
            # the object mask: pixels whose ray hits the sphere (rendered from the mesh), with a border of background pixels
            hit = rm.intersects_first(rays_o.reshape(-1, 3), rays_d.reshape(-1, 3)).reshape(H, W)
            mask = (hit >= len(hf))
            mask = mask | torch.roll(mask, 2, 1)
            o_m, d_m = rays_o[mask].reshape(-1, 3), rays_d[mask].reshape(-1, 3)
            index_tri = cast(o_m, d_m)
            naive[index_tri] += 1
            w2c = torch.inverse(c2w)
            xyz = centers[index_tri]
            xyz = torch.cat([xyz, torch.ones(xyz.size(0), 1, device=dev)], dim=1)
            xyz = torch.matmul(xyz, w2c.T)
            xyz = xyz[:, :3]
            xyz = xyz / xyz[:, 2].unsqueeze(1)
            uv = torch.matmul(xyz, torch.FloatTensor(K).to(dev).T)
            uv = uv[:, :2].round().long()
            valid_uv = (uv[:, 0] >= 0) & (uv[:, 0] < W) & (uv[:, 1] >= 0) & (uv[:, 1] < H)
            filtered = uv[valid_uv]
            in_mask_indices = torch.where(mask[filtered[:, 1], filtered[:, 0]])[0]
            in_mask = valid_uv.nonzero().flatten()[in_mask_indices]
            counter[index_tri[in_mask]] += 1
        return counter, naive

    ours = loop(lambda o, d: rm.intersects_first(o, d))
    ref = loop(lambda o, d: torch.tensor(R.first_hit(o.cpu().numpy(), d.cpu().numpy(), v, f)[0], dtype=torch.int32, device=dev))
    assert int(ours[1].sum()) > 0 and int(ours[0].sum()) > 0
    assert torch.equal(ours[0], ref[0]) and torch.equal(ours[1], ref[1])


def test_inpaint_masks(dev):
    from autovfx_b200.raycast import RayMesh, inpaint_mask
    pv, pf = heightfield(40, 40, seed=6)
    pv[:, 2] = 0.0  # the planar mesh
    sv, sf = icosphere(3, center=(5, 5, 0.5), radius=1.0)
    cv, cf = np.concatenate([pv + [0, 0, 0.004], sv]), np.concatenate([pf, sf + len(pv)])  # inpainted scene: a plane 4 mm above
    planar, combined = RayMesh(pv, pf), RayMesh(cv, cf)
    H, W = 40, 56
    views = [((5, -3, 4), (5, 5, 0)), ((12, 5, 3), (5, 5, 0)), ((5, 4, 6), (5, 5, 0)), ((50, 50, 3), (80, 80, 3))]
    nones = 0
    for eye, target in views:
        c2w, K, rays_o, rays_d = _camera(np.array(eye, np.float64), target, H, W, 50.0)
        w2c = torch.inverse(c2w)
        m = inpaint_mask(planar, combined, rays_o, rays_d, w2c)
        ref = R.inpaint_mask(rays_o.cpu().numpy(), rays_d.cpu().numpy(), (pv, pf), (cv, cf), w2c.cpu().numpy())
        if ref is None:
            nones += 1
            assert m is None
            continue
        assert m is not None and m.dtype == torch.uint8 and tuple(m.shape) == (H, W)
        assert np.array_equal(m.cpu().numpy(), ref)
        assert 0 < int((m == 255).sum()) < H * W
    assert nones == 1
    # no combined hit: a combined mesh away from every ray
    far = RayMesh(pv + [500, 0, 0], pf)
    c2w, K, rays_o, rays_d = _camera(np.array([5, -3, 4.0]), (5, 5, 0), H, W, 50.0)
    assert inpaint_mask(planar, far, rays_o, rays_d, torch.inverse(c2w)) is None
    assert R.inpaint_mask(rays_o.cpu().numpy(), rays_d.cpu().numpy(), (pv, pf), (pv + [500, 0, 0], pf), torch.inverse(c2w).cpu().numpy()) is None
