"""Closest-triangle queries without a GPU: the numpy restatement of Ericson's closest-point test (tests/closest_ref.py) against
hand-derived distances and exact rational arithmetic, its tie and validity rules, the library's new exports, and the argument
checks of RayMesh.closest, compute_closest_points and ResidentScene's melting frames."""
import os
import sys
from fractions import Fraction

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from autovfx_b200 import _lib  # noqa: E402
from autovfx_b200 import edit, raycast  # noqa: E402
from tests import closest_ref as R  # noqa: E402

UNIT_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float64)
UNIT_F = np.array([[0, 1, 2]], np.int64)


def query(p, v=UNIT_V, f=UNIT_F):
    tri, d2 = R.closest(np.array(p, np.float64).reshape(1, 3), v, f)
    return int(tri[0]), float(d2[0])


# the seven Voronoi regions of the unit triangle a = (0,0,0), b = (1,0,0), c = (0,1,0), from above (h = 0.5) and below (h = -2):
# (xy of the point, closest point's xy, squared distance in the plane)
REGIONS = {
    "vertex_a": ((-1, -1), 2.0), "vertex_b": ((2, -1), 2.0), "vertex_c": ((-1, 2), 2.0),
    "edge_ab": ((0.5, -1), 1.0), "edge_ac": ((-1, 0.5), 1.0), "edge_bc": ((1, 1), 0.5), "face": ((0.25, 0.25), 0.0),
}


@pytest.mark.parametrize("h", [0.5, -2.0, 0.0], ids=["above", "below", "in_plane"])
@pytest.mark.parametrize("region", list(REGIONS))
def test_voronoi_regions(region, h):
    (x, y), planar = REGIONS[region]
    assert query((x, y, h)) == (0, planar + h * h)


@pytest.mark.parametrize("p", [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0.5, 0, 0), (0, 0.5, 0), (0.5, 0.5, 0), (0.25, 0.5, 0)],
                         ids=["v0", "v1", "v2", "edge_ab", "edge_ac", "edge_bc", "interior"])
def test_points_on_the_triangle(p):
    assert query(p) == (0, 0.0)


def _exact_d2(p, t):
    """Squared distance to the closest point in exact rational arithmetic (Ericson's regions are exact there)."""
    p = [Fraction(x) for x in p]
    a, b, c = ([Fraction(x) for x in t[k]] for k in range(3))

    def sub(u, w):
        return [u[k] - w[k] for k in range(3)]

    def dot(u, w):
        return sum(u[k] * w[k] for k in range(3))
    ab, ac, ap, bp, cp = sub(b, a), sub(c, a), sub(p, a), sub(p, b), sub(p, c)
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    if d1 <= 0 and d2 <= 0:
        q = a
    elif d3 >= 0 and d4 <= d3:
        q = b
    elif vc <= 0 and d1 >= 0 and d3 <= 0:
        q = [a[k] + d1 / (d1 - d3) * ab[k] for k in range(3)]
    elif d6 >= 0 and d5 <= d6:
        q = c
    elif vb <= 0 and d2 >= 0 and d6 <= 0:
        q = [a[k] + d2 / (d2 - d6) * ac[k] for k in range(3)]
    elif va <= 0 and d4 - d3 >= 0 and d5 - d6 >= 0:
        w = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        q = [b[k] + w * (c[k] - b[k]) for k in range(3)]
    else:
        den = va + vb + vc
        q = [a[k] + vb / den * ab[k] + vc / den * ac[k] for k in range(3)]
    e = sub(p, q)
    return dot(e, e)


def test_against_exact_rationals():
    """|d2 - exact| <= 2^-40 (exact + S^2), S = |p|_inf + the largest |vertex coordinate|: the closest point carries a few
    float64 roundings of magnitude S, the squares a few more of d2."""
    rng = np.random.default_rng(0)
    tris = rng.uniform(-1, 1, (40, 3, 3))
    pts = np.concatenate([rng.uniform(-2, 2, (200, 3)), (tris[np.arange(100) % 40] * rng.dirichlet([1, 1, 1], 100)[:, :, None]).sum(1)
                          + 1e-3 * rng.standard_normal((100, 3))])
    dd = R.closest_d2(pts, tris)
    worst = 0.0
    for i in range(len(pts)):
        for j in range(0, len(tris), 7):
            ex = _exact_d2(pts[i], tris[j])
            S = Fraction(np.abs(pts[i]).max() + np.abs(tris[j]).max())
            err = abs(Fraction(dd[i, j]) - ex) / (ex + S * S)
            worst = max(worst, float(err))
    assert worst <= 2.0 ** -40, worst


def test_ties_go_to_the_lower_index():
    # two triangles sharing the edge y = z = 0 on either side: the point above the edge is at d2 = 1 from both
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, -1, 0]], np.float64)
    f = np.array([[0, 1, 2], [0, 1, 3]])
    assert query((0.5, 0, 1), v, f) == (0, 1.0)
    assert query((0.5, 0, 1), v, f[::-1]) == (0, 1.0)
    # a duplicated triangle behind a farther one
    v2 = np.concatenate([UNIT_V + [0, 0, 5], UNIT_V])
    assert query((0.25, 0.25, 1), v2, np.array([[0, 1, 2], [3, 4, 5], [3, 4, 5]])) == (1, 1.0)
    # the bisector plane of two parallel triangles
    v3 = np.concatenate([UNIT_V + [0, 0, 1], UNIT_V + [0, 0, -1]])
    assert query((0.2, 0.3, 0), v3, np.array([[3, 4, 5], [0, 1, 2]])) == (0, 1.0)


@pytest.mark.parametrize("tri", [[(0, 0, 0), (1, 1, 1), (2, 2, 2)], [(0, 0, 0), (1, 0, 0), (1, 0, 0)], [(0.5, 0.5, 0)] * 3],
                         ids=["collinear", "repeated_vertex", "point"])
def test_degenerate_never_wins(tri):
    v = np.concatenate([np.array(tri, np.float64), UNIT_V + [0, 0, 3]])
    f = np.array([[0, 1, 2], [3, 4, 5]])
    assert not R.valid(R.triangles(v, f))[0]
    assert query((0.5, 0.5, 0), v, f) == (1, 9.0)
    assert query((0.5, 0.5, 0), v, f[:1]) == (-1, np.inf)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_triangles_and_points(bad):
    v = np.concatenate([UNIT_V, UNIT_V + [0, 0, 2]])
    v[1, 0] = bad
    assert query((0.1, 0.1, 0), v, np.array([[0, 1, 2], [3, 4, 5]])) == (1, 4.0)
    assert query((bad, 0.25, 1)) == (-1, np.inf)
    assert query((0.25, 0.25, bad)) == (-1, np.inf)


def test_empty_mesh():
    tri, d2 = R.closest(np.ones((3, 3)), np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    assert tri.tolist() == [-1] * 3 and np.isinf(d2).all()
    tri, d2 = R.closest(np.zeros((0, 3)), UNIT_V, UNIT_F)
    assert tri.shape == (0,) and d2.shape == (0,)


def test_exports_of_the_built_library():
    for name in ("gsr_mesh_closest_bytes", "gsr_mesh_closest", "gsr_mesh_isin_rows_bytes", "gsr_mesh_isin_rows"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
    L = _lib.lib
    assert L.gsr_mesh_isin_rows_bytes(-1, 0) == 0 and L.gsr_mesh_isin_rows_bytes(0, -1) == 0
    assert L.gsr_mesh_isin_rows_bytes(3_000_000, 1000) >= 1000 + 4 * (3_000_000 // 1024)
    # argument errors are reported before anything is enqueued
    assert L.gsr_mesh_closest_bytes(-1) == 0 and L.gsr_mesh_closest_bytes(2 ** 31) == 0
    assert L.gsr_mesh_closest_bytes(3_000_000) >= 16 * 3_000_000
    assert L.gsr_mesh_closest(0, None, 1, None, 0, None, None, None, 0, None) == -1
    assert L.gsr_mesh_closest(0, 256, 1, 256, 2, 256, None, 256, 1 << 20, None) == -1
    assert L.gsr_mesh_closest(-1, 256, 0, None, 0, None, None, 256, 1 << 20, None) == -1
    assert L.gsr_mesh_closest(0, 256, 1, 256, 0, 256, None, None, 0, None) == -2
    assert L.gsr_mesh_isin_rows(-1, None, 0, None, 0, 0, None, None, None, 256, 256, 256, None) == -1
    assert L.gsr_mesh_isin_rows(0, None, 0, None, 0, 9, None, None, None, 256, 256, 256, None) == -1
    assert L.gsr_mesh_isin_rows(0, None, 0, None, 0, 0, None, None, None, None, 256, 256, None) == -1


def _stub_mesh():
    """A RayMesh without a device build: enough for the checks that run before anything is uploaded."""
    rm = object.__new__(raycast.RayMesh)
    rm.device, rm.V, rm.F = torch.device("cuda", 0), 3, 1
    return rm


@pytest.mark.parametrize("method", ["closest", "compute_closest_points"])
def test_closest_argument_validation(method):
    fn = getattr(_stub_mesh(), method)
    with pytest.raises(ValueError, match="points"):
        fn(np.zeros((4, 2)))
    with pytest.raises(ValueError, match="points"):
        fn(np.zeros((4,)))
    with pytest.raises(ValueError, match="points"):
        fn(np.array([["a", "b", "c"]]))
    with pytest.raises(ValueError, match="points"):
        fn(np.zeros((2, 3), bool))
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(torch.zeros((4, 3)))


def _raw(n, M):
    rng = np.random.default_rng(n)
    return {"xyz": rng.standard_normal((n, 3)).astype(np.float32), "f_dc": np.zeros((n, 1, 3), np.float32),
            "f_rest": np.zeros((n, M - 1, 3), np.float32), "opacity": np.zeros((n, 1), np.float32),
            "scaling": np.zeros((n, 3), np.float32), "rotation": np.ones((n, 4), np.float32)}


def test_resident_scene_melting_arguments():
    scene = _raw(8, 4)
    with pytest.raises(ValueError, match="SH coefficients"):
        edit.ResidentScene(scene, device="cuda:0", melting={"obj": (_raw(5, 1), _stub_mesh())})
    with pytest.raises(ValueError, match="RayMesh"):
        edit.ResidentScene(scene, device="cuda:0", melting={"obj": (_raw(5, 4), None)})
    with pytest.raises(ValueError, match="pair"):
        edit.ResidentScene(scene, device="cuda:0", melting={"obj": _raw(5, 4)})
    # compose's checks run before any device work: a scene object with a rigid and a melting object, no arrays
    rs = object.__new__(edit.ResidentScene)
    rs.P_scene, rs.objects, rs.melting_objects = 8, {"rigid": None}, {"obj": None}
    with pytest.raises(ValueError, match="exclusive"):
        rs.compose({"rigid": (np.zeros(3), np.eye(3), 1.0, np.zeros(3))}, melting={"obj": []})
    with pytest.raises(KeyError, match="unknown melting object"):
        rs.compose(melting={"other": [np.zeros((1, 3))]})
    with pytest.raises(ValueError, match="at most 2"):
        rs.compose(melting={"obj": [np.zeros((1, 3))] * 3})
