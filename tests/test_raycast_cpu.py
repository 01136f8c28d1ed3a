"""Mesh ray casts without a GPU: the numpy restatement of the watertight test (tests/raycast_ref.py) against hand-derived hits,
RayMesh's argument validation, and the library's new exports."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from autovfx_b200 import _lib  # noqa: E402
from autovfx_b200 import raycast  # noqa: E402
from tests import raycast_ref as R  # noqa: E402

UNIT_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float64)
UNIT_F = np.array([[0, 1, 2]], np.int64)


def cast(o, d, v=UNIT_V, f=UNIT_F):
    tri, t = R.first_hit(np.array(o, np.float64).reshape(1, 3), np.array(d, np.float64).reshape(1, 3), v, f)
    return int(tri[0]), float(t[0])


@pytest.mark.parametrize("o", [(0.25, 0.25, 1.0), (0.5, 0.0, 1.0), (0.0, 0.5, 1.0), (0.5, 0.5, 1.0)], ids=["interior", "edge_y0", "edge_x0", "hypotenuse"])
def test_hits_interior_and_edges(o):
    assert cast(o, (0, 0, -1)) == (0, 1.0)


@pytest.mark.parametrize("o", [(0, 0, 1), (1, 0, 1), (0, 1, 1)], ids=["v0", "v1", "v2"])
def test_hits_vertices(o):
    assert cast(o, (0, 0, -1)) == (0, 1.0)


def test_both_faces_and_unnormalised_direction():
    assert cast((0.25, 0.25, -1), (0, 0, 1)) == (0, 1.0)   # from behind
    assert cast((0.25, 0.25, 1), (0, 0, -2)) == (0, 0.5)   # t in units of the direction as given
    assert cast((0.25, 0.25, 3), (0, 0, -0.5)) == (0, 6.0)


def test_oblique_ray_t():
    # from (0, 0, 1) towards (0.25, 0.25, 0): d = (0.25, 0.25, -1), t = 1
    assert cast((0, 0, 1), (0.25, 0.25, -1)) == (0, 1.0)


def test_misses():
    assert cast((0.25, 0.25, 0), (0, 0, -1))[0] == -1     # t = 0 does not count
    assert cast((0.25, 0.25, 0), (0, 0, 1))[0] == -1
    assert cast((0.25, 0.25, 1), (0, 0, 1))[0] == -1      # t < 0
    assert cast((0.25, 0.25, 1), (1, 0, 0))[0] == -1      # parallel to the plane
    assert cast((-1, 0.25, 0), (1, 0, 0))[0] == -1        # in the plane: det = 0
    assert cast((1.01, 0.5, 1), (0, 0, -1))[0] == -1      # outside
    assert cast((0.6, 0.6, 1), (0, 0, -1))[0] == -1       # beyond the hypotenuse


@pytest.mark.parametrize("tri", [[(0, 0, 0), (1, 1, 1), (2, 2, 2)], [(0, 0, 0), (1, 0, 0), (1, 0, 0)], [(0.5, 0.5, 0)] * 3],
                         ids=["collinear", "repeated_vertex", "point"])
def test_degenerate_never_hit(tri):
    v = np.array(tri, np.float64)
    assert not R.valid(v[None])[0]
    for o, d in [((0.5, 0.5, 1), (0, 0, -1)), ((1, 0, 1), (0, 0, -1)), ((-1, -1, -1), (1, 1, 1)), ((1, 1, 0), (0, 0, 1))]:
        assert cast(o, d, v, UNIT_F)[0] == -1


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_triangle_and_rays(bad):
    v = UNIT_V.copy()
    v[1, 0] = bad
    assert cast((0.1, 0.1, 1), (0, 0, -1), v)[0] == -1
    assert cast((bad, 0.25, 1), (0, 0, -1))[0] == -1
    assert cast((0.25, 0.25, 1), (0, bad, -1))[0] == -1
    assert cast((0.25, 0.25, 1), (0, 0, 0))[0] == -1


def test_ties_go_to_the_lower_index():
    v = np.concatenate([UNIT_V, UNIT_V, UNIT_V + [0, 0, -1]])
    f = np.array([[6, 7, 8], [3, 4, 5], [0, 1, 2]])
    # faces 1 and 2 are the same triangle at t = 1; face 0 is behind them
    assert cast((0.25, 0.25, 1), (0, 0, -1), v, f) == (1, 1.0)
    # a shared edge: the ray through x + y = 1 of two triangles meeting there reports the lower index
    v2 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], np.float64)
    f2 = np.array([[1, 3, 2], [0, 1, 2]])
    assert cast((0.5, 0.5, 1), (0, 0, -1), v2, f2) == (0, 1.0)
    assert cast((0.5, 0.5, 1), (0, 0, -1), v2, f2[::-1]) == (0, 1.0)


def test_axis_choice_and_swap():
    ok, kx, ky, kz, Sx, Sy, Sz = R.ray_setup(np.zeros((4, 3)), np.array([[1, 1, 1], [0, -2, 1], [0, 0, -3], [0, 0, 0.]]))
    assert kz.tolist()[:3] == [0, 1, 2] and ok.tolist() == [True, True, True, False]
    assert (kx[1], ky[1]) == (0, 2)  # d[kz] < 0 swaps kx and ky
    assert (kx[2], ky[2]) == (1, 0)
    assert Sz[2] == 1 / -3.0


def test_locations_and_inpaint_restatement():
    o = np.array([[0.25, 0.25, 1], [5, 5, 1], [0.1, 0.2, 2]])
    d = np.array([[0, 0, -1], [0, 0, -1], [0, 0, -1.]])
    tri, t = R.first_hit(o, d, UNIT_V, UNIT_F)
    loc, ir, it = R.locations(o, d, tri, t)
    assert ir.tolist() == [0, 2] and it.tolist() == [0, 0]
    assert np.array_equal(loc, [[0.25, 0.25, 0], [0.1, 0.2, 0]])
    w2c = np.eye(4)
    w2c[2, 3] = 2.0
    # planar = the unit triangle; combined = the unit triangle and a blocker above ray 2
    block_v = np.concatenate([UNIT_V, [[0, 0, 1.5], [1, 0, 1.5], [0, 1, 1.5]]])
    block_f = np.array([[0, 1, 2], [3, 4, 5]])
    m = R.inpaint_mask(o.reshape(3, 1, 3), d.reshape(3, 1, 3), (UNIT_V, UNIT_F), (block_v, block_f), w2c)
    assert m.shape == (3, 1)
    # ray 0 starts below the blocker (z = 1 < 1.5): it reaches the planar triangle; ray 2 starts above and is blocked
    assert m[:, 0].tolist() == [255, 0, 0]
    assert R.inpaint_mask(o[1:2], d[1:2], (UNIT_V, UNIT_F), (block_v, block_f), w2c) is None  # no planar hit
    far = (UNIT_V + [10, 10, 0], UNIT_F)
    assert R.inpaint_mask(o, d, (UNIT_V, UNIT_F), far, w2c) is None  # no combined hit


def test_exports_of_the_built_library():
    for name in ("gsr_mesh_bvh_bytes", "gsr_mesh_build_bytes", "gsr_mesh_build", "gsr_mesh_first_hit", "gsr_mesh_inpaint_mask"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
    L = _lib.lib
    assert L.gsr_mesh_bvh_bytes(-1) == 0 and L.gsr_mesh_build_bytes(-1) == 0
    assert L.gsr_mesh_bvh_bytes(0) > 0
    assert L.gsr_mesh_bvh_bytes(1000) >= 64 * 999 + 72 * 1000 + 4 * 1000
    # argument errors are reported before anything is enqueued
    assert L.gsr_mesh_build(-1, 0, None, None, None, 0, None, 0, None) == -1
    assert L.gsr_mesh_first_hit(0, None, 1, None, None, 0, None, None, None, None) == -1
    assert L.gsr_mesh_first_hit(0, 256, 1, 256, 256, 2, None, 256, None, None) == -1
    assert L.gsr_mesh_inpaint_mask(-1, None, None, 0, None, None, None, None, None, None, None, None) == -1


def _expect(exc, match, *args, **kw):
    with pytest.raises(exc, match=match):
        raycast.RayMesh(*args, **kw)


def test_raymesh_argument_validation():
    v, f = UNIT_V, UNIT_F
    _expect(ValueError, "vertices", v[:, :2], f)
    _expect(ValueError, "vertices", v.astype(np.int64), f)
    _expect(ValueError, "faces", v, f.astype(np.float64))
    _expect(ValueError, "faces", v, f[:, :2])
    _expect(ValueError, "faces", v, f.astype(np.int16))
    _expect(ValueError, "faces", v, np.array([[0, 1, 3]]))
    _expect(ValueError, "faces", v, np.array([[0, -1, 2]]))
    _expect(ValueError, "vertices", np.array(["a", "b", "c"]), f)
    _expect(RuntimeError, "CUDA", torch.from_numpy(v), f)
    _expect(RuntimeError, "CUDA", v, torch.from_numpy(f))


def test_inpaint_mask_needs_raymeshes():
    with pytest.raises(ValueError, match="RayMesh"):
        raycast.inpaint_mask(None, None, np.zeros((1, 3)), np.zeros((1, 3)), np.eye(4))
