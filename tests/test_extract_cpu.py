"""MaskScorer without a GPU: the threshold semantics against numpy, the view/mask pairing of extract_object's loop, argument
validation and the library's new exports."""
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from autovfx_b200 import extract  # noqa: E402
from autovfx_b200 import scene  # noqa: E402
from tests import extract_ref as X  # noqa: E402


def test_threshold_is_float32_as_numpy_compares():
    t = extract.ALPHA_THRESHOLD
    assert t.dtype == np.float32 and t == np.float32(0.8)
    below, above = np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))
    alpha = np.array([below, t, above, np.nan, np.inf, -np.inf], np.float32)
    # the reference's `object_alpha_image >= 0.8` on a float32 image (NumPy >= 2, NEP 50: the Python float is weak)
    assert (alpha >= 0.8).tolist() == [False, True, True, False, True, False]
    # the kernel's float32 comparison; float(0.8) itself lies below float32(0.8), so a float64 comparison would admit `below`
    assert float(below) < 0.8 < float(t)
    assert [bool(a >= t) for a in alpha] == (alpha >= 0.8).tolist()
    # the value handed to the C call is float32(0.8) exactly
    assert np.float32(float(t)) == t


def test_tracked_views_pair_by_file_name():
    views = ["v%d" % i for i in range(12)]
    masks = {"00000.png": "m0", "00003.png": "m3", "00011.png": "m11", "00012.png": "past the end", "3.png": "unpadded",
             "00005.jpg": "other suffix"}
    assert extract.tracked_views(views, masks) == [(0, "v0", "m0"), (3, "v3", "m3"), (11, "v11", "m11")]
    assert extract.tracked_views(views, {}) == []


def _cpu_scene(P=64):
    g = scene.synthetic_gaussians(P, seed=2)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 40, 30, 60.0)
    return X.model_from(g, "cpu"), [X.render_camera(cam, "cpu"), X.render_camera(cam, "cpu")]


def test_validation_names_the_argument():
    pc, views = _cpu_scene()
    ok = np.zeros((30, 40), np.uint8)
    with pytest.raises(ValueError, match=r"obj_masks\['00001.png'\] has shape \(40, 30\)"):
        extract.MaskScorer(pc, views, {"00000.png": ok, "00001.png": np.zeros((40, 30), np.uint8)})
    with pytest.raises(ValueError, match=r"obj_masks\['00000.png'\] must be uint8"):
        extract.MaskScorer(pc, views, {"00000.png": ok.astype(bool)})
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=True, convert_SHs_python=False)
    with pytest.raises(ValueError, match="pipe.compute_cov3D_python"):
        extract.MaskScorer(pc, views, {"00000.png": ok}, pipe)
    # a mask for a view that does not exist is never read, whatever its shape (the loop never looks it up)
    with pytest.raises(RuntimeError, match="CUDA"):
        extract.MaskScorer(pc, views, {"00000.png": ok, "00009.png": np.zeros((1, 1), np.uint8)})


def test_cpu_tensors_raise_runtime_error():
    pc, views = _cpu_scene()
    with pytest.raises(RuntimeError, match="CUDA"):
        extract.MaskScorer(pc, views, {"00001.png": torch.zeros((30, 40), dtype=torch.uint8)}, X.PIPE)


def test_new_symbols_are_exported():
    from autovfx_b200 import _lib
    for name in ("gsr_select_rows_bytes", "gsr_select_rows", "gsr_pack_masks", "gsr_mask_disagreement"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
    tiles = -(-3_000_000 // 1024)
    assert _lib.lib.gsr_select_rows_bytes(3_000_000) == 4 * (tiles + 1)
    assert _lib.lib.gsr_select_rows_bytes(0) == 4 and _lib.lib.gsr_select_rows_bytes(-1) == 0
    assert set(extract.__all__) == {"MaskScorer", "ALPHA_THRESHOLD", "tracked_views"}
