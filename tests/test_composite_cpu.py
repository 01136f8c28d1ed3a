"""CPU checks of frame compositing (autovfx_b200.composite): the exports, every argument error of composite_frame, and the numpy
restatement of tests/composite_ref.py against the reference's own blend_frames (when build() staged it) and its golden frames."""
from __future__ import annotations

import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import composite_ref as CR  # noqa: E402


def test_exports():
    from autovfx_b200 import composite, _lib
    assert composite.__all__ == ["composite_frame", "percentile_low", "blend_frames"]
    assert hasattr(_lib.lib, "gsr_composite") and hasattr(_lib.lib, "gsr_percentile_low")
    hdr = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    assert "#define GSR_PERCENTILE_BYTES %d" % composite.PERCENTILE_BYTES in hdr


def _layers(H=3, W=5, device="cpu", **over):
    c4 = lambda: torch.zeros((H, W, 4), dtype=torch.uint8, device=device)  # noqa: E731
    d2 = lambda: torch.zeros((H, W), dtype=torch.float32, device=device)  # noqa: E731
    a = {"rgba8": c4(), "depth": d2(), "obj": c4(), "obj_depth": d2(), "shadow": c4(), "shadow_depth": d2(), "all_": c4()}
    a.update(over)
    return a


@pytest.mark.parametrize("over,name", [
    ({"obj": torch.zeros((3, 5, 4), dtype=torch.float32)}, "obj"),
    ({"depth": torch.zeros((3, 5), dtype=torch.float64)}, "depth"),
    ({"shadow": torch.zeros((3, 5, 3), dtype=torch.uint8)}, "shadow"),
    ({"all_": torch.zeros((3, 6, 4), dtype=torch.uint8)}, "all_"),
    ({"obj_depth": torch.zeros((4, 5), dtype=torch.float32)}, "obj_depth"),
    ({"shadow_depth": torch.zeros((5, 3), dtype=torch.float32).t()}, "shadow_depth"),
    ({"obj3dgs": torch.zeros((3, 5, 4), dtype=torch.uint8)}, "obj3dgs"),
    ({"obj3dgs_depth": torch.zeros((3, 5), dtype=torch.float32)}, "obj3dgs_depth"),
    ({"smoke": torch.zeros((3, 5, 4), dtype=torch.uint8)}, "smoke"),
    ({"smoke_depth": torch.zeros((3, 5), dtype=torch.float32)}, "smoke_depth"),
    ({"fire": torch.zeros((3, 5, 4), dtype=torch.uint8)}, "fire"),
    ({"smoke": torch.zeros((3, 5, 4), dtype=torch.uint8), "smoke_depth": torch.zeros((2, 5), dtype=torch.float32)}, "smoke_depth"),
    ({"out": torch.zeros((3, 5, 4), dtype=torch.int32)}, "out"),
    ({"rgba8": torch.zeros((3, 5, 3), dtype=torch.uint8)}, "rgba8"),
    ({"rgba8": torch.zeros((0, 5, 4), dtype=torch.uint8)}, "rgba8"),
    ({"obj": torch.zeros((3, 5, 4), dtype=torch.uint8, device="meta")}, "obj"),
])
def test_argument_errors_name_the_argument(over, name):
    from autovfx_b200.composite import composite_frame
    with pytest.raises(ValueError, match=r"\b%s\b" % name):
        composite_frame(**_layers(**over))


def test_cpu_tensors_raise_runtime_error():
    from autovfx_b200.composite import composite_frame, percentile_low
    with pytest.raises(RuntimeError, match="CUDA"):
        composite_frame(**_layers())
    with pytest.raises(RuntimeError, match="CUDA"):
        percentile_low(torch.zeros(4))
    with pytest.raises(ValueError):
        percentile_low(torch.zeros(0))


def test_drop_in_needs_installing():
    from autovfx_b200 import composite
    with pytest.raises(RuntimeError, match="blend_frames"):
        composite.blend_frames("/nonexistent/a/b", None)


def test_numpy_cast_of_nan_on_this_host_is_zero():
    # the kernels write 0 for a NaN pixel (none can arise from byte inputs), as numpy's clip + astype(uint8) does on x86
    with np.errstate(invalid="ignore"):
        assert np.clip(np.float32([np.nan]), 0, 255).astype(np.uint8)[0] == 0


@pytest.mark.parametrize("name,seed,H,W,g,s,f,nf", CR.GOLDEN_CASES)
def test_restatement_matches_golden(name, seed, H, W, g, s, f, nf):
    case = CR.make_case(seed, H, W, g, s, f, nf)
    z = np.load(CR.golden_path(name))
    assert str(z["digest"]) == CR.case_digest(case), "synthetic layers drifted from the goldens"
    assert np.array_equal(CR.composite_np(**case), z["frame"])


@pytest.mark.parametrize("g,s,f", CR.COMBOS)
def test_restatement_matches_reference_blend_frames(g, s, f):
    mod = CR.load_reference()
    if mod is None:
        pytest.skip("the reference's blend_all.py is not staged (build() stages it where the reference sources are)")
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = CR.write_dir(tmp, 2, 900 + 4 * g + 2 * s + f, 67, 1009, g, s, f)
        frames = CR.run_reference(mod, results, cfg)
    for fr, c in zip(frames, cases):
        assert np.array_equal(fr, CR.composite_np(**c))


def test_golden_directory_matches_reference():
    mod = CR.load_reference()
    if mod is None:
        pytest.skip("the reference's blend_all.py is not staged")
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = CR.write_dir(tmp, 5, 500, 31, 45)
        frames = CR.run_reference(mod, results, cfg)
    assert np.array_equal(frames, np.load(CR.golden_path("dir5"))["frames"])
