"""Frame compositing on the GPU (autovfx_b200.composite) bit for bit against the numpy restatement of blend_frames' loop body
(tests/composite_ref.py) and the reference's golden frames (tests/golden/ref/composite_*.npz): every layer combination, the edge
values of the synthetic layers, sizes from 1x1 to 2160x3840, the percentile against np.percentile, no host synchronisation, a
non-default stream, the drop-in blend_frames' PNGs and the FrameLoop(pack8=True) consume path."""
from __future__ import annotations

import hashlib
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import composite_ref as CR  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _on_gpu(case, dev):
    t = lambda k: None if k not in case else torch.from_numpy(np.ascontiguousarray(case[k])).to(dev)  # noqa: E731
    return dict(rgba8=t("bg_c"), depth=None, obj=t("o_c"), obj_depth=t("o_d"), shadow=t("s_c"), shadow_depth=t("s_d"), all_=t("o_s_c"),
                obj3dgs=t("o_gs_c"), obj3dgs_depth=t("o_gs_d"), smoke=t("s_f_c"), smoke_depth=t("s_f_d"), fire=t("s_f_c_pre"))


def _composite(case, dev):
    from autovfx_b200.composite import composite_frame
    return composite_frame(**_on_gpu(case, dev)).cpu().numpy()


def _first_diff(a, b):
    bad = np.argwhere(a != b)
    return None if bad.size == 0 else (bad[0].tolist(), a[tuple(bad[0])], b[tuple(bad[0])], len(bad))


@pytest.mark.parametrize("name,seed,H,W,g,s,f,nf", CR.GOLDEN_CASES)
def test_golden_cases_bit_exact(dev, name, seed, H, W, g, s, f, nf):
    case = CR.make_case(seed, H, W, g, s, f, nf)
    z = np.load(CR.golden_path(name))
    assert str(z["digest"]) == CR.case_digest(case)
    got = _composite(case, dev)
    assert _first_diff(got, z["frame"]) is None, _first_diff(got, z["frame"])


@pytest.mark.parametrize("g,s,f", CR.COMBOS)
@pytest.mark.parametrize("H,W", [(1, 1), (1, 7), (33, 1), (61, 129), (1080, 1920)])
def test_every_combination_and_size_matches_restatement(dev, g, s, f, H, W):
    case = CR.make_case(1000 + H + W + 4 * g + 2 * s + f, H, W, g, s, f)
    got, want = _composite(case, dev), CR.composite_np(**case)
    assert _first_diff(got, want) is None, _first_diff(got, want)


@pytest.mark.parametrize("nonfinite", [False, True])
def test_4k_all_layers(dev, nonfinite):
    case = CR.make_case(77 + nonfinite, 2160, 3840, True, True, True, nonfinite)
    got, want = _composite(case, dev), CR.composite_np(**case)
    assert _first_diff(got, want) is None, _first_diff(got, want)


def test_clip_and_truncation_edges(dev):
    """Fire over a bright frame exceeds 255 (clip); object blends over every (colour, alpha) byte pair land on and just below
    integers (truncation)."""
    H, W = 256, 256
    case = CR.make_case(5, H, W, False, True, True)
    i = np.arange(H * W)
    fl = {k: v.reshape((H * W,) + v.shape[2:]) for k, v in case.items()}
    fl["o_c"][i, 0] = i % 256
    fl["o_c"][i, 3] = i // 256
    fl["o_d"][:] = 0.5
    fl["s_d"][:] = 1.0
    fl["s_f_c_pre"][i, 1] = 255
    got, want = _composite(case, dev), CR.composite_np(**case)
    assert _first_diff(got, want) is None
    assert (want[..., 1] == 255).any() and (want[..., 0] == 0).any()


def _pct_cases():
    r = np.random.default_rng(3)
    cases = {"n1": np.float32([2.5]), "n1_inf": np.float32([np.inf]), "n2": np.float32([3.0, -1.0]), "ties": np.float32([1, 1, 1, 2, 0, 0] * 5),
             "all_equal": np.full(100000, 7.25, np.float32), "zeros": np.float32([-0.0, 0.0] * 50000),
             "nan": np.concatenate([r.random(1000).astype(np.float32), np.float32([np.nan])]),
             "neg_inf": np.concatenate([r.random(200001).astype(np.float32), np.float32([-np.inf] * 3)]),
             "1080p": r.normal(3, 1, 1080 * 1920).astype(np.float32), "4k": r.uniform(-5, 5, 2160 * 3840).astype(np.float32),
             "background": np.where(r.random(1080 * 1920) < 0.9, np.float32(1e10), r.random(1080 * 1920).astype(np.float32) * 4)}
    # n where numpy's float32 gamma is just below and just above 0.5
    q = np.float32(0.001) / np.float32(100)
    n = np.arange(2, 300000)
    v = (n - 1).astype(np.float32) * q
    t = v - np.floor(v)
    cases["t_below"] = r.random(int(n[(t > 0.49) & (t < 0.5)][0])).astype(np.float32) * 10
    cases["t_above"] = r.random(int(n[(t >= 0.5) & (t < 0.51)][0])).astype(np.float32) * 10
    return cases


_PCT = _pct_cases()


@pytest.mark.parametrize("name", sorted(_PCT))
def test_percentile_matches_numpy(dev, name):
    from autovfx_b200.composite import percentile_low
    x = _PCT[name]
    with np.errstate(invalid="ignore"):
        want = np.float32(np.percentile(x, 0.001))
    got = percentile_low(torch.from_numpy(x).to(dev)).item()
    assert (np.isnan(want) and np.isnan(got)) or np.float32(got) == want, (got, want)  # -0.0 == +0.0 (sign not pinned)


def test_no_host_synchronisation_and_side_stream(dev):
    from autovfx_b200.composite import composite_frame
    case = CR.make_case(21, 540, 960, True, True, True)
    want = CR.composite_np(**case)
    args = _on_gpu(case, dev)
    torch.cuda.synchronize()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            out = composite_frame(**args)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    side.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)


def _install(mod):
    """The drop-in installed on a module with blend_all's loaders and a recording generate_video_from_frames."""
    from autovfx_b200 import composite
    mod.blend_frames = composite.blend_frames
    got = {}
    mod.generate_video_from_frames = lambda frames, path, fps=30: got.setdefault("frames", np.array(frames))
    return got


def _loaders_module():
    """blend_all's three loaders (BA/:56-75), restated so that the GPU machine needs no reference file."""
    import cv2
    from PIL import Image
    os.environ["OPENCV_IO_ENABLE_OPENEXR"] = "1"
    m = types.ModuleType("blend_all_loaders")
    m.load_rgb = lambda p: None if not os.path.exists(p) else np.array(Image.open(p).convert("RGBA"))
    m.load_depth = lambda p: None if not os.path.exists(p) else np.load(p)
    m.load_depth_exr = lambda p: None if not os.path.exists(p) else cv2.imread(p, cv2.IMREAD_ANYCOLOR | cv2.IMREAD_ANYDEPTH)[:, :, 0]
    sys.modules[m.__name__] = m
    return m


def test_drop_in_blend_frames_writes_the_golden_pngs(dev):
    m = _loaders_module()
    got = _install(m)
    z = np.load(CR.golden_path("dir5"))
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = CR.write_dir(tmp, 5, 500, 31, 45)
        assert [CR.case_digest(c) for c in cases] == list(z["digests"])
        m.blend_frames(results, cfg)
        shas = [hashlib.sha256(open(os.path.join(results, "frames", "%04d.png" % i), "rb").read()).hexdigest() for i in range(5)]
    assert np.array_equal(got["frames"], z["frames"])
    assert shas == list(z["png_sha"])


def test_frame_loop_consume_path_equals_the_file_path(dev):
    """FrameLoop(pack8=True, to_host=False): compositing the device rgba8 in consume gives the frames the drop-in makes from the
    same frames saved as images/*.png and depth/*.npy."""
    from PIL import Image
    from autovfx_b200 import render_loop as RL, scene
    from autovfx_b200.composite import composite_frame
    W, H = 160, 96
    g = scene.synthetic_gaussians(20000, seed=4)
    cams = [scene.lookat_camera((0.3 * i, -3.0, 0.4), (0, 0, 0), W, H, 60.0) for i in range(3)]
    m = _loaders_module()
    got_files = _install(m)
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = CR.write_dir(tmp, 3, 40, H, W)
        layers = [{k: v for k, v in _on_gpu(c, dev).items() if k not in ("rgba8", "depth")} for c in cases]
        resident = {}
        scene_dir = os.path.dirname(os.path.dirname(results))

        def consume(i, fr, stats):
            resident[i] = composite_frame(fr["rgba8"], fr["depth"], **layers[i]).cpu().numpy()
            Image.fromarray(fr["rgba8"].cpu().numpy()).save(os.path.join(scene_dir, "images", "%05d.png" % i))
            np.save(os.path.join(scene_dir, "depth", "%05d.npy" % i), fr["depth"].cpu().numpy())
        loop = RL.FrameLoop({k: v.to(dev) for k, v in g.items()}, 3, W, H, device=dev, to_host=False, pack8=True)
        loop.render(RL.pack_cameras(cams), consume)
        m.blend_frames(results, cfg)
    assert len(resident) == 3
    for i in range(3):
        assert np.array_equal(resident[i], got_files["frames"][i]), i
