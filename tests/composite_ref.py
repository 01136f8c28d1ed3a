"""Frame compositing test support ("BA/" = blender/blend_all.py of the reference):

  * ``composite_np``: a numpy restatement of blend_frames' loop body (BA/:206-342) on decoded arrays, same operations in the same
    order, pinned against the reference's own ``blend_frames`` (tests/test_composite_cpu.py) and used by the GPU tests;
  * ``make_case``: seeded synthetic layers with the values the kernels must get right (depth ties, +-inf and NaN, alpha bytes
    0, 1, 254 and 255, shadow colour 0, every (rgb_all, rgb_shadow) byte pair around the 0.01 threshold);
  * ``write_dir``: a blend_frames directory of such layers (PNG, NPY, EXR);
  * ``load_reference``: the reference's blend_all.py as staged by ``build()`` under oracle/_ref_py/blender (None when absent),
    imported with stand-ins for the modules it imports and this environment lacks (tqdm, skimage, imageio).

Golden frames of the reference (tests/golden/ref/composite_*.npz) are written by ``python -m tests.composite_ref``; GPU tests read
those, never the reference.
"""
from __future__ import annotations

import hashlib
import importlib.util
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BLEND_ALL = os.path.join(ROOT, "oracle", "_ref_py", "blender", "blend_all.py")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")

# (gs, smoke, fire): every combination the reference accepts (fire needs smoke)
COMBOS = [(g, s, f) for g in (False, True) for s in (False, True) for f in (False, True) if s or not f]


# ------------------------------------------------------------------------------------------------------------ restatement
def composite_np(bg_c, o_c, o_d, s_c, s_d, o_s_c, o_gs_c=None, o_gs_d=None, s_f_c=None, s_f_d=None, s_f_c_pre=None):
    """BA/:206-342 for one frame of equal-sized layers (downsample_image is the identity there).  Inputs are the decoded arrays:
    uint8 [H,W,4] colours, float32 [H,W] depths.  Returns uint8 [H,W,4]."""
    has_3dgs, has_smoke, has_fire = o_gs_c is not None, s_f_c is not None, s_f_c_pre is not None
    if has_smoke:
        s_f_d = s_f_d.copy()
        mask = (s_f_c[..., 3] / 255.) > 0.0
        s_f_d[mask] = np.percentile(s_f_d, 0.001)
    bg_c, o_c, s_c, o_s_c = (a.astype(np.float32) for a in (bg_c, o_c, s_c, o_s_c))
    if has_3dgs:
        o_gs_c = o_gs_c.astype(np.float32)
    if has_smoke:
        s_f_c = s_f_c.astype(np.float32)
        if has_fire:
            s_f_c_pre = s_f_c_pre.astype(np.float32)
    frame = bg_c.copy()
    if has_3dgs:
        depth_mask = s_d <= o_gs_d
        non_obj_3dgs_alpha = 1. - o_gs_c[..., 3] / 255.
        non_obj_3dgs_alpha[depth_mask] = 1.0
    obj_alpha = o_c[..., 3] / 255.
    depth_mask = o_d <= s_d
    if has_smoke or has_fire:
        obj_alpha_smoke = s_f_c[..., 3] / 255.
        depth_mask_smoke = s_f_d <= s_d
        obj_alpha = np.maximum(obj_alpha, obj_alpha_smoke)
        depth_mask = np.logical_or(depth_mask, depth_mask_smoke)
    obj_mask = obj_alpha > 0.0
    mask = np.logical_and(obj_mask, depth_mask)
    obj_alpha[~mask] = 0.0
    non_object_alpha = 1. - obj_alpha
    if has_3dgs:
        front = o_gs_d <= o_d
        obj_alpha[front] *= non_obj_3dgs_alpha[front]
    fg_alpha = o_s_c[..., 3] / 255.
    sca = non_object_alpha * fg_alpha * non_obj_3dgs_alpha if has_3dgs else non_object_alpha * fg_alpha
    scm = sca > 0.0
    color_diff = np.ones_like(o_c)
    color_diff[scm, 0:3] = o_s_c[scm, :3] / (s_c[scm, :3] + 1e-6)
    color_diff = np.clip(color_diff, 0, 1)
    m = np.logical_not(np.all(np.abs(color_diff - 1) < 0.01, axis=-1))
    frame[m] = frame[m] * color_diff[m] * sca[m, None] + frame[m] * (1 - sca[m, None])
    frame_tmp = frame.copy()
    mask = np.logical_and(obj_mask, depth_mask)
    frame[:, :, :3][mask] = o_c[:, :, :3][mask] * obj_alpha[mask, None] + frame_tmp[:, :, :3][mask] * (1 - obj_alpha[mask, None])
    if has_fire:
        mask = depth_mask_smoke
        frame[:, :, :3][mask] = s_f_c_pre[:, :, :3][mask] + frame_tmp[:, :, :3][mask] * (1 - obj_alpha_smoke[mask, None])
    with np.errstate(invalid="ignore"):
        return np.clip(frame, 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------------ synthetic layers
SPECIAL_BYTES = np.array([0, 1, 254, 255], np.uint8)


def _bytes(rng, shape):
    b = rng.integers(0, 256, shape, dtype=np.uint8)
    sp = rng.random(shape) < 0.35
    b[sp] = SPECIAL_BYTES[rng.integers(0, 4, int(sp.sum()))]
    return b


def _depth(rng, shape, nonfinite=True):
    d = rng.uniform(0.5, 4.0, shape).astype(np.float32)
    r = rng.random(shape)
    d[r < 0.3] = np.float32([1.0, 2.0, 3.0])[rng.integers(0, 3, int((r < 0.3).sum()))]  # ties across layers
    if nonfinite:
        d[(r >= 0.3) & (r < 0.34)] = np.inf
        d[(r >= 0.34) & (r < 0.36)] = -np.inf
        d[(r >= 0.36) & (r < 0.38)] = np.nan
    d[(r >= 0.38) & (r < 0.39)] = -0.0
    d[(r >= 0.39) & (r < 0.40)] = 0.0
    return d


def _rgba(rng, shape, zero_alpha=0.3):
    c = _bytes(rng, shape + (4,))
    c[..., 3][rng.random(shape) < zero_alpha] = 0
    return c


def make_case(seed, H, W, gs, smoke, fire, smoke_nonfinite=False):
    """Decoded layers of one frame: a dict of composite_np's keyword arguments (rgb_* as uint8 [H,W,4], depths as float32 [H,W]).
    When H*W >= 65536 the first 65536 pixels hold every (rgb_all, rgb_shadow) byte pair with rgb_all's alpha 255 and no object,
    so color_diff meets the 0.01 threshold from both sides and s_c = 0 takes the 1e-6 path."""
    rng = np.random.default_rng(seed)
    sh = (H, W)
    c = {"bg_c": _rgba(rng, sh, 0.05), "o_c": _rgba(rng, sh), "o_d": _depth(rng, sh), "s_c": _rgba(rng, sh), "s_d": _depth(rng, sh),
         "o_s_c": _rgba(rng, sh)}
    if gs:
        c["o_gs_c"], c["o_gs_d"] = _rgba(rng, sh), _depth(rng, sh)
    if smoke:
        c["s_f_c"], c["s_f_d"] = _rgba(rng, sh, 0.6), _depth(rng, sh, nonfinite=smoke_nonfinite)
        if fire:
            c["s_f_c_pre"] = _rgba(rng, sh)
    if H * W >= 65536:
        flat = {k: v.reshape((H * W,) + v.shape[2:]) for k, v in c.items()}
        i = np.arange(65536)
        flat["o_s_c"][i, :3] = (i % 256)[:, None]
        flat["o_s_c"][i, 3] = 255
        flat["s_c"][i, :3] = (i // 256)[:, None]
        flat["o_c"][i, 3] = 0
        for k in ("o_gs_c", "s_f_c"):
            if k in flat:
                flat[k][i, 3] = 0
    return c


def case_digest(case):
    h = hashlib.sha256()
    for k in sorted(case):
        h.update(k.encode())
        h.update(np.ascontiguousarray(case[k]).tobytes())
    return h.hexdigest()


# the golden cases: every layer combination at an odd size and one with the exhaustive byte-pair block
# (a finite smoke depth keeps the percentile finite; +-inf or NaN in it makes the percentile NaN, the last case)
GOLDEN_CASES = [("combo_%d%d%d" % (g, s, f), 11 + 4 * i, 37, 53, g, s, f, False) for i, (g, s, f) in enumerate(COMBOS)] + \
               [("pairs_%d%d%d" % c, 101 + i, 257, 263) + c + (False,) for i, c in enumerate([(False, False, False), (True, True, True)])] + \
               [("smoke_nonfinite", 7, 29, 31, True, True, True, True)]


# ------------------------------------------------------------------------------------------------------------ directories
def write_dir(base, n_frames, seed, H, W, gs=True, smoke=True, fire=True, smoke_nonfinite=False, write_exr=None):
    """A blend_frames layout under ``base``: <base>/scene/images/*.png and depth/*.npy (the 3DGS frames),
    <base>/cache/out/rgb_*/NNN.png and depth_*/NNN/ImageNNNN.exr (the Blender layers), <base>/scene/blend/results (the results
    directory) and <base>/config.json.  Returns (results_dir, config_path, cases) with cases[i] the decoded arrays of frame i.
    ``write_exr(path, array)`` writes one depth layer (default cv2.imwrite of a 3-channel float32 EXR)."""
    from PIL import Image
    if write_exr is None:
        os.environ["OPENCV_IO_ENABLE_OPENEXR"] = "1"
        import cv2

        def write_exr(path, d):
            assert cv2.imwrite(path, np.repeat(d[..., None], 3, axis=2)), path
    scene = os.path.join(base, "scene")
    results = os.path.join(scene, "blend", "results")
    cache = os.path.join(base, "cache", "out")
    for d in (os.path.join(scene, "images"), os.path.join(scene, "depth"), results):
        os.makedirs(d, exist_ok=True)
    cases = []
    for i in range(n_frames):
        c = make_case(seed + i, H, W, gs, smoke, fire, smoke_nonfinite)
        cases.append(c)
        Image.fromarray(c["bg_c"]).save(os.path.join(scene, "images", "%05d.png" % i))
        np.save(os.path.join(scene, "depth", "%05d.npy" % i), np.ones((H, W), np.float32))
        layers = {"rgb_obj": c["o_c"], "rgb_shadow": c["s_c"], "rgb_all": c["o_s_c"], "rgb_obj_3dgs": c.get("o_gs_c"),
                  "rgb_smoke_fire": c.get("s_f_c"), "rgb_smoke_fire_pre": c.get("s_f_c_pre")}
        depths = {"depth_obj": c["o_d"], "depth_shadow": c["s_d"], "depth_all": np.zeros((H, W), np.float32), "depth_obj_3dgs": c.get("o_gs_d"),
                  "depth_smoke_fire": c.get("s_f_d"), "depth_smoke_fire_pre": np.zeros((H, W), np.float32) if fire else None}
        for name, a in layers.items():
            if a is not None:
                os.makedirs(os.path.join(cache, name), exist_ok=True)
                Image.fromarray(a).save(os.path.join(cache, name, "%03d.png" % (i + 1)))
        for name, a in depths.items():
            if a is not None:
                d = os.path.join(cache, name, "%03d" % (i + 1))
                os.makedirs(d, exist_ok=True)
                write_exr(os.path.join(d, "Image%04d.exr" % (i + 1)), a)
    cfg = os.path.join(base, "config.json")
    with open(cfg, "w") as f:
        json.dump({"blender_cache_dir": os.path.join(base, "cache"), "output_dir_name": "out"}, f)
    return results, cfg, cases


# ------------------------------------------------------------------------------------------------------------ the reference
def _install_stubs():
    """Stand-ins for the imports of blend_all.py that are not installed here; blend_frames only reaches tqdm (an iterable
    wrapper), and generate_video_from_frames (skimage resize, imageio.mimsave) is replaced by the callers that need it."""
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
        except ImportError:
            t = types.ModuleType("tqdm")
            t.tqdm = lambda it, *a, **k: it
            sys.modules["tqdm"] = t
    for name in ("skimage", "imageio", "imageio.v2"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except ImportError:
                sys.modules[name] = types.ModuleType(name)
    if not hasattr(sys.modules["imageio"], "v2"):
        sys.modules["imageio"].v2 = sys.modules["imageio.v2"]


def load_reference(name="_ref_blend_all"):
    """A fresh module object of the reference's blend_all.py, or None when build() has not staged it."""
    if not os.path.exists(REF_BLEND_ALL):
        return None
    _install_stubs()
    spec = importlib.util.spec_from_file_location(name, REF_BLEND_ALL)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def run_reference(mod, results, cfg):
    """mod.blend_frames on a directory; returns the frames handed to generate_video_from_frames (which records them instead of
    encoding a video)."""
    got = {}
    mod.generate_video_from_frames = lambda frames, path, fps=30: got.setdefault("frames", np.array(frames))
    mod.blend_frames(results, cfg)
    return got["frames"]


def golden_path(name):
    return os.path.join(GOLDEN, "composite_%s.npz" % name)


def write_goldens():
    """Run the reference's blend_frames on a one-frame directory per golden case and store its frame with the case digest."""
    import tempfile
    mod = load_reference()
    assert mod is not None, "the reference's blend_all.py is not staged (run build())"
    for name, seed, H, W, g, s, f, nf in GOLDEN_CASES:
        with tempfile.TemporaryDirectory() as tmp:
            results, cfg, cases = write_dir(tmp, 1, seed, H, W, g, s, f, nf)
            frame = run_reference(mod, results, cfg)[0]
        assert np.array_equal(frame, composite_np(**cases[0])), name
        np.savez_compressed(golden_path(name), frame=frame, digest=np.array(case_digest(cases[0])))
    with tempfile.TemporaryDirectory() as tmp:
        results, cfg, cases = write_dir(tmp, 5, 500, 31, 45)
        frames = run_reference(mod, results, cfg)
        pngs = [open(os.path.join(results, "frames", "%04d.png" % i), "rb").read() for i in range(5)]
    np.savez_compressed(golden_path("dir5"), frames=frames, digests=np.array([case_digest(c) for c in cases]),
                        png_sha=np.array([hashlib.sha256(p).hexdigest() for p in pngs]))


if __name__ == "__main__":
    write_goldens()
