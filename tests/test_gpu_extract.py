"""MaskScorer and its kernels (gsr_select_rows, gsr_pack_masks, gsr_mask_disagreement).  Run with -m gpu on an H100.

  1. scorer.count(m) equals extract_object's loop restated on render() in exact mode (tests/extract_ref.py) as integers, on the
     golden scenes and a 200k-Gaussian scene at 1080p, 8 views of which 2 have no mask, for the empty, full, single, random-half
     and box subsets and all-0, all-255 and rendered-then-flipped masks;
  2. the same counts from the compiled reference rasterizer's alpha (replayed from tests/golden/ref/ where it is not built);
  3. each kernel on its own against torch / numpy;
  4. a binning overflow: only the overflowed views are rendered again, and the count stays exact.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import extract_ref as X  # noqa: E402
from tests import helpers as Hh  # noqa: E402

pytestmark = pytest.mark.gpu

SCENES = ["config1", "dense_tile", "big_splats", "coplanar", "synthetic_1080p"]
SUBSETS = ["empty", "full", "single", "half", "box"]
N_VIEWS = 8
UNMASKED = (4, 7)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import rasterizer  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


@pytest.fixture
def exact_images():
    from autovfx_b200 import rasterizer as R
    R.set_exact_images(True)
    yield
    R.set_exact_images(False)


def _scene(name, dev):
    if name == "synthetic_1080p":
        from autovfx_b200 import scene
        g = scene.synthetic_gaussians(200_000, seed=31, extent=(1.5, 1.5, 0.5), log_scale_mean=np.log(0.01), log_scale_std=0.5)
        cam = scene.lookat_camera((0.0, -4.0, 1.5), (0, 0, 0), 1920, 1080, 60.0)
        return X.model_from(g, dev), cam
    c = Hh.case_inputs(name)
    return X.model_from(c["g"], dev), c["cam"]


def _subset(kind, xyz):
    P = xyz.shape[0]
    gen = torch.Generator().manual_seed(P)
    if kind == "empty":
        m = torch.zeros(P, dtype=torch.bool)
    elif kind == "full":
        m = torch.ones(P, dtype=torch.bool)
    elif kind == "single":
        m = torch.zeros(P, dtype=torch.bool)
        m[P // 3] = True
    elif kind == "half":
        m = torch.rand(P, generator=gen) < 0.5
    else:
        return X.box_subset(xyz, 0.2)
    return m.to(xyz.device)


def _masks(pc, views, dev):
    """Tracking masks of the views with one: all 0, all 255, or a random half-subset's render (alpha >= 0.8 -> 255) with 3 % of
    the pixels flipped and 1 % set to 254 (not 255, so off)."""
    from autovfx_b200.renderer import render
    half = X.crop(pc, _subset("half", pc.get_xyz))
    masks = {}
    for idx, view in enumerate(views):
        if idx in UNMASKED:
            continue
        H, W = int(view.image_height), int(view.image_width)
        if idx % 3 == 1:
            m = np.zeros((H, W), np.uint8)
        elif idx % 3 == 2:
            m = np.full((H, W), 255, np.uint8)
        else:
            with torch.no_grad():
                a = render(view, half, X.PIPE, torch.zeros(3, device=dev))["render"][3].cpu().numpy()
            m = np.where(a >= 0.8, 255, 0).astype(np.uint8)
            rng = np.random.default_rng(idx)
            flip = rng.random((H, W)) < 0.03
            m[flip] = 255 - m[flip]
            m[rng.random((H, W)) < 0.01] = 254
        masks["{0:05d}.png".format(idx)] = m
    return masks


def _ref_count(pc, views, masks, mask3d):
    """The loop's count with the compiled reference rasterizer's alpha."""
    from oracle import ref_cuda
    sub = X.crop(pc, mask3d)
    total = 0
    for idx, view in enumerate(views):
        if "{0:05d}.png".format(idx) not in masks:
            continue
        H, W = int(view.image_height), int(view.image_width)
        if sub.get_xyz.shape[0] == 0:
            alpha = np.zeros((H, W), np.float32)
        else:
            fw = ref_cuda.forward(sub.get_xyz, sub.get_opacity, view.world_view_transform, view.full_proj_transform, view.camera_center,
                                  W, H, float(np.tan(view.FoVx * 0.5)), float(np.tan(view.FoVy * 0.5)), shs=sub.get_features,
                                  scales=sub.get_scaling, rotations=sub.get_rotation, sh_degree=sub.active_sh_degree)
            alpha = fw["alpha"][0].cpu().numpy()
        total += int(np.count_nonzero(np.logical_xor(alpha >= 0.8, np.array(masks["{0:05d}.png".format(idx)]) == 255)))
    return total


@pytest.mark.parametrize("name", SCENES)
def test_count_matches_reference_loop(name, dev, exact_images):
    from autovfx_b200.extract import MaskScorer
    pc, cam = _scene(name, dev)
    views = X.orbit_views(cam, N_VIEWS, dev)
    masks = _masks(pc, views, dev)
    scorer = MaskScorer(pc, views, masks, X.PIPE)
    assert scorer.num_views == N_VIEWS - len(UNMASKED)
    bg = torch.zeros(3, device=dev)
    for kind in SUBSETS:
        m = _subset(kind, pc.get_xyz)
        got = scorer.count(m)
        assert got.dtype == torch.int64 and got.dim() == 0 and got.device == dev
        want = X.missed_pixels(pc, views, masks, m, bg)
        assert int(got) == want, (kind, int(got), want)
        assert int(scorer.count(m.cpu().numpy())) == want  # numpy selection, and the same count again
        if kind == "empty":
            assert want == sum(int(np.count_nonzero(v == 255)) for v in masks.values())
        if Hh.have_ref():
            assert int(got) == Hh.ref_value(lambda: _ref_count(pc, views, masks, m)), kind


def test_count_rejects_bad_selection(dev):
    from autovfx_b200.extract import MaskScorer
    pc, cam = _scene("config1", dev)
    views = X.orbit_views(cam, 2, dev)
    scorer = MaskScorer(pc, views, {"00001.png": np.zeros((cam.image_height, cam.image_width), np.uint8)})
    P = pc.get_xyz.shape[0]
    with pytest.raises(ValueError, match="selection"):
        scorer.count(torch.ones(P - 1, dtype=torch.bool, device=dev))
    with pytest.raises(ValueError, match="selection"):
        scorer.count(np.ones(P, np.int64))


def test_binning_overflow_rerenders_only_overflowed_views(dev, exact_images):
    from autovfx_b200 import rasterizer as R
    from autovfx_b200.extract import MaskScorer
    pc, cam = _scene("big_splats", dev)
    views = X.orbit_views(cam, N_VIEWS, dev)
    masks = _masks(pc, views, dev)
    full = _subset("full", pc.get_xyz)
    want = X.missed_pixels(pc, views, masks, full, torch.zeros(3, device=dev))
    st = R._state(dev)
    st.capacity, st.slab_want = 1, 0  # the next frames start from the smallest binning buffer
    scorer = MaskScorer(pc, views, masks, X.PIPE)
    assert int(scorer.count(full)) == want
    assert 0 < scorer.rerendered <= scorer.num_views
    again = scorer.rerendered
    assert int(scorer.count(full)) == want and scorer.rerendered == again  # the grown capacity holds every view now


# ------------------------------------------------------------------------------------------------------------- kernels alone
def _select(P, keep, rows, dev):
    from autovfx_b200 import _lib
    from autovfx_b200._lib import lib as L
    outs = [torch.full((max(P, 1), r.shape[1]), -7.0, device=dev) for r in rows]
    count = torch.full((), -1, dtype=torch.int32, device=dev)
    ws = torch.empty(max(int(L.gsr_select_rows_bytes(P)), 4), dtype=torch.uint8, device=dev)
    p = lambda t: t.data_ptr() if t.numel() else None  # noqa: E731
    _lib.check(L.gsr_select_rows(P, p(keep), *(p(r) for r in rows), *(o.data_ptr() for o in outs), count.data_ptr(), ws.data_ptr(),
                                 ws.numel(), _lib.stream_ptr(dev)), "gsr_select_rows")
    return outs, int(count)


@pytest.mark.parametrize("P", [0, 1, 1023, 1025, 3_000_000])
@pytest.mark.parametrize("kind", ["random", "all", "none"])
def test_select_rows_is_boolean_indexing(P, kind, dev):
    gen = torch.Generator(device=dev).manual_seed(P + len(kind))
    # every bit pattern, NaN payloads and negative zeros included
    rows = [torch.randint(-2**31, 2**31 - 1, (P, w), generator=gen, device=dev, dtype=torch.int32).view(torch.float32) for w in (3, 1, 3, 4)]
    keep = {"random": torch.rand(P, generator=gen, device=dev) < 0.37, "all": torch.ones(P, dtype=torch.bool, device=dev),
            "none": torch.zeros(P, dtype=torch.bool, device=dev)}[kind]
    outs, n = _select(P, keep, rows, dev)
    assert n == int(keep.sum())
    for r, o in zip(rows, outs):
        assert torch.equal(o[:n].view(torch.int32), r[keep].view(torch.int32))


def _unpack(bits, H):
    """[H, 32 * words] bool: every bit of the packed rows, the padding past W included."""
    b = bits.to(torch.int64) & 0xffffffff
    shifts = torch.arange(32, device=bits.device)
    return ((b.view(H, -1, 1) >> shifts) & 1).view(H, -1).bool()


@pytest.mark.parametrize("HW", [(1, 1), (33, 47), (1080, 1920)])
def test_pack_masks_is_eq_255(HW, dev):
    from autovfx_b200 import _lib
    from autovfx_b200._lib import lib as L
    H, W = HW
    V = 3
    gen = torch.Generator(device=dev).manual_seed(H * W)
    m = torch.randint(0, 256, (V, H, W), generator=gen, device=dev, dtype=torch.int32).to(torch.uint8)
    m[m > 200] = 255
    m[1] = 255
    wpr = (W + 31) // 32
    bits = torch.full((V, H, wpr), -1, dtype=torch.int32, device=dev)
    _lib.check(L.gsr_pack_masks(V, W, H, m.data_ptr(), bits.data_ptr(), _lib.stream_ptr(dev)), "gsr_pack_masks")
    for v in range(V):
        got = _unpack(bits[v], H)
        assert torch.equal(got[:, :W], m[v] == 255)
        assert not got[:, W:].any()


@pytest.mark.parametrize("HW", [(1, 1), (33, 47), (1080, 1920)])
def test_mask_disagreement_is_numpy_xor_count(HW, dev):
    from autovfx_b200 import _lib
    from autovfx_b200._lib import lib as L
    from autovfx_b200.extract import ALPHA_THRESHOLD
    H, W = HW
    rng = np.random.default_rng(H + W)
    t = ALPHA_THRESHOLD
    special = np.array([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(2)), np.nan, np.inf, -np.inf, 0.0, 1.0],
                       np.float32)
    alpha = np.where(rng.random((H, W)) < 0.5, rng.choice(special, (H, W)), rng.random((H, W)).astype(np.float32)).astype(np.float32)
    mask = np.where(rng.random((H, W)) < 0.5, 255, rng.integers(0, 255, (H, W))).astype(np.uint8)
    want = int(np.count_nonzero(np.logical_xor(alpha >= 0.8, mask == 255)))
    s = _lib.stream_ptr(dev)
    bits = torch.empty((H, (W + 31) // 32), dtype=torch.int32, device=dev)
    m = torch.from_numpy(mask).to(dev)
    _lib.check(L.gsr_pack_masks(1, W, H, m.data_ptr(), bits.data_ptr(), s), "gsr_pack_masks")
    a = torch.from_numpy(alpha).to(dev)
    count = torch.full((), 5, dtype=torch.int64, device=dev)
    for _ in range(2):  # it accumulates
        _lib.check(L.gsr_mask_disagreement(W, H, a.data_ptr(), bits.data_ptr(), float(t), count.data_ptr(), s), "gsr_mask_disagreement")
    assert int(count) == 5 + 2 * want
