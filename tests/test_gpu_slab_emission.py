"""Slab emission (k_project writes every sort pair into its tile's slab, no k_emit) against the ranked emission (k_emit), driven
through the C ABI on the same inputs: every output bit for bit, overflow of an undersized slab without a write past any slab, the
safe mode's re-run with a grown stride, and the host's fall-back to the ranked emission on a scene that crowds one tile."""
import ctypes as C

import pytest
import torch

from autovfx_b200 import _lib, scene
from autovfx_b200 import rasterizer as R

from . import helpers as Hh

pytestmark = pytest.mark.gpu

CASES = ("config1", "small_sh", "small_deg1_m25", "deg3_m25", "deg2_m25", "small_precomp", "big_splats", "dense_tile", "coplanar")
FILL = 0xA5  # workspace bytes before the call: 0xA5A5A5A5 is a negative float, never the depth word of a pair


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _forward(a, S, flags=0, extra=None, cap=None):
    """One gsr_forward_multi with slab stride S (0: ranked emission) into freshly filled workspaces."""
    L = _lib.lib
    P, W, H = a["means3D"].shape[0], a["W"], a["H"]
    dev = a["means3D"].device
    cap = cap if cap is not None else 8 * P + 65536
    geom = torch.empty(L.gsr_geom_bytes(P), dtype=torch.uint8, device=dev)
    binning = torch.full((L.gsr_binning_bytes_slab(cap, W, H, S),), FILL, dtype=torch.uint8, device=dev)
    image = torch.empty(L.gsr_image_bytes(W, H), dtype=torch.uint8, device=dev)
    color, depth, alpha = (torch.empty((c, H, W), device=dev) for c in (3, 1, 1))
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    extra_out = None if extra is None else torch.empty((3, H, W), device=dev)
    shs = a["shs"]
    fr = _lib.gsr_frame(P, a["sh_degree"], 0 if shs is None else shs.shape[1], W, H, a["scale_modifier"], a["tanfovx"], a["tanfovy"], 0, 0,
                        _ptr(a["bg"]), _ptr(a["means3D"]), _ptr(shs), _ptr(a["colors_precomp"]), _ptr(a["opacities"]), _ptr(a["scales"]),
                        _ptr(a["rotations"]), _ptr(a["cov3D_precomp"]), _ptr(a["view"]), _ptr(a["proj"]), _ptr(a["campos"]))
    ws = _lib.gsr_workspace(geom.data_ptr(), geom.numel(), binning.data_ptr(), binning.numel(), image.data_ptr(), image.numel())
    flags |= _lib.GSR_FLAG_SORTED_KEYS | R.slab_flags(S)
    rc = L.gsr_forward_multi(C.byref(fr), C.byref(ws), color.data_ptr(), depth.data_ptr(), alpha.data_ptr(), radii.data_ptr(), _ptr(extra),
                             _ptr(extra_out), flags, None)
    _lib.check(rc, "gsr_forward_multi")
    torch.cuda.synchronize()
    views = R.debug_views((geom, binning, image), P, W, H)
    stats = [int(x) for x in views["counters"].tolist()]
    Rn = stats[0]
    out = dict(color=color, depth=depth, alpha=alpha, radii=radii, extra=extra_out, ranges=views["ranges"].clone(),
               point_list=views["point_list"][:Rn].clone(), sorted_keys=views["sorted_keys"][:Rn].clone(), overflow=stats[1],
               max_tile=stats[2], num_rendered=Rn, binning=binning, tile_count=views["tile_count"].clone())
    if flags & _lib.GSR_FLAG_FOR_BACKWARD:
        out["n_contrib"] = views["n_contrib"].clone()
    return out


def _stride(max_tile):
    return -(-int(max_tile * 1.25) // 32) * 32


def _assert_same(x, y):
    assert x["overflow"] == 0 and y["overflow"] == 0
    assert x["num_rendered"] == y["num_rendered"] and x["max_tile"] == y["max_tile"]
    for k in ("color", "depth", "alpha", "radii", "extra", "ranges", "point_list", "sorted_keys", "n_contrib"):
        if x.get(k) is not None:
            assert torch.equal(x[k], y[k]), k


FLAG_SETS = {"default": 0, "exact": _lib.GSR_FLAG_EXACT_IMAGES, "tight": _lib.GSR_FLAG_TIGHT_TILES, "backward": _lib.GSR_FLAG_FOR_BACKWARD}


@pytest.mark.parametrize("mode", sorted(FLAG_SETS))
@pytest.mark.parametrize("name", CASES)
def test_slab_equals_ranked_emission(dev, name, mode):
    """Every golden case under every mode: images, radii, ranges, point_list, sorted keys and n_contrib bit for bit (tight tiles
    ignore the stride and run the ranked emission)."""
    a = Hh.resolve(Hh.case_inputs(name), dev)
    extra = torch.rand(a["means3D"].shape[0], 3, generator=torch.Generator().manual_seed(5)).to(dev) if mode == "default" else None
    ranked = _forward(a, 0, FLAG_SETS[mode], extra)
    slab = _forward(a, _stride(ranked["max_tile"]), FLAG_SETS[mode], extra)
    _assert_same(ranked, slab)


def test_slab_gradients_equal_ranked_emission(dev):
    """A training step through the public API with the slab disabled (budget 0) and enabled: the same images, and gradients equal up
    to the order of the backward's float atomics (its inputs, lists and n_contrib, are compared bit for bit above)."""
    a = Hh.resolve(Hh.case_inputs("config1"), dev)
    dc, dd, da = Hh.image_grads(a, device=dev)
    old = R.SLAB_BUDGET
    try:
        R.SLAB_BUDGET = 0
        assert R._state(dev).slab_stride(a["means3D"].shape[0], a["W"], a["H"]) == 0
        out0, g0 = Hh.ours_backward(a, dc, dd, da)
    finally:
        R.SLAB_BUDGET = old
    assert R._state(dev).slab_stride(a["means3D"].shape[0], a["W"], a["H"]) > 0
    out1, g1 = Hh.ours_backward(a, dc, dd, da)
    for x, y in zip(out0, out1):
        assert torch.equal(x, y)
    for k, v in g0.items():
        if v is not None:
            assert Hh.relerr(g1[k], v) < 1e-5, k


@pytest.fixture(scope="module")
def scene3m(dev):
    return scene.config3_scene(), scene.cameras_from_trajectory(scene.trajectory_dict(num_views=300))


@pytest.mark.parametrize("cam", [0, 42, 150])
def test_slab_equals_ranked_emission_3m_1080p(dev, scene3m, cam):
    g, cams = scene3m
    a = Hh.resolve(dict(g=g, cam=cams[cam], sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), dev)
    ranked = _forward(a, 0, _lib.GSR_FLAG_FOR_BACKWARD, cap=12_000_000)
    S = _stride(ranked["max_tile"])
    slab = _forward(a, S, _lib.GSR_FLAG_FOR_BACKWARD, cap=12_000_000)
    _assert_same(ranked, slab)
    tiles = ranked["ranges"].shape[0]
    print("cam %d: R %d max_tile %d S %d slab MB %.1f" % (cam, ranked["num_rendered"], ranked["max_tile"], S, tiles * S * 8 / 2 ** 20))


def test_small_slab_overflows_without_writing_past_a_slab(dev):
    """S below the longest tile list: the overflow flag is set, the counts keep rising (max_tile says what is needed), and every
    slab holds exactly min(count, S) pairs — nothing spilled into a neighbour — while the bytes around the slab region stay as filled."""
    a = Hh.resolve(Hh.case_inputs("config1"), dev)
    ranked = _forward(a, 0)
    S = 32
    assert ranked["max_tile"] > S
    out = _forward(a, S)
    assert out["overflow"] == 1 and out["max_tile"] == ranked["max_tile"] and out["num_rendered"] == ranked["num_rendered"]
    L = _lib.lib
    W, H = a["W"], a["H"]
    tiles = out["ranges"].shape[0]
    binning = out["binning"]
    cap_all = L.gsr_binning_capacity(binning.numel())
    off = (8 * (cap_all - tiles * S)) & ~255
    words = binning[off:off + 8 * tiles * S].view(torch.int32).view(tiles, S, 2)
    written = (words[:, :, 1] != int.from_bytes(bytes([FILL] * 4), "little", signed=True)).sum(1)
    want = torch.clamp(out["tile_count"], max=S)
    assert torch.equal(written.to(torch.int64), want.to(torch.int64))
    assert bool((binning[:off] == FILL).all()) and bool((binning[off + 8 * tiles * S:] == FILL).all())
    assert L.gsr_binning_capacity_slab(binning.numel(), W, H, S) == off // 8


def test_safe_mode_grows_the_slab_and_returns_the_same_frame(dev):
    a = Hh.resolve(Hh.case_inputs("config1"), dev)
    ranked = _forward(a, 0)
    st = R._state(dev)
    old = st.slab_want
    try:
        st.slab_want = 32  # far below max_tile
        st.cache.clear()
        out = Hh.run_ours(a, debug=False)
        assert out["stats"]["overflow"] == 0 and st.slab_want == _stride(ranked["max_tile"])
        assert st.slab_stride(a["means3D"].shape[0], a["W"], a["H"]) == st.slab_want
    finally:
        st.slab_want = old
    for k in ("color", "depth", "alpha", "radii"):
        assert torch.equal(out[k], ranked[k]), k


def test_crowded_tile_selects_the_ranked_emission(dev):
    """Most Gaussians in one tile of a 1080p image: the slab a stride of 1.25 x max_tile needs exceeds the budget, so the host
    renders with the ranked emission, and the frame equals the C ABI's ranked result."""
    g = scene.synthetic_gaussians(120_000, seed=41, extent=(0.005, 0.005, 0.005), log_scale_mean=-7.0, log_scale_std=0.2)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 1920, 1080, 60.0)
    a = Hh.resolve(dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), dev)
    st = R._state(dev)
    old = (st.capacity, st.slab_want)
    try:
        st.cache.clear()
        st.capacity, st.slab_want = 1 << 20, 0
        out = Hh.run_ours(a, debug=False)
        P = a["means3D"].shape[0]
        assert out["stats"]["max_tile"] > P // 4 and st.slab_stride(P, 1920, 1080) == 0
    finally:
        st.capacity, st.slab_want = max(old[0], st.capacity), old[1]
    ranked = _forward(a, 0)
    for k in ("color", "depth", "alpha", "radii"):
        assert torch.equal(out[k], ranked[k]), k
