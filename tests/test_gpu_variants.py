"""GPU tests of the kernel variants the named cases of test_gpu_parity.py never dispatch to (run with -m gpu on an H100).

Which colour + emission kernel runs depends on the SH storage: M coefficients per row, the active degree D (clamped to 3)
and the alignment of the shs rows (16-byte aligned rows with M % 4 == 0 are staged with vector copies, 16-byte aligned
rows of other widths through an aligned window when it fits, everything else one float at a time), and the backward's
Gaussian kernel has a special case for M = 16.  One more path is selected per process: GSR_PACKED_KEYS=0 (the general
sort and emission that scenes of more than 2^24 Gaussians use).  This file runs each of them:

  A. the layout matrix: every (M, D) a GaussianModel can store, with shs rows 16-byte aligned and 4 bytes off, against each
     other (bit identity), the CPU oracle, the compiled reference (bit identity in exact mode) and the exact-mode images;
  B. per-Gaussian gradients against fp64 autograd (tests/torch_ref.py) with each image gradient isolated, judged against the
     CPU oracle's own error on the same case, and the gradients that must be exactly zero;
  C. the general path, in a fresh process, against the in-process default on part of the layout matrix, the gradient cases
     and the named cases (tiles in every sort regime), and the real P > 2^24 switch;
  D. distCUDA2 against an exact float64 k-d tree, at the sizes and shapes its search treats specially.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402
from autovfx_b200 import scene  # noqa: E402

pytestmark = pytest.mark.gpu

IMG_TOL = 1e-4  # against the CPU oracle (BASELINE.json: "within 1e-4 max abs per channel")

# (M, D) pairs of the layout matrix: M = (max_sh_degree + 1)^2 of a GaussianModel, or 25 (SuGaR), at every degree it can
# render; D = 5 is clamped to 3
LAYOUTS = [(1, 0), (4, 0), (4, 1), (9, 1), (9, 2), (16, 0), (16, 1), (16, 2), (16, 3), (16, 5), (25, 0), (25, 1), (25, 2), (25, 3)]
MATRIX = [(M, D, off) for (M, D) in LAYOUTS for off in (False, True)] + [(None, 0, False)]


def layout_id(M, D, off):
    return "precomp" if M is None else "M%d-D%d-%s" % (M, D, "off4" if off else "al16")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import rasterizer  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


def _forward(a, exact):
    """Every output of one forward (for_backward: n_contrib is written) as CPU tensors."""
    o = Hh.run_ours(a, for_backward=True, exact=exact)
    v = o["views"]
    R = o["stats"]["num_rendered"]
    return {"color": o["color"].cpu(), "depth": o["depth"].cpu(), "alpha": o["alpha"].cpu(), "radii": o["radii"].cpu(),
            "point_list": v["point_list"][:R].cpu(), "ranges": v["ranges"].cpu(), "n_contrib": v["n_contrib"].cpu()}


def _assert_same(got, want, what):
    for k in want:
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), "%s: %s differs" % (what, k)


# ---- A. the layout matrix -------------------------------------------------------------------------------------------------

def _groups():
    """Layouts that render the same coefficients, keyed by the effective degree."""
    out = {}
    for M, D, off in MATRIX:
        if M is not None:
            out.setdefault(min(D, 3), []).append((M, D, off))
    return out


@pytest.mark.parametrize("deg", sorted(_groups()))
def test_layouts_render_bit_identical_outputs(dev, deg):
    """The same active coefficients stored in every layout (different data in the unused tail, rows aligned or 4 bytes off):
    images, radii, tile lists and n_contrib are bit-identical in exact and in default mode."""
    layouts = _groups()[deg]
    assert len(layouts) >= 4
    for exact in (True, False):
        first = None
        for M, D, off in layouts:
            a = Hh.layout_args(M, D, off, dev)
            assert (a["shs"].data_ptr() % 16 == 4) == off
            out = _forward(a, exact)
            if first is None:
                first = out
            else:
                _assert_same(out, first, "%s exact=%s" % (layout_id(M, D, off), exact))


@pytest.mark.parametrize("M,D,off", MATRIX, ids=[layout_id(*m) for m in MATRIX])
def test_layout_against_oracle_reference_and_exact_mode(dev, M, D, off):
    a = Hh.layout_args(M, D, off, dev)
    exact = _forward(a, True)
    default = _forward(a, False)
    # the oracle: images within 1e-4, radii equal
    orc = Hh.run_oracle(a)
    assert torch.equal(exact["radii"], torch.from_numpy(orc["radii"]))
    for k in ("color", "depth", "alpha"):
        assert Hh.maxabs(exact[k], orc[k]) <= IMG_TOL, k
        assert Hh.maxabs(default[k], orc[k]) <= IMG_TOL, k
    if M is not None:
        assert orc["clamped"].any()  # channels below -0.5 before the offset: the clamp bits are exercised
    # default mode against exact mode: same decisions, images within the fast-blend tolerance
    Hh.assert_images_close(default, exact)
    assert torch.equal(default["n_contrib"], exact["n_contrib"])
    for k in ("radii", "point_list", "ranges"):
        assert torch.equal(default[k], exact[k]), k
    # the compiled reference (live, or its recorded digests): exact-mode images and radii bit-identical
    if not Hh.have_ref():
        pytest.skip("no compiled reference and no recorded reference values")
    ref = Hh.run_ref(a)
    assert Hh.ref_same(exact["radii"], lambda: ref["radii"])
    for k in ("color", "depth", "alpha"):
        assert Hh.ref_same(exact[k], lambda: ref[k]), k


# ---- B. per-Gaussian gradients against fp64 autograd ------------------------------------------------------------------------
# e = ||g - g64|| / ||g64|| per Gaussian (rows with ||g64|| > 1e-6 of the largest row), for each gradient tensor.  The GPU's
# median and 99th percentile must stay within GRAD_FACTOR times the CPU oracle's on the same case plus GRAD_FLOOR.  The oracle
# makes the same fp32 skip / termination decisions as the GPU, so decisions that fp32 and fp64 would take differently cost both
# the same, and the oracle itself is pinned against fp64 in test_variants_cpu.py.
# Measured on an H100 80GB HBM3 over the 128 (family, term, tensor) combinations: GPU / oracle is at most 1.09 at the median
# (typically 0.93) and at most 2.14 at the 99th percentile (typically 0.90; the largest is dL/dopacity of M16_D3 under the
# colour term, 3.7e-5 against 1.7e-5); the GPU's medians are <= 1.3e-6 and its 99th percentiles <= 1.2e-4.
GRAD_FACTOR = 3.0
GRAD_FLOOR = 2e-6
TERMS = ("color", "depth", "alpha", "all")
NAMES = {"means3D": "dL_dmeans3D", "means2D": "dL_dmeans2D", "opacities": "dL_dopacity", "shs": "dL_dsh", "scales": "dL_dscales",
         "rotations": "dL_drotations", "colors_precomp": "dL_dcolors", "cov3D_precomp": "dL_dcov3D"}


def _ours_backward(a, dc, dd, da):
    """Forward + backward through GaussianRasterizer with leaves that keep the case's shs layout (a 4-byte offset view stays a
    view of its flat buffer).  Returns (radii, {dL_d* name: gradient})."""
    from autovfx_b200.rasterizer import GaussianRasterizer
    leaves, inputs = {}, {}
    for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"):
        t = a[k]
        if t is None:
            inputs[k] = None
        elif k == "shs" and t.data_ptr() % 16:
            buf = torch.zeros(t.numel() + 1, device=t.device)
            buf[1:] = t.reshape(-1)
            leaves[k] = buf.requires_grad_(True)
            inputs[k] = buf[1:].view(t.shape)
            assert inputs[k].data_ptr() % 16 == t.data_ptr() % 16
        else:
            leaves[k] = inputs[k] = t.detach().clone().requires_grad_(True)
    means2D = torch.zeros_like(a["means3D"], requires_grad=True)
    rast = GaussianRasterizer(Hh.settings_from(a))
    color, depth, alpha, radii = rast(inputs["means3D"], means2D, inputs["opacities"], shs=inputs["shs"],
                                      colors_precomp=inputs["colors_precomp"], scales=inputs["scales"], rotations=inputs["rotations"],
                                      cov3D_precomp=inputs["cov3D_precomp"])
    ((color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()).backward()
    g = {NAMES[k]: (v.grad[1:].view(a[k].shape) if v.dim() == 1 and k == "shs" else v.grad) for k, v in leaves.items()}
    g["dL_dmeans2D"] = means2D.grad
    return radii, g


@pytest.fixture(scope="module", params=list(Hh.GRAD_FAMILIES))
def family(request, dev):
    a = Hh.grad_args(request.param, dev)
    fw = Hh.run_oracle(a)
    return request.param, a, fw, Hh.fp64_grads(a, fw, TERMS)


@pytest.mark.parametrize("term", TERMS)
def test_gradients_per_gaussian_against_fp64(family, term):
    name, a, fw, g64 = family
    dc, dd, da = Hh.isolated_image_grads(a, term, device=a["means3D"].device)
    radii, ours = _ours_backward(a, dc, dd, da)
    assert torch.equal(radii.cpu(), torch.from_numpy(fw["radii"]))  # same culling as the oracle whose decisions g64 replays
    ours = Hh.comparable_grads({k: v.cpu() for k, v in ours.items()}, a)
    orc = Hh.comparable_grads(Hh.oracle_backward(a, fw, dc, dd, da), a)
    checked = 0
    for k, want in g64[term].items():
        if float(want.abs().max()) == 0.0:  # e.g. dL/dsh under a depth-only loss
            assert float(ours[k].abs().max()) == 0.0, k
            continue
        e_gpu, e_orc = Hh.row_errors(ours[k], want), Hh.row_errors(orc[k], want)
        for q in (0.5, 0.99):
            got, base = float(np.quantile(e_gpu, q)), float(np.quantile(e_orc, q))
            assert got <= GRAD_FACTOR * base + GRAD_FLOOR, "%s %s %s: q%g per-row error %.3g, oracle %.3g" % (name, term, k, 100 * q, got, base)
        checked += 1
    assert checked >= 4


def test_gradients_that_must_be_exactly_zero(family):
    """dL/dsh beyond the active degree (hence beyond 16 coefficients for M = 25) and every gradient of a Gaussian that is not
    rendered (radii == 0) are exactly 0."""
    name, a, fw, _ = family
    dc, dd, da = Hh.image_grads(a, device=a["means3D"].device)
    radii, ours = _ours_backward(a, dc, dd, da)
    off = radii == 0
    assert off.any() and not off.all()
    for k, v in ours.items():
        assert torch.count_nonzero(v[off]) == 0, k
    if a["shs"] is not None:
        n = (min(a["sh_degree"], 3) + 1) ** 2
        assert torch.count_nonzero(ours["dL_dsh"][:, n:]) == 0
        assert torch.count_nonzero(ours["dL_dsh"][~off][:, :n]) > 0


def _clamped_alpha_args(dev):
    a = Hh.grad_args("M16_D3", dev, opacity_cap=1.0)
    a["opacities"] = a["opacities"].clone()
    a["opacities"][::3] = 0.995  # alpha reaches the 0.99 clamp near these centres
    return a


def test_clamped_alpha_gradients_against_oracle_and_reference(dev):
    """Where alpha is clamped at 0.99 the reference differentiates as if the clamp were absent; the GPU follows it.  Compared
    per Gaussian with the oracle (same quantiles as above, the oracle standing in for fp64) and with the compiled reference."""
    a = _clamped_alpha_args(dev)
    fw = Hh.run_oracle(a)
    dc, dd, da = Hh.image_grads(a, device=dev)
    radii, ours = _ours_backward(a, dc, dd, da)
    orc = Hh.oracle_backward(a, fw, dc, dd, da)
    assert torch.equal(radii.cpu(), torch.from_numpy(fw["radii"]))
    # alpha before the clamp, opacity * exp(power), at the pixel nearest each visible centre: several exceed 0.99
    vis = fw["radii"] > 0
    m2, co = fw["means2D"][vis].astype(np.float64), fw["conic_opacity"][vis].astype(np.float64)
    px = np.rint(m2)
    inside = (px[:, 0] >= 0) & (px[:, 0] < a["W"]) & (px[:, 1] >= 0) & (px[:, 1] < a["H"])
    d = m2 - px
    power = -0.5 * (co[:, 0] * d[:, 0] ** 2 + co[:, 2] * d[:, 1] ** 2) - co[:, 1] * d[:, 0] * d[:, 1]
    assert int(((co[:, 3] * np.exp(power) > 0.99) & inside).sum()) >= 5
    for k in ("dL_dmeans3D", "dL_dmeans2D", "dL_dopacity", "dL_dsh", "dL_dscales", "dL_drotations"):
        # measured on an H100: medians <= 1.2e-6, 99th percentiles <= 6.7e-5 (dL/dopacity)
        e = Hh.row_errors(ours[k].cpu(), torch.from_numpy(orc[k]).double())
        assert np.median(e) <= 1e-5 and np.quantile(e, 0.99) <= 5e-4, (k, np.median(e), np.quantile(e, 0.99))
    if not Hh.have_ref():
        pytest.skip("no compiled reference and no recorded reference values")
    gr = Hh.ref_backward(a, dc, dd, da)
    for k in ("dL_dmeans3D", "dL_dmeans2D", "dL_dopacity", "dL_dsh", "dL_dscales", "dL_drotations"):
        assert Hh.ref_relerr(ours[k], lambda: gr[k]) < 2e-4, k


# ---- C. per-process variants -------------------------------------------------------------------------------------------------
# the 16-byte aligned M = 16 rows take the vector staging at every degree
VARIANT_LAYOUTS = [(1, 0, False), (4, 1, False), (9, 2, False), (16, 0, False), (16, 2, False), (16, 3, True), (25, 3, False),
                   (25, 1, False), (None, 0, False)]
# named cases of test_gpu_parity.py (dense_tile: tiles of > 4096 instances; coplanar: equal depths, ties broken by id), a scene
# with tiles in each of the three sort regimes, so that the general (unpacked) path runs every per-tile sort, and the dense
# gradient cases that reach the blend backward's redo band, ballot block edge, partial footprints and deep termination
# (tests/helpers.DENSE_CASES)
VARIANT_CASES = ["dense_tile", "coplanar", "config1", "deg3_m25", "sort_regimes", "skip_band", "faint_slab"]


def _case_args(name, dev):
    return Hh.dense_case(name, dev)


def _variant_outputs(dev):
    """What the variants must reproduce: forward outputs of part of the layout matrix and of the named cases (exact and default
    mode) and backward of the named cases and of every gradient family, as a flat dict of CPU tensors."""
    out = {}
    for M, D, off in VARIANT_LAYOUTS:
        a = Hh.layout_args(M, D, off, dev)
        for exact in (True, False):
            for k, v in _forward(a, exact).items():
                out["%s/%s/%s" % (layout_id(M, D, off), exact, k)] = v
    for name in VARIANT_CASES:
        a = _case_args(name, dev)
        for exact in (True, False):
            for k, v in _forward(a, exact).items():
                out["%s/%s/%s" % (name, exact, k)] = v
        _, g = _ours_backward(a, *Hh.image_grads(a, device=dev))
        for k, v in g.items():
            out["%s/grad/%s" % (name, k)] = v.detach().cpu()
    for fam in Hh.GRAD_FAMILIES:
        a = Hh.grad_args(fam, dev)
        for k, v in _forward(a, False).items():
            out["%s/fw/%s" % (fam, k)] = v
        _, g = _ours_backward(a, *Hh.image_grads(a, device=dev))
        for k, v in g.items():
            out["%s/grad/%s" % (fam, k)] = v.detach().cpu()
    return out


def _tile_counts(ranges):
    r = ranges.long().reshape(-1, 2)
    return r[:, 1] - r[:, 0]


def _run_variant(env_update, tmp_path):
    out = tmp_path / ("variant_%s.npz" % "_".join("%s-%s" % kv for kv in env_update.items()))
    env = dict(os.environ, **env_update)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--variant-worker", str(out)]
    res = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return {k: torch.from_numpy(v) for k, v in np.load(out).items()}


@pytest.fixture(scope="module")
def default_outputs(dev):
    return _variant_outputs(dev)


def test_variant_cases_cover_every_tile_sort_regime(default_outputs):
    """The per-tile sort has three regimes: <= 2048 instances (single pass), <= 4096 (one shared-memory sort) and more (chunks
    merged through global memory).  The cases the variants replay must reach all three."""
    n = torch.cat([_tile_counts(default_outputs["%s/False/ranges" % c]) for c in VARIANT_CASES])
    assert ((n > 0) & (n <= 2048)).any() and ((n > 2048) & (n <= 4096)).any() and (n > 4096).any()


@pytest.mark.parametrize("env", [{"GSR_PACKED_KEYS": "0"}], ids=["packed_keys_off"])
def test_process_variant_matches_the_default_path(dev, default_outputs, env, tmp_path):
    got = _run_variant(env, tmp_path)
    assert sorted(got) == sorted(default_outputs)
    bad = []
    for k, want in default_outputs.items():
        if "/grad/" in k:
            # the backward accumulates with atomics, so the two runs agree per Gaussian, not in bits.  A reordered fp32 sum moves
            # a row by a few ulp of its largest terms: where terms of both signs cancel (dL/dopacity of coplanar) that is 6e-4 of
            # the row, while it stays ~2e-6 of the largest row (fp32 against fp64 on coplanar, CPU oracle).  Hence each row must
            # agree within 1e-4 of itself plus 2e-5 of the largest row, and half the rows within 2e-6 of themselves.
            g, w = got[k].double().reshape(want.shape[0], -1), want.double().reshape(want.shape[0], -1)
            d, n = (g - w).norm(dim=1), w.norm(dim=1)
            if n.numel() == 0 or float(n.max()) == 0.0:
                if torch.count_nonzero(d):
                    bad.append((k, "nonzero where the default is zero"))
                continue
            excess = float((d / (1e-4 * n + 2e-5 * n.max())).max())
            med = float(np.median(Hh.row_errors(g, w)))
            if excess > 1.0 or med > 2e-6:
                bad.append((k, "worst row at %.3g of its bound, median relative error %.3g" % (excess, med)))
        elif not torch.equal(got[k], want):
            bad.append((k, "differs"))
    assert not bad, bad


@pytest.mark.parametrize("P", [2 ** 24, 2 ** 24 + 16000], ids=["packed_ids", "wide_ids"])
def test_more_than_2_pow_24_gaussians_switch_to_the_general_path(dev, P):
    """Ids above 2^24 do not fit next to the packed footprint bits, so such scenes take the general sort and emission.  Only
    the last 16,000 Gaussians face the camera (the sort_regimes scene: tiles in all three sort regimes); the image must equal
    rendering those alone, bit for bit."""
    case = Hh.sort_regimes_case()
    front, cam = case["g"], case["cam"]
    n = front["means3D"].shape[0]
    colors = torch.rand(n, 3, generator=torch.Generator().manual_seed(72))
    small = dict(means3D=front["means3D"], opacities=front["opacities"], scales=front["scales"], rotations=front["rotations"],
                 colors_precomp=colors, shs=None, cov3D_precomp=None, view=cam.world_view_transform, proj=cam.full_proj_transform,
                 campos=cam.camera_center, W=cam.image_width, H=cam.image_height, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                 sh_degree=0, scale_modifier=1.0, bg=torch.tensor([0.1, 0.2, 0.3]))
    small = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in small.items()}
    want = _forward(small, False)
    t = _tile_counts(want["ranges"])
    assert ((t > 2048) & (t <= 4096)).any() and (t > 4096).any()
    # P - n Gaussians behind the camera: mirrored through the camera centre, they have view-space depth < 0 and are culled
    behind = (2 * small["campos"]).expand(P - n, 3)  # the camera looks at the origin
    big = dict(small)
    big["means3D"] = torch.cat([behind, small["means3D"]])
    big["opacities"] = torch.cat([torch.full((P - n, 1), 0.5, device=dev), small["opacities"]])
    big["scales"] = torch.cat([torch.full((P - n, 3), 0.01, device=dev), small["scales"]])
    big["rotations"] = torch.cat([torch.tensor([1.0, 0, 0, 0], device=dev).expand(P - n, 4), small["rotations"]])
    big["colors_precomp"] = torch.cat([torch.zeros(P - n, 3, device=dev), small["colors_precomp"]])
    got = _forward(big, False)
    del big
    assert torch.count_nonzero(got["radii"][:P - n]) == 0
    assert torch.equal(got["radii"][P - n:], want["radii"])
    assert torch.equal(got["point_list"].long() - (P - n), want["point_list"].long())
    for k in ("color", "depth", "alpha", "ranges", "n_contrib"):
        assert torch.equal(got[k], want[k]), k
    torch.cuda.empty_cache()


# ---- D. distCUDA2 against an exact k-d tree ----------------------------------------------------------------------------------

def _knn_exact(pts: torch.Tensor) -> torch.Tensor:
    """Mean of the three smallest squared distances to other points (self excluded by index, duplicates count), in float64."""
    from scipy.spatial import cKDTree
    p = pts.double().numpy()
    d, i = cKDTree(p).query(p, k=4)
    d2 = np.where(i == np.arange(len(p))[:, None], np.inf, d * d)
    d2.sort(axis=1)
    return torch.from_numpy(d2[:, :3].mean(axis=1))


def _dist2(pts, dev):
    from simple_knn._C import distCUDA2
    return distCUDA2(pts.to(dev)).cpu()


def _assert_knn_exact(got, pts):
    want = _knn_exact(pts)
    bad = (got.double() - want).abs() > 2e-6 * want
    assert not bad.any(), "%d of %d points, e.g. %s vs %s" % (int(bad.sum()), len(pts), got[bad][:4].tolist(), want[bad][:4].tolist())


@pytest.mark.parametrize("P", [1, 2, 3, 4, 5])
def test_dist2_tiny_point_counts(dev, P):
    """Fewer than four points leave FLT_MAX in the sum of the three nearest: the value must be the reference's, bit for bit."""
    pts = torch.randn(P, 3, generator=torch.Generator().manual_seed(100 + P)) * 0.7 + 0.2
    got = _dist2(pts, dev)
    if P >= 4:
        _assert_knn_exact(got, pts)
    elif not Hh.have_ref():
        pytest.skip("no compiled reference and no recorded reference values")
    if Hh.have_ref():
        from oracle import ref_cuda
        assert Hh.ref_same(got, lambda: ref_cuda.dist2(pts.to(dev)))


def test_dist2_coincident_points(dev):
    """5,000 copies of one point among 3,000 noise points: every copy has three neighbours at distance 0."""
    gen = torch.Generator().manual_seed(5)
    pts = torch.cat([torch.tensor([[0.3, -0.2, 0.1]]).expand(5000, 3), torch.randn(3000, 3, generator=gen) * 0.5])
    pts = pts[torch.randperm(len(pts), generator=gen)].contiguous()
    got = _dist2(pts, dev)
    _assert_knn_exact(got, pts)
    assert int((got == 0).sum()) == 5000


def test_dist2_planar_cloud(dev):
    """z == 0 everywhere: the bounding box has no extent along z (the Morton code divides 0 by 0 there)."""
    xy = torch.rand(20000, 2, generator=torch.Generator().manual_seed(6)) * 4 - 2
    pts = torch.cat([xy, torch.zeros(20000, 1)], dim=1)
    _assert_knn_exact(_dist2(pts, dev), pts)


def test_dist2_beyond_the_candidate_box_list(dev):
    """1.2M uniform points (1172 boxes of 1024) and a few far outliers: the CTA holding an outlier has a seed bound that lists
    more boxes than its candidate list holds, and falls back to testing every box (checked once with a counter in the kernel:
    the two CTAs holding outliers list all 1172 boxes)."""
    gen = torch.Generator().manual_seed(7)
    pts = torch.rand(1_200_000, 3, generator=gen) * 2 - 1
    pts[::240_000] = torch.tensor([[40.0, 35.0, -30.0], [-45.0, 30.0, 38.0], [33.0, -41.0, 44.0], [-39.0, -37.0, -36.0], [50.0, 0.0, 0.0]])
    _assert_knn_exact(_dist2(pts, dev), pts)


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--variant-worker":
    # fresh-process side of test_process_variant_matches_the_default_path (the library reads GSR_* once per process)
    res = _variant_outputs(torch.device("cuda:0"))
    np.savez(sys.argv[2], **{k: v.numpy() for k, v in res.items()})
