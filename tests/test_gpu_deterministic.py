"""Deterministic rasterizer gradients under torch.use_deterministic_algorithms(True) (gsr_backward_det).

1. repeatability: five backwards of the same frame give bit-identical gradients (compared as int32 views, so NaNs compare too);
2. scheduling: the same under a concurrent stream's large forward + backward, and in a fresh process;
3. the documented order: one backward per 8x4 footprint, the image gradients zero outside it, summed on the host in float32 in
   DESIGN.md §4's order, equals the full deterministic run bit for bit (means2D, opacity and colour gradients are those sums);
4. accuracy: within the per-row bound the suite holds the fused backward to against the default path, the golden reference
   gradients, and fp64 autograd;
5. trainers: 30 steps of train.py's loop with densification and the library's Adam, twice in fresh processes, end bit-identical;
   five render_sugar_raw backwards are bit-identical;
6. errors of gsr_backward_det: NULL, misaligned and too-small scratch.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = ["dense_tile", "big_splats", "config1", "coplanar", "deg3_m25", "small_precomp"]
ROW_REL, ROW_ABS = 5e-5, 1e-5  # the per-row bound test_gpu_fused_grads holds two summation orders of one gradient to
PIPE = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import rasterizer  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


@pytest.fixture
def deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was)


def _args(name, dev):
    return Hh.dense_case(name, dev) if name in Hh.DENSE_CASES else Hh.resolve(Hh.case_inputs(name), dev)


def _extra(P, dev):
    return torch.rand(P, 3, generator=torch.Generator().manual_seed(21)).to(dev)


def _grads(a, multi, loss_imgs=None):
    """One forward + backward through the autograd Function (rasterize_gaussians_multi with a second colour set when multi); the
    gradient of every input that has one."""
    from autovfx_b200.rasterizer import rasterize_gaussians, rasterize_gaussians_multi
    leaves = {k: a[k].detach().clone().requires_grad_(True) for k in ("means3D", "opacities", "shs", "colors_precomp", "scales",
                                                                      "rotations", "cov3D_precomp") if a[k] is not None}
    leaves["means2D"] = torch.zeros_like(leaves["means3D"], requires_grad=True)
    x = {k: leaves.get(k, torch.Tensor([])) for k in ("means3D", "means2D", "shs", "colors_precomp", "opacities", "scales", "rotations",
                                                       "cov3D_precomp")}
    if multi:
        leaves["extra"] = _extra(a["means3D"].shape[0], a["means3D"].device).requires_grad_(True)
        out = rasterize_gaussians_multi(x["means3D"], x["means2D"], x["shs"], x["colors_precomp"], leaves["extra"], x["opacities"],
                                        x["scales"], x["rotations"], x["cov3D_precomp"], Hh.settings_from(a))
        imgs = out[:4]
    else:
        imgs = rasterize_gaussians(x["means3D"], x["means2D"], x["shs"], x["colors_precomp"], x["opacities"], x["scales"], x["rotations"],
                                   x["cov3D_precomp"], Hh.settings_from(a))[:3]
    if loss_imgs is None:
        dc, dd, da = Hh.image_grads(a, device=a["means3D"].device)
        loss_imgs = (dc, dd, da, Hh.extra_image_grad(a, "all", device=a["means3D"].device))
    sum((o * w).sum() for o, w in zip(imgs, loss_imgs)).backward()
    return {k: v.grad.detach().clone() for k, v in leaves.items() if v.grad is not None}


def _assert_bits(got, want, what):
    assert sorted(got) == sorted(want), what
    for k in want:
        g, w = got[k].contiguous(), want[k].contiguous()
        assert g.shape == w.shape and torch.equal(g.view(torch.int32), w.view(torch.int32)), (what, k)


def _all_grads(dev):
    out = {}
    for name in CASES:
        a = _args(name, dev)
        for multi in (False, True):
            for k, v in _grads(a, multi).items():
                out["%s/%d/%s" % (name, multi, k)] = v.cpu()
    return out


@pytest.fixture(scope="module")
def det_grads(dev):
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        return _all_grads(dev)
    finally:
        torch.use_deterministic_algorithms(was)


# ---- 1. repeatability ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("multi", [False, True], ids=["single", "extra"])
def test_repeated_backwards_are_bit_identical(dev, deterministic, det_grads, name, multi):
    a = _args(name, dev)
    want = {k.split("/")[2]: v for k, v in det_grads.items() if k.startswith("%s/%d/" % (name, multi))}
    assert "means2D" in want and ("extra" in want) == multi
    for i in range(5):
        _assert_bits({k: v.cpu() for k, v in _grads(a, multi).items()}, want, (name, multi, i))


# ---- 2. scheduling independence ---------------------------------------------------------------------------------------------------
def test_bit_identical_next_to_a_concurrent_stream(dev, deterministic, det_grads):
    from autovfx_b200 import scene
    big = Hh.resolve(dict(g=scene.config3_scene(P=300_000), cam=Hh.case_inputs("config1")["cam"], sh_degree=3, bg=(0.0, 0.0, 0.0),
                          scale_modifier=1.0), dev)
    side = torch.cuda.Stream(dev)
    for name in CASES:
        a = _args(name, dev)
        for multi in (False, True):
            torch.cuda.synchronize(dev)
            with torch.cuda.stream(side):
                _grads(big, True)  # a large forward + backward queued on the other stream
                _grads(big, False)
            got = _grads(a, multi)
            torch.cuda.synchronize(dev)
            want = {k.split("/")[2]: v for k, v in det_grads.items() if k.startswith("%s/%d/" % (name, multi))}
            _assert_bits({k: v.cpu() for k, v in got.items()}, want, (name, multi))


def test_bit_identical_in_a_fresh_process(det_grads, tmp_path):
    path = tmp_path / "det.npz"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--det-worker", str(path)]
    res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    got = {k: torch.from_numpy(v) for k, v in np.load(path).items()}
    _assert_bits(got, det_grads, "fresh process")


# ---- 3. the documented summation order, bit for bit ------------------------------------------------------------------------------
def test_sum_order_is_the_documented_one(dev, deterministic):
    """small_precomp renders on 5 x 5 tiles.  A backward whose image gradients are zero outside one footprint returns that footprint's
    partials (every other visited partial is +-0, and adding +-0 to a sum that starts from +0.0 changes nothing); summing them over
    all footprints in the order ty, tx, f on the host must give the full run's bits."""
    from autovfx_b200.rasterizer import rasterize_gaussians
    a = _args("small_precomp", dev)
    W, H = a["W"], a["H"]
    assert a["colors_precomp"] is not None and W % 16 == 0 and H % 16 == 0
    leaves = {k: a[k].detach().clone().requires_grad_(True) for k in ("means3D", "opacities", "colors_precomp", "cov3D_precomp")}
    m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
    e = torch.Tensor([])
    color, depth, alpha, radii = rasterize_gaussians(leaves["means3D"], m2d, e, leaves["colors_precomp"], leaves["opacities"], e, e,
                                                     leaves["cov3D_precomp"], Hh.settings_from(a))
    dc, dd, da = Hh.image_grads(a, device=dev)
    ins = [m2d, leaves["opacities"], leaves["colors_precomp"]]

    def run(mask):
        g = torch.autograd.grad((color, depth, alpha), ins, (dc * mask, dd * mask, da * mask), retain_graph=True)
        return torch.cat([g[0][:, :2], g[1].reshape(-1, 1), g[2]], dim=1).cpu().numpy()

    full = run(torch.ones(H, W, device=dev))
    acc = np.zeros_like(full)
    nonzero = 0
    for ty in range(H // 16):
        for tx in range(W // 16):
            for f in range(8):
                mask = torch.zeros(H, W, device=dev)
                y0, x0 = 16 * ty + 4 * (f >> 1), 16 * tx + 8 * (f & 1)
                mask[y0:y0 + 4, x0:x0 + 8] = 1.0
                part = run(mask)
                nonzero += int(np.count_nonzero(part))
                acc = (acc + part).astype(np.float32)  # float32 + float32: one IEEE rounding per add, in order
    assert nonzero > 1000
    assert np.array_equal(acc.view(np.int32), full.view(np.int32)), int((acc != full).sum())


# ---- 4. accuracy ----------------------------------------------------------------------------------------------------------------------
def _row_share(got, want):
    """Worst row's share of the bound ROW_REL ||want_row|| + ROW_ABS max_row ||want_row||."""
    g, w = got.double().cpu().reshape(want.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    d, n = (g - w).norm(dim=1), w.norm(dim=1)
    if float(n.max()) == 0.0:
        return 0.0 if not torch.count_nonzero(d) else math.inf
    return float((d / (ROW_REL * n + ROW_ABS * n.max())).max())


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("multi", [False, True], ids=["single", "extra"])
def test_deterministic_rows_match_the_default_path(dev, det_grads, name, multi):
    a = _args(name, dev)
    default = _grads(a, multi)  # the flag is off here: the atomic path
    want = {k.split("/")[2]: v for k, v in det_grads.items() if k.startswith("%s/%d/" % (name, multi))}
    assert sorted(default) == sorted(want)
    for k, v in want.items():
        assert torch.isfinite(v).all() == torch.isfinite(default[k]).all(), (name, k)
        share = _row_share(v, default[k])
        assert share <= 1.0, (name, multi, k, share)


@pytest.mark.parametrize("case", ["config1", "deg3_m25"])
def test_deterministic_gradients_match_the_golden_reference(dev, deterministic, case):
    gold = Hh.load_golden(os.path.join(ROOT, "tests", "golden", case + ".npz"))
    a = Hh.resolve(Hh.case_inputs(case), dev)
    dc, dd, da = Hh.image_grads(a, device=dev)
    _, g = Hh.ours_backward(a, dc, dd, da)
    pairs = [("means3D", "dL_dmeans3D"), ("means2D", "dL_dmeans2D"), ("opacities", "dL_dopacity"), ("scales", "dL_dscales"),
             ("rotations", "dL_drotations")]
    for mine, theirs in pairs:
        assert Hh.relerr(g[mine].reshape(gold[theirs].shape), gold[theirs]) < 2e-4, mine


@pytest.mark.parametrize("family", ["precomp", "M16_D3"])
def test_deterministic_rows_against_fp64(dev, family):
    a = Hh.grad_args(family, dev)
    fw = Hh.run_oracle(a)
    g64 = Hh.fp64_grads(a, fw, ("all",), oracle_decisions=True)["all"]
    dc, dd, da = Hh.isolated_image_grads(a, "all", device=dev)
    default = Hh.ours_backward(a, dc, dd, da)[1]
    torch.use_deterministic_algorithms(True)
    try:
        det = Hh.ours_backward(a, dc, dd, da)[1]
    finally:
        torch.use_deterministic_algorithms(False)
    names = {"means3D": "dL_dmeans3D", "opacities": "dL_dopacity", "shs": "dL_dsh", "scales": "dL_dscales", "rotations": "dL_drotations",
             "colors_precomp": "dL_dcolors", "cov3D_precomp": "dL_dcov3D", "means2D": "dL_dmeans2D"}
    checked = 0
    for k, key in names.items():
        if det.get(k) is None or key not in g64:
            continue
        want = g64[key]
        got_d, got_a = det[k], default[k]
        if k == "means2D":
            got_d, got_a = got_d[:, :2], got_a[:, :2]
        e_det, e_def = Hh.row_errors(got_d, want), Hh.row_errors(got_a, want)
        assert np.quantile(e_det, 0.99) <= 2.0 * np.quantile(e_def, 0.99) + 1e-6, (family, k)
        assert e_det.max() <= 2.0 * e_def.max() + 1e-5, (family, k)
        checked += 1
    assert checked >= 4


# ---- 5. trainers ------------------------------------------------------------------------------------------------------------------------
def _train(dev):
    """30 steps of train.py's loop on a small seeded scene: render_raw, the objective with the normal terms, backward, the
    densification statistics, densify_and_prune at steps 10 and 20 (clone and split), the library's Adam."""
    from torch import nn
    from autovfx_b200 import densify, losses, renderer
    from autovfx_b200.optim import use_cuda_adam
    from tests.test_gpu_fused_grads import _cam
    c = Hh.case_inputs("small_sh")
    g = c["g"]
    op = g["opacities"].clamp(1e-4, 1 - 1e-4)
    raw = {"xyz": g["means3D"], "f_dc": g["shs"][:, :1], "f_rest": g["shs"][:, 1:], "opacity": torch.log(op / (1 - op)),
           "scaling": torch.log(g["scales"]), "rotation": g["rotations"]}
    attrs = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
             "rotation": "_rotation"}
    lrs = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 0.05, "scaling": 5e-3, "rotation": 1e-3}
    m = types.SimpleNamespace()
    for n, at in attrs.items():
        setattr(m, at, nn.Parameter(raw[n].detach().clone().to(dev).contiguous().requires_grad_(True)))
    m.optimizer = use_cuda_adam(torch.optim.Adam([{"params": [getattr(m, at)], "lr": lrs[n], "name": n} for n, at in attrs.items()],
                                                 lr=0.0, eps=1e-15))
    P = m._xyz.shape[0]
    m.xyz_gradient_accum, m.denom = torch.zeros(P, 1, device=dev), torch.zeros(P, 1, device=dev)
    m.max_radii2D = torch.zeros(P, device=dev)
    m.percent_dense = 0.01
    m.scaling_activation, m.opacity_activation = torch.exp, torch.sigmoid
    m.rotation_activation = torch.nn.functional.normalize
    m.active_sh_degree, m.max_sh_degree = 3, 3
    cam, bg = _cam(c["cam"], dev), torch.tensor(c["bg"], device=dev)
    gt = torch.rand(4, c["cam"].image_height, c["cam"].image_width, generator=torch.Generator().manual_seed(5)).to(dev)
    sizes = [P]
    for it in range(30):
        out = renderer.render_raw(cam, m, PIPE, bg)
        loss = losses.photometric_loss(out["render"], gt, 0.2) + 0.01 * losses.normal_loss(out["normal"], out["pseudo_normal"].detach())
        loss = loss + 0.1 * losses.anisotropic_loss(torch.exp(m._scaling))
        loss.backward()
        with torch.no_grad():
            densify.update_densification_stats(m, out["viewspace_points"], out["radii"], out["visibility_filter"])
        m.optimizer.step()
        m.optimizer.zero_grad(set_to_none=True)
        if it in (9, 19):
            densify.densify_and_prune(m, 1e-6, 0.005, 4.0, 20)  # percent_dense * extent = 0.04: small ones clone, large ones split
            sizes.append(m._xyz.shape[0])
    res = {"sizes": np.asarray(sizes)}
    for n, at in attrs.items():
        p = getattr(m, at)
        res[n] = p.detach().cpu().numpy()
        st = m.optimizer.state[p]
        res[n + "/exp_avg"], res[n + "/exp_avg_sq"] = st["exp_avg"].cpu().numpy(), st["exp_avg_sq"].cpu().numpy()
    return res


def test_training_runs_are_bit_identical(tmp_path):
    outs = []
    for i in range(2):
        path = tmp_path / ("train%d.npz" % i)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--train-worker", str(path)]
        res = subprocess.run(cmd, env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"), cwd=ROOT, capture_output=True, text=True,
                             timeout=900)
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        outs.append(dict(np.load(path)))
    a, b = outs
    sizes = a["sizes"]
    assert sizes[1] > sizes[0] and sizes[2] > sizes[1], sizes  # both densifications added Gaussians
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.int32) if a[k].dtype == np.float32 else a[k],
                                                           b[k].view(np.int32) if b[k].dtype == np.float32 else b[k]), k


def test_render_sugar_raw_backwards_are_bit_identical(dev, deterministic):
    from autovfx_b200.renderer import render_sugar_raw
    from tests import sugar_colors_ref as SC
    from tests import test_gpu_sugar_render as TS
    model = TS._scene(dev, M=16, grad=True)
    model.__class__ = SC.SugarModel4
    leaves = {k: v for k, v in vars(model).items() if isinstance(v, torch.Tensor) and v.requires_grad}
    assert leaves
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    want = None
    for i in range(5):
        for v in leaves.values():
            v.grad = None
        img = render_sugar_raw(model, camera_indices=1, bg_color=bg, sh_deg=3)
        w = torch.randn(img.shape, generator=torch.Generator().manual_seed(3)).to(dev)
        (img * w).sum().backward()
        got = {k: v.grad.detach().cpu().clone() for k, v in leaves.items() if v.grad is not None}
        assert len(got) >= 3
        if want is None:
            want = got
        else:
            _assert_bits(got, want, i)


# ---- 6. errors ------------------------------------------------------------------------------------------------------------------------
def test_scratch_errors(dev):
    from autovfx_b200 import _lib
    from autovfx_b200 import rasterizer as R
    a = Hh.resolve(Hh.case_inputs("small_sh"), dev)
    s = Hh.settings_from(a)
    color, depth, alpha, radii, (geom, binning, image), ticket, keep = R.forward_raw(
        a["means3D"], a["shs"], None, a["opacities"], a["scales"], a["rotations"], None, s, for_backward=True, sync=True)
    P, W, H, M = a["means3D"].shape[0], a["W"], a["H"], a["shs"].shape[1]
    fr = _lib.gsr_frame()
    R._fill_frame(fr, P, a["sh_degree"], M, W, H, s, keep[7], keep[0], keep[1], None, None, keep[4], keep[5], None, keep[8], keep[9],
                  keep[10])
    ws = R._workspace(geom, binning, image)
    f32 = dict(dtype=torch.float32, device=dev)
    bufs = [torch.zeros(P, n, **f32) for n in (3, 4, 1, 3, 1, 3, 6, 3 * M, 3, 4)]
    gr = _lib.gsr_grads(*[b.data_ptr() for b in bufs])
    dc, dd, da = Hh.image_grads(a, device=dev)
    R_ = ticket.stats()["num_rendered"]
    need = _lib.lib.gsr_backward_det_bytes(R_, W, H, 0)
    scratch = torch.empty(need + 64, dtype=torch.uint8, device=dev)
    L = _lib.lib

    def call(ptr, nbytes):
        return L.gsr_backward_det(C.byref(fr), C.byref(ws), radii.data_ptr(), alpha.data_ptr(), dc.data_ptr(), dd.data_ptr(), da.data_ptr(),
                                  None, None, None, C.byref(gr), ptr, nbytes, _lib.stream_ptr(dev))

    assert call(None, need) == -1 and b"scratch is NULL" in L.gsr_last_error()
    assert call(scratch.data_ptr() + 4, need) == -1 and b"16-byte aligned" in L.gsr_last_error()
    small = L.gsr_backward_det_bytes(0, W, H, 0) - 16
    assert call(scratch.data_ptr(), small) == -2 and b"too small" in L.gsr_last_error()
    torch.cuda.synchronize(dev)
    assert all(int(torch.count_nonzero(b)) == 0 for b in bufs)  # nothing was enqueued
    assert call(scratch.data_ptr(), need) == 0
    torch.cuda.synchronize(dev)
    assert int(torch.count_nonzero(bufs[0])) > 0
    # a scratch sized for fewer instances than the frame rendered: no write beyond it, NaN rows where partials did not fit
    assert call(scratch.data_ptr(), L.gsr_backward_det_bytes(R_ // 2, W, H, 0)) == 0
    torch.cuda.synchronize(dev)
    assert bool(torch.isnan(bufs[0]).any())


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--det-worker":
    torch.use_deterministic_algorithms(True)
    res = _all_grads(torch.device("cuda:0"))
    np.savez(sys.argv[2], **{k: v.numpy() for k, v in res.items()})

if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--train-worker":
    torch.use_deterministic_algorithms(True)
    torch.manual_seed(0)  # train.py's safe_state: the split's draws from the CUDA generator
    np.savez(sys.argv[2], **_train(torch.device("cuda:0")))
