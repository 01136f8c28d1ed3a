"""The training objective in CUDA (autovfx_b200.losses) on an H100, run with -m gpu.  Every value and every gradient element is held
to the per-element float32 error bound tests/losses_ref.py derives from the operand magnitudes around its fp64 restatement, and
the reference's own float32 torch graph (loss_utils.l1_loss / ssim / normal_loss / anisotropic_loss, restated below) is held to
the same bound.  Also: the trainers' layouts and edge shapes, ties, determinism, no host synchronisation, and one train.py
objective on render_raw outputs end to end."""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tests import losses_ref as LR  # noqa: E402

pytestmark = pytest.mark.gpu
LAMBDA_DSSIM = 0.2


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import losses  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


# -- the reference's float32 graph (loss_utils.py), for the same bound ----------------------------------------------------------
def torch_ssim(x, y):
    from autovfx_b200.losses import ssim_window
    w1 = ssim_window().unsqueeze(1)
    ch = x.size(-3)
    win = w1.mm(w1.t()).float().unsqueeze(0).unsqueeze(0).expand(ch, 1, 11, 11).contiguous().to(x.device)
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=ch), F.conv2d(y, win, padding=5, groups=ch)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = F.conv2d(x * x, win, padding=5, groups=ch) - mu1_sq
    s2 = F.conv2d(y * y, win, padding=5, groups=ch) - mu2_sq
    s12 = F.conv2d(x * y, win, padding=5, groups=ch) - mu1_mu2
    return (((2 * mu1_mu2 + LR.C1) * (2 * s12 + LR.C2)) / ((mu1_sq + mu2_sq + LR.C1) * (s1 + s2 + LR.C2))).mean()


def torch_photometric(x, y, lam=LAMBDA_DSSIM):
    return (1.0 - lam) * torch.abs(x - y).mean() + lam * (1.0 - torch_ssim(x, y))


def torch_normal_loss(network_output, gt, depth=None, scene_scale=5.0):
    n, g = F.normalize(network_output, p=2, dim=-1), F.normalize(gt, p=2, dim=-1)
    if depth is not None:
        mask = torch.logical_and(depth > 0, depth < scene_scale)
        n, g = n[mask], g[mask]
    return torch.abs(n - g).mean() + 0.1 * (-torch.sum(n * g, axis=-1).mean())


def torch_anisotropic_loss(s, r=3):
    return torch.mean(torch.clamp(torch.max(s, dim=-1).values / (torch.min(s, dim=-1).values + 1e-6), min=r) - r)


def _grad_of(fn, x, *args):
    xr = x.detach().clone().requires_grad_(True)
    v = fn(xr, *args)
    v.backward()
    return v.detach(), xr.grad


def _assert_within(got, want, bound, what):
    err = (got.double() - want.double()).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), float((err / bound.clamp_min(1e-300)).max()))


# -- photometric term ------------------------------------------------------------------------------------------------------------
def _images(kind, dev):
    gen = torch.Generator().manual_seed(len(kind))
    r = lambda *s: torch.rand(*s, generator=gen)  # noqa: E731
    if kind == "1080p":
        return r(4, 1080, 1920), r(4, 1080, 1920)
    if kind == "coarse_hwc":  # coarse_density's [1,4,H,W] render against a channel-innermost view of the ground truth
        return r(1, 4, 270, 481), r(270, 481, 4).permute(2, 0, 1).unsqueeze(0)
    if kind == "c3":
        return r(3, 64, 80), r(3, 64, 80)
    if kind == "batch":
        return r(3, 2, 40, 50), r(3, 2, 40, 50)
    if kind == "below_window":
        return r(4, 7, 9), r(4, 7, 9)
    if kind == "one_pixel":
        return r(1, 1, 1, 1), r(1, 1, 1, 1)
    if kind == "thin":
        return r(2, 5, 200), r(2, 200, 5).transpose(1, 2)
    if kind == "tile_remainder":
        return r(1, 3, 33, 65), r(1, 3, 33, 65)
    if kind == "constant":  # sigma = 0 over whole windows, and exact ties of the L1 term
        x = torch.full((3, 48, 64), 0.25)
        x[:, :, 32:] = 0.75
        y = x.clone()
        y[:, 24:] = 0.5
        return x, y
    if kind == "outside01":
        return r(4, 50, 70) * 5 - 2, r(4, 50, 70) * 3 - 1
    raise KeyError(kind)


PHOTO_KINDS = ["1080p", "coarse_hwc", "c3", "batch", "below_window", "one_pixel", "thin", "tile_remainder", "constant", "outside01"]


@pytest.mark.parametrize("kind", PHOTO_KINDS)
def test_photometric_values_and_gradients(dev, kind):
    from autovfx_b200 import losses as L
    x, y = (t.to(dev) for t in _images(kind, dev))
    lam = LAMBDA_DSSIM
    l1_64, s64, g64, parts = LR.photometric64(x, y, g_l1=1.0 - lam, g_ssim=-lam)
    sb, gb = LR.photometric_bounds(parts, g_l1=1.0 - lam, g_ssim=-lam)
    l1b = 64 * LR.U32 * float(l1_64)
    ref64 = (1.0 - lam) * float(l1_64) + lam * (1.0 - float(s64))
    vb = (1.0 - lam) * l1b + lam * sb + 4 * LR.U32 * abs(ref64)
    xr = x.clone().requires_grad_(True)
    s = L.ssim(xr, y)
    assert s.dim() == 0 and s.is_cuda and s.dtype == torch.float32
    assert abs(float(s) - float(s64)) <= sb, (kind, float(s) - float(s64), sb)
    v = L.photometric_loss(xr, y, lam)
    v.backward()
    assert abs(float(v) - ref64) <= vb, (kind, float(v) - ref64, vb)
    _assert_within(xr.grad, g64, gb, (kind, "library gradient"))
    tv, tg = _grad_of(torch_photometric, x, y)
    assert abs(float(tv) - ref64) <= vb, (kind, "torch value", float(tv) - ref64, vb)
    _assert_within(tg, g64, gb, (kind, "torch gradient"))


def test_ssim_alone_gradient(dev):
    from autovfx_b200 import losses as L
    x, y = (t.to(dev) for t in _images("tile_remainder", dev))
    _, _, g64, parts = LR.photometric64(x, y, g_l1=0.0, g_ssim=1.0)
    _, gb = LR.photometric_bounds(parts, g_l1=0.0, g_ssim=1.0)
    xr = x.clone().requires_grad_(True)
    L.ssim(xr, y).backward()
    _assert_within(xr.grad, g64, gb, "ssim alone")


def test_nan_pixel_makes_the_loss_nan(dev):
    from autovfx_b200 import losses as L
    x, y = (t.to(dev) for t in _images("c3", dev))
    x[1, 10, 20] = float("nan")
    assert torch.isnan(L.ssim(x, y)) and torch.isnan(L.photometric_loss(x, y, LAMBDA_DSSIM))
    assert torch.isnan(torch_ssim(x, y))


def test_no_grad_keeps_nothing(dev):
    from autovfx_b200 import losses as L
    x, y = (t.to(dev) for t in _images("c3", dev))
    xr = x.clone().requires_grad_(True)
    with torch.no_grad():
        for v in (L.ssim(xr, y), L.photometric_loss(xr, y, 0.2), L.normal_loss(xr.permute(1, 2, 0), y.permute(1, 2, 0)),
                  L.anisotropic_loss(xr.reshape(-1, 3))):
            assert v.grad_fn is None and not v.requires_grad
    assert L.ssim(x, y).grad_fn is None


# -- normal term -----------------------------------------------------------------------------------------------------------------
def _normals(dev, H=270, W=480):
    gen = torch.Generator().manual_seed(11)
    n = torch.randn(H, W, 3, generator=gen)
    n[:5, :7] = 0.0                     # zero norm: below the clamp
    n[5, :3] *= 1e-14                   # below the clamp, not zero
    g = torch.randn(3, H, W, generator=gen).permute(1, 2, 0)  # pseudo_normal's layout: an HWC view of a CHW map
    g[0, :2] = 0.0
    depth = torch.rand(H, W, generator=gen) * 7 - 1
    return n.to(dev), g.to(dev), depth.to(dev)


@pytest.mark.parametrize("masked", [False, True], ids=["all", "depth"])
def test_normal_loss_values_and_gradients(dev, masked):
    from autovfx_b200 import losses as L
    n, g, depth = _normals(dev)
    d = depth if masked else None
    v64, g64, gb = LR.normal64(n, g, d)
    vb = 64 * LR.U32 * (abs(float(v64)) + 0.2)
    nr = n.clone().requires_grad_(True)
    v = L.normal_loss(nr, g, d)
    v.backward()
    assert v.dim() == 0 and abs(float(v) - float(v64)) <= vb, (float(v) - float(v64), vb)
    _assert_within(nr.grad, g64, gb, ("library", masked))
    tv, tg = _grad_of(torch_normal_loss, n, g, d)
    assert abs(float(tv) - float(v64)) <= vb
    _assert_within(tg, g64, gb, ("torch", masked))
    assert torch.count_nonzero(nr.grad[:5, :7]) > 0  # the zero-norm pixels carry the clamp's gradient, as in torch


def test_normal_loss_empty_mask(dev):
    from autovfx_b200 import losses as L
    n, g, depth = _normals(dev, 16, 16)
    nr = n.clone().requires_grad_(True)
    v = L.normal_loss(nr, g, torch.full_like(depth, -1.0))
    v.backward()
    assert torch.isnan(v) and torch.isnan(torch_normal_loss(n, g, torch.full_like(depth, -1.0)))
    assert (nr.grad == 0).all()


# -- anisotropic term ------------------------------------------------------------------------------------------------------------
def _ratio_exactly_r():
    """A row whose max / (min + 1e-6) is exactly 3 in float32."""
    d = torch.tensor(0.5)
    mn = torch.tensor(0.5) - torch.tensor(1e-6)
    while float(mn + torch.tensor(1e-6)) != 0.5:
        mn = torch.nextafter(mn, d)
    row = torch.tensor([float(mn), 1.5, 0.9])
    assert float(row[1] / (row[0] + 1e-6)) == 3.0
    return row


def _scales(P, seed=5):
    gen = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.randn(P, 3, generator=gen) * 1.5 - 4)
    return s


TIE_ROWS = torch.tensor([[2.0, 2.0, 0.1], [0.1, 2.0, 2.0], [2.0, 0.1, 2.0], [0.1, 0.1, 2.0], [2.0, 0.1, 0.1], [0.1, 2.0, 0.1],
                         [0.5, 0.5, 0.5], [0.0, 0.0, 1.0], [0.0, 1e-3, 0.0], [0.0, 0.0, 0.0], [1e-8, 1.0, 1e-8]])


@pytest.mark.parametrize("P", [1, 20_000, 3_000_000])
def test_anisotropic_loss_values_and_gradients(dev, P):
    from autovfx_b200 import losses as L
    s = _scales(P)
    if P > 1:
        s[:len(TIE_ROWS)] = TIE_ROWS
        s[len(TIE_ROWS)] = _ratio_exactly_r()
        s[len(TIE_ROWS) + 1:len(TIE_ROWS) + 20] = 0.0
    s = s.to(dev)
    v64, g64, gb = LR.anisotropic64(s)
    vb = 64 * LR.U32 * abs(float(v64)) + 1e-30
    sr = s.clone().requires_grad_(True)
    v = L.anisotropic_loss(sr)
    v.backward()
    assert v.dim() == 0 and abs(float(v) - float(v64)) <= vb, (float(v) - float(v64), vb)
    _assert_within(sr.grad, g64, gb, "library")
    tv, tg = _grad_of(torch_anisotropic_loss, s)
    assert abs(float(tv) - float(v64)) <= vb
    _assert_within(tg, g64, gb, "torch")
    if P > 1:
        k = len(TIE_ROWS) + 1
        assert torch.equal(sr.grad[:k] != 0, tg[:k] != 0)  # same receiving index on every tie, and clamp_min's rule at ratio == r
        assert sr.grad[len(TIE_ROWS)].abs().sum() > 0


def test_torch_tie_indices_on_this_gpu(dev):
    """torch's max(dim) / min(dim) on the GPU return the first extreme index on 2- and 3-way ties: the rule the backward follows."""
    s = TIE_ROWS.to(dev)
    imax, imin = LR.first_extremes(s)
    assert torch.equal(torch.max(s, dim=-1).indices, imax)
    assert torch.equal(torch.min(s, dim=-1).indices, imin)
    assert imax.tolist()[:7] == [0, 1, 0, 2, 0, 1, 0] and imin.tolist()[:7] == [2, 0, 1, 0, 1, 0, 0]


# -- determinism and synchronisation --------------------------------------------------------------------------------------------
def _objective_grads(dev, x, y, n, g, s):
    from autovfx_b200 import losses as L
    xr, nr, sr = (t.clone().requires_grad_(True) for t in (x, n, s))
    parts = (L.photometric_loss(xr, y, LAMBDA_DSSIM), L.normal_loss(nr, g), L.anisotropic_loss(sr))
    (parts[0] + 0.01 * parts[1] + 0.1 * parts[2]).backward()
    return [p.detach() for p in parts] + [xr.grad, nr.grad, sr.grad]


def test_determinism(dev):
    x, y = (t.to(dev) for t in _images("1080p", dev))
    n, g, _ = _normals(dev, 1080, 1920)
    s = _scales(3_000_000).to(dev)
    a = _objective_grads(dev, x, y, n, g, s)
    b = _objective_grads(dev, x, y, n, g, s)
    for u, v in zip(a, b):
        assert torch.equal(u, v) or (torch.isnan(u).equal(torch.isnan(v)) and torch.equal(u.nan_to_num(), v.nan_to_num()))


def test_no_host_synchronisation(dev):
    from autovfx_b200 import losses as L
    x, y = (t.to(dev) for t in _images("tile_remainder", dev))
    n, g, depth = _normals(dev, 32, 40)
    s = _scales(1000).to(dev)
    xr, nr, sr = (t.clone().requires_grad_(True) for t in (x, n, s))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = L.photometric_loss(xr, y, LAMBDA_DSSIM) + L.ssim(xr, y) + 0.01 * L.normal_loss(nr, g, depth) + \
            0.1 * L.anisotropic_loss(sr)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert xr.grad is not None and nr.grad is not None and sr.grad is not None


# -- end to end: train.py's objective on render_raw outputs ---------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small_sh", "config1"])
def test_train_objective_on_render_raw(dev, name):
    """train.py:98-132 with train_3dgs.sh's lambdas (dssim 0.2, pseudo-normal 0.01, anisotropic 0.1) on render_raw outputs: the raw
    parameter gradients through the library's objective against the same render with the torch objective, within
    test_gpu_raw_render.py's end-to-end bound."""
    from autovfx_b200 import losses as L, renderer
    from tests.test_gpu_raw_render import PIPE, _RawPC, _assert_e2e, _case
    raw, cam, bg, D, mod, offset = _case(name, dev)
    H, W = int(cam.image_height), int(cam.image_width)
    gt = torch.rand(4, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    grads = {}
    for which in ("library", "torch"):
        pc = _RawPC(raw, D, offset)
        out = renderer.render_raw(cam, pc, PIPE, bg, scaling_modifier=mod)
        scaling = torch.exp(pc._scaling)
        if which == "library":
            loss = L.photometric_loss(out["render"], gt, 0.2) + 0.01 * L.normal_loss(out["normal"], out["pseudo_normal"].detach()) + \
                0.1 * L.anisotropic_loss(scaling)
        else:
            loss = torch_photometric(out["render"], gt, 0.2) + \
                0.01 * torch_normal_loss(out["normal"], out["pseudo_normal"].detach()) + 0.1 * torch_anisotropic_loss(scaling)
        loss.backward()
        grads[which] = pc.grads()
    _assert_e2e(grads["library"], grads["torch"], name)
