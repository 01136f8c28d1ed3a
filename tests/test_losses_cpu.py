"""CPU checks of the training objective (autovfx_b200.losses): the fp64 restatement of tests/losses_ref.py against fp64 autograd of
the reference formulas (sugar/gaussian_splatting/utils/loss_utils.py), the separable window against create_window's 2-D one, every
argument error, CPU tensors, and the exports."""
from __future__ import annotations

import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tests import losses_ref as LR  # noqa: E402


def _ssim_autograd64(x, y):
    """The reference's _ssim (grouped 11x11 conv2d, padding 5) in fp64 with the exact 2-D window."""
    w = LR.window64()
    ch = x.shape[-3]
    win = torch.outer(w, w).expand(ch, 1, 11, 11).contiguous()
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=ch), F.conv2d(y, win, padding=5, groups=ch)
    s1 = F.conv2d(x * x, win, padding=5, groups=ch) - mu1.pow(2)
    s2 = F.conv2d(y * y, win, padding=5, groups=ch) - mu2.pow(2)
    s12 = F.conv2d(x * y, win, padding=5, groups=ch) - mu1 * mu2
    m = ((2 * mu1 * mu2 + LR.C1) * (2 * s12 + LR.C2)) / ((mu1.pow(2) + mu2.pow(2) + LR.C1) * (s1 + s2 + LR.C2))
    return m.mean()


@pytest.mark.parametrize("shape", [(1, 3, 17, 23), (2, 4, 12, 9), (1, 1, 5, 7), (1, 2, 1, 1)])
def test_photometric_restatement_matches_fp64_autograd(shape):
    gen = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=gen, dtype=torch.float64) * 1.4 - 0.2
    y = torch.rand(shape, generator=gen, dtype=torch.float64)
    y.view(-1)[::5] = x.detach().view(-1)[::5]  # exact ties of the L1 term
    xr = x.clone().requires_grad_(True)
    ref = 0.8 * (xr - y).abs().mean() + 0.2 * (1.0 - _ssim_autograd64(xr, y))
    ref.backward()
    l1, s, g, _ = LR.photometric64(x, y, g_l1=0.8, g_ssim=-0.2)
    assert abs(float(0.8 * l1 + 0.2 * (1 - s)) - ref.item()) < 1e-14
    torch.testing.assert_close(g, xr.grad, rtol=1e-10, atol=1e-15)


def test_separable_window_within_rounding_of_2d_window():
    """create_window's 2-D window is the float32 product of the 1-D weights, one rounding each: the separable application uses the
    unrounded products, within one unit roundoff of every 2-D weight.  The float32 1-D weights are within a few units of the
    exact Gaussian."""
    from autovfx_b200.losses import ssim_window
    w = ssim_window()
    assert w.dtype == torch.float32 and w.shape == (11,)
    w2 = w.unsqueeze(1).mm(w.unsqueeze(1).t())  # create_window's expression
    exact = torch.outer(w.double(), w.double())
    assert ((w2.double() - exact).abs() <= LR.U32 * exact).all()
    assert ((w.double() - LR.window64()).abs() <= 4 * LR.U32 * LR.window64()).all()


@pytest.mark.parametrize("masked", [False, True])
def test_normal_restatement_matches_fp64_autograd(masked):
    gen = torch.Generator().manual_seed(7)
    pred = torch.randn(9, 11, 3, generator=gen, dtype=torch.float64)
    pred[0, 0] = 0.0  # zero norm: below the clamp
    gt = torch.randn(9, 11, 3, generator=gen, dtype=torch.float64)
    depth = torch.rand(9, 11, generator=gen, dtype=torch.float64) * 8 - 1 if masked else None
    pr = pred.clone().requires_grad_(True)
    n, g = F.normalize(pr, p=2, dim=-1), F.normalize(gt, p=2, dim=-1)
    if masked:
        m = torch.logical_and(depth > 0, depth < 5.0)
        n, g = n[m], g[m]
    ref = (n - g).abs().mean() + 0.1 * (-torch.sum(n * g, axis=-1).mean())
    ref.backward()
    val, grad, _ = LR.normal64(pred, gt, depth)
    assert abs(float(val) - float(ref)) < 1e-14
    torch.testing.assert_close(grad, pr.grad, rtol=1e-10, atol=1e-15)


def test_normal_restatement_empty_mask_is_nan():
    val, grad, _ = LR.normal64(torch.ones(4, 3), torch.ones(4, 3), torch.zeros(4))
    assert torch.isnan(val) and (grad == 0).all()


def test_anisotropic_restatement_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(3)
    s = torch.rand(500, 3, generator=gen, dtype=torch.float64) * 2
    s[:7, 0] = 0.0
    sr = s.clone().requires_grad_(True)
    mx, mn = torch.max(sr, dim=-1).values, torch.min(sr, dim=-1).values
    ref = torch.mean(torch.clamp(mx / (mn + 1e-6), min=3) - 3)
    ref.backward()
    val, grad, _ = LR.anisotropic64(s, 3.0)
    assert abs(float(val) - float(ref)) < 1e-12 * abs(float(ref))
    torch.testing.assert_close(grad, sr.grad, rtol=1e-10, atol=1e-18)


def test_first_extremes_rule():
    s = torch.tensor([[1.0, 1.0, 0.5], [2.0, 2.0, 2.0], [0.5, 3.0, 3.0], [1.0, float("nan"), float("nan")], [0.2, 0.2, 0.9]])
    imax, imin = LR.first_extremes(s)
    assert imax.tolist() == [0, 0, 1, 1, 2]
    assert imin.tolist() == [2, 0, 0, 1, 0]


# -- argument errors ------------------------------------------------------------------------------------------------------------

def _img(*shape, **kw):
    return torch.rand(*shape, **kw)


def test_ssim_argument_errors():
    from autovfx_b200 import losses as L
    a, b = _img(3, 8, 8), _img(3, 8, 8)
    with pytest.raises(ValueError, match="window_size"):
        L.ssim(a, b, window_size=7)
    with pytest.raises(ValueError, match="size_average"):
        L.ssim(a, b, size_average=False)
    with pytest.raises(ValueError, match="img2"):
        L.ssim(a, _img(3, 8, 9))
    with pytest.raises(ValueError, match="img1"):
        L.ssim(a.double(), b)
    with pytest.raises(ValueError, match="img2"):
        L.ssim(a, b.half())
    with pytest.raises(ValueError, match="img2 requires grad"):
        L.ssim(a, b.requires_grad_(True))
    with pytest.raises(ValueError, match="empty"):
        L.ssim(_img(3, 0, 8), _img(3, 0, 8))
    with pytest.raises(ValueError, match="img1"):
        L.ssim(_img(8, 8), _img(8, 8))


def test_photometric_argument_errors():
    from autovfx_b200 import losses as L
    a = _img(4, 6, 6)
    with pytest.raises(ValueError, match="gt"):
        L.photometric_loss(a, _img(3, 6, 6), 0.2)
    with pytest.raises(ValueError, match="gt requires grad"):
        L.photometric_loss(a, _img(4, 6, 6).requires_grad_(True), 0.2)
    with pytest.raises(ValueError, match="image"):
        L.photometric_loss(a.to(torch.float16), _img(4, 6, 6), 0.2)


def test_normal_loss_argument_errors():
    from autovfx_b200 import losses as L
    a, b = _img(5, 4, 3), _img(5, 4, 3)
    with pytest.raises(ValueError, match="last dimension of 3"):
        L.normal_loss(_img(5, 4, 2), _img(5, 4, 2))
    with pytest.raises(ValueError, match="gt"):
        L.normal_loss(a, _img(5, 5, 3))
    with pytest.raises(ValueError, match="gt requires grad"):
        L.normal_loss(a, b.requires_grad_(True))
    with pytest.raises(ValueError, match="depth"):
        L.normal_loss(a, _img(5, 4, 3), depth=_img(5, 5))
    with pytest.raises(ValueError, match="depth"):
        L.normal_loss(a, _img(5, 4, 3), depth=_img(5, 4).double())
    with pytest.raises(ValueError, match="empty"):
        L.normal_loss(_img(0, 3), _img(0, 3))


def test_anisotropic_loss_argument_errors():
    from autovfx_b200 import losses as L
    with pytest.raises(ValueError, match="last dimension of 3"):
        L.anisotropic_loss(_img(10, 2))
    with pytest.raises(ValueError, match="float32"):
        L.anisotropic_loss(_img(10, 3).double())
    with pytest.raises(ValueError, match="empty"):
        L.anisotropic_loss(_img(0, 3))


@pytest.mark.skipif(not torch.cuda.is_available(), reason="mixed devices need a CUDA device")
def test_mixed_devices_raise_value_error():
    from autovfx_b200 import losses as L
    with pytest.raises(ValueError, match="img2"):
        L.ssim(_img(3, 8, 8, device="cuda"), _img(3, 8, 8))


def test_cpu_tensors_raise_runtime_error():
    from autovfx_b200 import losses as L
    with pytest.raises(RuntimeError, match="CUDA"):
        L.ssim(_img(3, 8, 8), _img(3, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        L.photometric_loss(_img(4, 8, 8), _img(4, 8, 8), 0.2)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.normal_loss(_img(8, 8, 3), _img(8, 8, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        L.anisotropic_loss(_img(8, 3))


def test_exports_and_workspace_sizes():
    from autovfx_b200 import _lib
    for n in ("gsr_photometric_loss_bytes", "gsr_photometric_loss", "gsr_photometric_loss_backward", "gsr_normal_loss",
              "gsr_normal_loss_backward", "gsr_anisotropic_loss", "gsr_anisotropic_loss_backward"):
        assert n in _lib.EXPORTS and hasattr(_lib.lib, n)
    f = _lib.lib.gsr_photometric_loss_bytes
    n = 4 * 1080 * 1920
    assert f(1, 4, 1080, 1920, 1) - f(1, 4, 1080, 1920, 0) >= 3 * 4 * n
    assert f(1, 4, 1080, 1920, 0) < 1 << 20
    assert f(0, 4, 8, 8, 0) == 0 and f(1, 65536, 8, 8, 0) == 0
    hdr = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    assert "#define GSR_LOSS_REDUCE_BYTES (256 + 16 * 1024)" in hdr and _lib.GSR_LOSS_REDUCE_BYTES == 256 + 16 * 1024


def test_null_arguments_are_refused():
    from autovfx_b200 import _lib
    s4 = (C.c_int64 * 4)(0, 0, 0, 0)
    w = (C.c_float * 11)()
    rc = _lib.lib.gsr_photometric_loss(1, 1, 4, 4, None, s4, None, s4, w, 0, None, None, None, 0, None)
    assert rc == -1 and b"gsr_photometric_loss" in _lib.lib.gsr_last_error()
    assert _lib.lib.gsr_anisotropic_loss(0, None, 3.0, None, None, 0, None) == -1
    s2 = (C.c_int64 * 2)(3, 1)
    assert _lib.lib.gsr_normal_loss(4, 8, s2, 8, s2, None, 0, 5.0, 8, None, 0, None) == -2  # workspace missing
