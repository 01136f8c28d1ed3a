"""Per-Gaussian gradients of the blend backward where its machinery is under load (run with -m gpu on an H100).

k_blend_backward walks each 8x4-pixel footprint's survivors back to front through a 128-entry ring refilled from 32-row blocks
of ballot words, prefetches the next batch ahead of the refill, masks the top row at the footprint's last contributor and redoes
a batch with expf when an ex2.approx evaluation lands near the 1/255 skip threshold.  The cases (tests/helpers.DENSE_CASES) reach
each of these, which is asserted first from the oracle's forward.  Then, for every loss term and gradient tensor:

  * the Gaussians with a non-zero row are exactly the oracle's (a lost, invented or mis-decided survivor changes the set);
  * per row, the GPU's error against fp64 autograd (tests/torch_ref.py, on the oracle's fp32 decisions) is held to the oracle's
    own error on the same row: the quantiles as in test_gpu_variants.py, and row by row with a handful of rows allowed over.
    dense_tile, whose fp64 reference costs minutes, is held to the oracle instead (the same decisions, so rows differ only by
    summation order and the GPU's approximate exp and reciprocal); the oracle is pinned to fp64 on the other cases in
    test_dense_grads_cpu.py.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from tests import helpers as Hh  # noqa: E402
from tests.test_gpu_variants import _ours_backward  # noqa: E402

pytestmark = pytest.mark.gpu

TERMS = ("color", "depth", "alpha", "all")

# Paired per-row bound: row i is over when e_gpu[i] > ROW_FACTOR * e_oracle[i] + ROW_FLOOR_Q99 * q99(e_oracle) + ROW_FLOOR, with
# e = ||g - g64|| / ||g64|| (rows with ||g64|| > 1e-6 of the largest).  At most ROW_ALLOWANCE rows of a tensor may be over, and
# none by more than ROW_CAP.  Under the alpha and depth terms dL/dalpha of a splat is (D - R) T with D and R nearly equal, so rows
# of dL/dopacity and dL/dmeans2D that sum hundreds of such differences cancel, and two summation orders disagree on a few of them
# by far more than the oracle's error on that row.  Measured on an H100 80GB HBM3 (700 W limit) over every case, term and tensor:
# at most 16 rows over (sort_regimes, alpha term, dL/dopacity; the worst of them 0.148 against the oracle's 0.047), then 14
# (faint_slab, alpha term, dL/dopacity, worst 0.119) and 7 (sort_regimes, depth term, dL/dopacity).  The same run puts the GPU's 50th and 99th percentiles at most 1.56x and 2.22x the oracle's, and every
# non-zero row set equal to the oracle's.  The allowance and the cap leave 1.5x and 2x.
ROW_FACTOR = 3.0
ROW_FLOOR_Q99 = 3.0
ROW_FLOOR = 1e-5
ROW_ALLOWANCE = 24
ROW_CAP = 0.3
Q_FACTOR = 3.0
Q_FLOOR = 2e-6
# dense_tile, against the oracle: at most ORACLE_ROWS_OVER rows differ from it by more than ORACLE_ROW_TOL, none by more than
# ORACLE_ROW_CAP.  Measured: at most 78 rows of 23,155 over (alpha term, dL/dopacity), the worst 0.072.
ORACLE_ROW_TOL = 1e-2
ORACLE_ROWS_OVER = 120
ORACLE_ROW_CAP = 0.15


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from autovfx_b200 import rasterizer  # noqa: F401  (fails loudly if the CUDA library is missing)
    return torch.device("cuda:0")


@pytest.fixture(scope="module", params=list(Hh.DENSE_CASES))
def case(request, dev):
    name = request.param
    a = Hh.dense_case(name, dev)
    fw = Hh.run_oracle(a)
    o = Hh.run_ours(a, for_backward=True)
    rec = o["views"]["records"].cpu().numpy()[o["radii"].cpu().numpy() > 0]  # the redo band is counted on the GPU's own records
    Hh.assert_dense_coverage(name, a, fw, records=rec)
    g64 = None if name == "dense_tile" else Hh.fp64_grads(a, fw, TERMS, oracle_decisions=True)
    band = None
    if name == "skip_band":
        # the forward's own decision for each band splat: it alone can reach its pixel, so it was blended iff n_contrib > 0 there
        px = Hh.band_pixels(a)
        gpu_hit = o["views"]["n_contrib"].cpu().numpy()[px[:, 1], px[:, 0]] > 0
        orc_hit = fw["n_contrib"][px[:, 1], px[:, 0]] > 0
        band = (torch.from_numpy(gpu_hit), torch.from_numpy(orc_hit))
    return name, a, fw, g64, band


def compare(case, term):
    """{tensor: (e_gpu, e_oracle)} per-row errors against the reference, the list of tensors whose non-zero rows differ, and (band
    case) the band splats whose non-zero rows differ from the forward's decisions.  Band splats that the oracle's fp32 evaluation
    (no fused multiply-add, expf correctly rounded) decides otherwise than the GPU forward are left out of the comparisons with
    the oracle and fp64; their rows are judged against the forward's decisions."""
    name, a, fw, g64, band = case
    dc, dd, da = Hh.isolated_image_grads(a, term, device=a["means3D"].device)
    radii, ours = _ours_backward(a, dc, dd, da)
    assert torch.equal(radii.cpu(), torch.from_numpy(fw["radii"]))
    ours = Hh.comparable_grads({k: v.cpu() for k, v in ours.items()}, a)
    orc = Hh.comparable_grads(Hh.oracle_backward(a, fw, dc, dd, da), a)
    keep = torch.ones(fw["radii"].shape[0], dtype=torch.bool)
    band_bad = []
    if band is not None:
        gpu_hit, orc_hit = band
        keep[:len(gpu_hit)] = gpu_hit == orc_hit
        nz = torch.zeros(len(gpu_hit), dtype=torch.bool)
        for v in ours.values():
            nz |= v[:len(gpu_hit)].reshape(len(gpu_hit), -1).ne(0).any(dim=1)
        band_bad = torch.nonzero(nz != gpu_hit).reshape(-1).tolist()
    errs, support = {}, []
    for k, o in orc.items():
        if k not in ours:  # intermediate gradients of the oracle (dL/dconic, dL/dcov3D, ...)
            continue
        nz_gpu = ours[k].reshape(o.shape[0], -1).ne(0).any(dim=1)[keep]
        nz_orc = o.reshape(o.shape[0], -1).ne(0).any(dim=1)[keep]
        if not torch.equal(nz_gpu, nz_orc):
            support.append((k, int((nz_gpu & ~nz_orc).sum()), int((nz_orc & ~nz_gpu).sum())))
        if not bool(nz_orc.any()):
            continue
        if g64 is None:
            errs[k] = (Hh.row_errors(ours[k][keep], o[keep]), None)
        else:
            want = g64[term][k][keep]
            errs[k] = (Hh.row_errors(ours[k][keep], want), Hh.row_errors(o[keep], want))
    return errs, support, band_bad


def row_check(e_gpu, e_orc):
    """(rows over the paired bound, the worst of them); with no oracle error (dense_tile) the rows over ORACLE_ROW_TOL."""
    if e_orc is None:
        over = e_gpu > ORACLE_ROW_TOL
    else:
        over = e_gpu > ROW_FACTOR * e_orc + ROW_FLOOR_Q99 * float(np.quantile(e_orc, 0.99)) + ROW_FLOOR
    return int(over.sum()), float(e_gpu[over].max()) if over.any() else 0.0


@pytest.mark.parametrize("term", TERMS)
def test_dense_gradients_per_gaussian(case, term):
    name = case[0]
    errs, support, band_bad = compare(case, term)
    assert not band_bad, "%s %s: band splats whose rows disagree with the forward's skip decision: %s" % (name, term, band_bad)
    assert not support, "%s %s: non-zero rows differ from the oracle's (tensor, GPU only, oracle only): %s" % (name, term, support)
    assert len(errs) >= 4
    for k, (e_gpu, e_orc) in errs.items():
        n, worst = row_check(e_gpu, e_orc)
        if e_orc is None:
            assert n <= ORACLE_ROWS_OVER and worst <= ORACLE_ROW_CAP, "%s %s %s: %d rows differ from the oracle by more than %g (worst %.3g)" % (
                name, term, k, n, ORACLE_ROW_TOL, worst)
            continue
        for q in (0.5, 0.99):
            got, base = float(np.quantile(e_gpu, q)), float(np.quantile(e_orc, q))
            assert got <= Q_FACTOR * base + Q_FLOOR, "%s %s %s: q%g per-row error %.3g, oracle %.3g" % (name, term, k, 100 * q, got, base)
        assert n <= ROW_ALLOWANCE and worst <= ROW_CAP, "%s %s %s: %d rows over the paired bound (worst %.3g)" % (name, term, k, n, worst)


def test_band_decisions_are_near_the_threshold(case):
    """The band case's splats sit where ex2.approx and expf can disagree, and the forward blends some and skips others."""
    name, a, fw, _, band = case
    if band is None:
        pytest.skip("not the band case")
    gpu_hit, orc_hit = band
    assert 0.3 * len(gpu_hit) < int(gpu_hit.sum()) < 0.7 * len(gpu_hit)
    # the oracle's sequence (no fused multiply-add, expf correctly rounded) decides most of them the same way: 13 of 240 differ
    assert int((gpu_hit != orc_hit).sum()) <= 0.1 * len(gpu_hit)
