"""CPU pinning of the oracle on the dense gradient cases of tests/test_gpu_dense_grads.py (no GPU).

The GPU's per-Gaussian gradients on those cases are judged against the oracle's own per-row error with respect to fp64 autograd,
so the oracle is pinned here on the same cases, and each case is shown to reach the regimes of the blend backward it is there
for (tests/helpers.DENSE_CASES) before any GPU time is spent.  dense_tile's fp64 reference costs minutes; sort_regimes, with
tiles of over 4,096 entries, stands in for it.
"""
import numpy as np
import pytest

from tests import helpers as Hh

TERMS = ("color", "depth", "alpha", "all")
PINNED = ("sort_regimes", "faint_slab", "skip_band")

# Oracle against fp64 autograd on the oracle's decisions, per-Gaussian relative error (rows with ||g64|| > 1e-6 of the largest).
# Sums over hundreds of survivors cancel more than on the small cases of test_variants_cpu.py: measured over every case, term and
# tensor, median <= 1.0e-4 (dL/dmeans3D of faint_slab, whose splats' screen-position and conic terms largely cancel) and 99th
# percentile <= 4.9e-3 (dL/dopacity of faint_slab).  Single rows of dL/dopacity, sums of terms of both signs that nearly cancel,
# reach 1.5 on faint_slab, so no bound is put on the worst row here; the GPU is held to the oracle row by row.
ORACLE_MEDIAN_TOL = 5e-4
ORACLE_Q99_TOL = 2e-2


@pytest.mark.parametrize("name", list(Hh.DENSE_CASES))
def test_dense_case_reaches_its_regimes(name):
    a = Hh.dense_case(name)
    Hh.assert_dense_coverage(name, a, Hh.run_oracle(a))


@pytest.fixture(scope="module", params=PINNED)
def pinned(request):
    a = Hh.dense_case(request.param)
    fw = Hh.run_oracle(a)
    return request.param, a, fw, Hh.fp64_grads(a, fw, TERMS, oracle_decisions=True)


@pytest.mark.parametrize("term", TERMS)
def test_oracle_dense_gradients_per_gaussian_match_fp64(pinned, term):
    name, a, fw, g64 = pinned
    og = Hh.comparable_grads(Hh.oracle_backward(a, fw, *Hh.isolated_image_grads(a, term)), a)
    checked = 0
    for k, want in g64[term].items():
        # on the same decisions, the same Gaussians have a non-zero row
        nz = want.reshape(want.shape[0], -1).ne(0).any(dim=1)
        assert bool((og[k].reshape(want.shape[0], -1).ne(0).any(dim=1) == nz).all()), (name, term, k)
        if not bool(nz.any()):
            continue
        e = Hh.row_errors(og[k], want)
        stats = (np.median(e), np.quantile(e, 0.99), e.max())
        assert stats[0] <= ORACLE_MEDIAN_TOL and stats[1] <= ORACLE_Q99_TOL, (name, term, k, stats)
        checked += 1
    assert checked >= 4


def test_skip_band_splats_contribute_at_one_pixel_or_nowhere():
    """Each band splat is blended at its own pixel or nowhere: its gradient row is non-zero exactly where n_contrib at that pixel
    (which no other splat reaches) is, and the oracle blends some of the splats and skips others."""
    a = Hh.skip_band_case()
    fw = Hh.run_oracle(a)
    og = Hh.oracle_backward(a, fw, *Hh.image_grads(a))
    px = Hh.band_pixels(a)
    blended = fw["n_contrib"][px[:, 1], px[:, 0]] > 0
    nz = np.zeros(Hh.BAND_SPLATS, bool)
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dsh", "dL_dmeans3D"):
        nz |= (og[k][:Hh.BAND_SPLATS].reshape(Hh.BAND_SPLATS, -1) != 0).any(axis=1)
    assert np.array_equal(nz, blended)
    assert 0.3 * Hh.BAND_SPLATS < blended.sum() < 0.7 * Hh.BAND_SPLATS
    assert len(set(map(tuple, px))) == Hh.BAND_SPLATS
