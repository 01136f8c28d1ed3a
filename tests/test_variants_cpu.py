"""CPU pinning of the oracle on the SH storage layouts of tests/test_gpu_variants.py (no GPU).

The GPU's per-Gaussian gradients are judged against the oracle's own error with respect to fp64 autograd (tests/torch_ref.py)
on the same case, so the oracle itself is pinned here: its forward against the fp64 restatement and its backward per
Gaussian, with each image gradient (colour, depth, alpha) isolated and all three together.
"""
import numpy as np
import pytest
import torch

from tests import helpers as Hh
from tests import torch_ref

FAMILIES = list(Hh.GRAD_FAMILIES)
TERMS = ("color", "depth", "alpha", "all")

# Oracle against fp64 autograd, per-Gaussian relative error (rows with ||g64|| > 1e-6 of the largest), measured on these
# cases over every tensor, family and term: median <= 1.4e-6, 99th percentile <= 1.6e-4, worst row 3.6e-3 (dL/dopacity, a
# sum of terms of both signs).  The bounds leave a factor of 5 to 7.
ORACLE_MEDIAN_TOL = 1e-5
ORACLE_Q99_TOL = 1e-3
ORACLE_MAX_TOL = 2e-2


@pytest.fixture(scope="module", params=FAMILIES)
def family(request):
    a = Hh.grad_args(request.param)
    fw = Hh.run_oracle(a)
    return request.param, a, fw, Hh.fp64_grads(a, fw, TERMS)


def test_oracle_forward_matches_fp64_on_every_layout(family):
    _, a, fw, _ = family
    color, depth, alpha, _, _ = torch_ref.render(a, fw)
    assert Hh.maxabs(color.detach(), fw["color"]) < 2e-5
    assert Hh.maxabs(depth.detach(), fw["depth"]) < 2e-5
    assert Hh.maxabs(alpha.detach(), fw["alpha"]) < 2e-5
    assert (fw["radii"] == 0).any() and (fw["radii"] > 0).any()
    if a["shs"] is not None:
        assert fw["clamped"].any() and not fw["clamped"].all()  # the clamp masks are exercised


@pytest.mark.parametrize("term", TERMS)
def test_oracle_backward_per_gaussian_matches_fp64(family, term):
    name, a, fw, g64 = family
    og = Hh.comparable_grads(Hh.oracle_backward(a, fw, *Hh.isolated_image_grads(a, term)), a)
    checked = 0
    for k, want in g64[term].items():
        if float(want.abs().max()) == 0.0:
            assert float(og[k].abs().max()) == 0.0, k  # e.g. dL/dsh under a depth-only loss
            continue
        e = Hh.row_errors(og[k], want)
        stats = (np.median(e), np.quantile(e, 0.99), e.max())
        assert stats[0] <= ORACLE_MEDIAN_TOL and stats[1] <= ORACLE_Q99_TOL and stats[2] <= ORACLE_MAX_TOL, (name, term, k, stats)
        checked += 1
    assert checked >= 4


def test_oracle_dL_dsh_is_zero_beyond_the_active_degree_and_off_screen(family):
    name, a, fw, _ = family
    if a["shs"] is None:
        pytest.skip("colours precomputed")
    og = Hh.oracle_backward(a, fw, *Hh.image_grads(a))
    n = (min(a["sh_degree"], 3) + 1) ** 2
    assert np.all(og["dL_dsh"][:, n:] == 0)
    assert np.all(og["dL_dsh"][fw["radii"] == 0] == 0)
    assert np.any(og["dL_dsh"][:, :n] != 0)
