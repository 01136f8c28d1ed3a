"""The case builders of tests/test_gpu_blend_decisions.py, pinned on the CPU oracle: each termination stack's pixel is reached by
its own splats alone and its deciding splat is placed where the designed share of stacks puts it (a float32 replay of the exact
drain, and the oracle's own blend); the far-edge skips sit at 1/255 where power, not log2(opacity), dominates."""
import numpy as np
import pytest

from tests import helpers as Hh


@pytest.fixture(scope="module")
def stacks():
    a, facts = Hh.termination_stacks_case(256, 160)
    return a, facts, Hh.run_oracle(a)


def test_stack_pixels_are_reached_by_their_own_splats(stacks):
    a, facts, fw = stacks
    x, y = facts["pix"][:, 0], facts["pix"][:, 1]
    # the last contributor of every stack pixel is the stack's C or one of the splats in front of it
    W = a["W"]
    tile = (y // 16) * ((W + 15) // 16) + x // 16
    nc = fw["n_contrib"][y, x].astype(np.int64)
    assert (nc > 0).all()
    last = fw["point_list"][fw["ranges"][tile, 0].astype(np.int64) + nc - 1].astype(np.int64)
    first_of_stack = np.r_[0, facts["c_idx"][:-1] + 1 + facts["after"][:-1]]
    assert ((last >= first_of_stack) & (last <= facts["c_idx"])).all()
    # with one-hot colours on a zero background the channels sum to 1 - T at the pixel: only the stack's splats blended there
    col = fw["color"][:, y, x].astype(np.float64).sum(axis=0)
    assert np.abs(col - fw["alpha"].reshape(a["H"], W)[y, x]).max() < 1e-5


def test_stacks_sweep_the_termination_threshold(stacks):
    a, facts, fw = stacks
    S = len(facts["r"])
    # a float32 replay of the exact drain: every stack's test value within the window, about half on each side
    near, far = ~facts["far"], facts["far"]
    assert (np.abs(facts["r"][near]) <= Hh.STACK_WINDOW * (1 + 1e-3)).all() and near.sum() > 0.75 * S
    lo, hi = Hh.STACK_FAR
    assert ((np.abs(facts["r"][far]) >= lo * (1 - 1e-3)) & (np.abs(facts["r"][far]) <= hi * (1 + 1e-3))).all()
    assert 0.4 * S < int((facts["r"] >= 0).sum()) < 0.6 * S
    assert set(np.unique(facts["kind"])) == {1, 2, 3} and 0.4 * S < int(facts["after"].sum()) < 0.6 * S
    assert (facts["T_front"] >= 1.6e-4).all() and (facts["T_front"] <= 2.1e-3).all()
    # the oracle's blend takes the designed decision at C (red carries T alpha_C of C alone); expf's last bit may flip the few
    # stacks within ~1e-6 of the threshold
    x, y = facts["pix"][:, 0], facts["pix"][:, 1]
    red = fw["color"][0, y, x].astype(np.float64)
    off = (red > 0) != (facts["r"] >= 0)
    assert (np.abs(facts["r"][off]) < 2e-6).all() and int(off.sum()) <= max(2, S // 1000)
    o = a["opacities"].numpy().reshape(-1)[facts["c_idx"]].astype(np.float64)
    rec = np.concatenate([fw["means2D"], fw["conic_opacity"]], axis=1)[facts["c_idx"]]
    a_c = o * np.exp(Hh.forward_power(rec, facts["pix"].astype(np.float32)).astype(np.float64))
    got = red[red > 0] / a_c[red > 0]
    assert np.abs(got / facts["T_front"][red > 0] - 1.0).max() < 1e-5


def test_stack_fronts_drift_past_the_fast_termination_band():
    """The fronts' alpha / (1 - alpha) summed per stack (the factor by which ex2.approx's relative error moves the fast T) reaches
    the range where a 2e-7 error exceeds 1e-5."""
    a, facts = Hh.termination_stacks_case(256, 160)
    rec = Hh._records(a)[0]
    o = a["opacities"].numpy().reshape(-1).astype(np.float64)
    al = o * np.exp(Hh.forward_power(rec, np.rint(rec[:, :2])).astype(np.float64))
    S = len(facts["r"])
    starts = np.r_[0, facts["c_idx"][:-1] + 1 + facts["after"][:-1]]
    amp = np.array([sum(v / (1 - v) for v in al[starts[s]:facts["c_idx"][s]] if v < 0.99) for s in range(S)])
    assert (amp > 50).sum() > 0.2 * S


def test_far_edge_skip_case():
    a, tpix = Hh.far_edge_skip_case(256, 160)
    rec = Hh._records(a)[0]
    o = a["opacities"].numpy().reshape(-1)
    assert (o >= 0.5).all() and (o < 1.0).all()
    power = Hh.forward_power(rec, tpix.astype(np.float32))
    assert (power <= -4.0).all() and (power * np.log2(np.e) < -6.0).all()
    prod = (o * np.exp(power.astype(np.float64)).astype(np.float32)).astype(np.float32)
    k = (prod.astype(np.float64) - np.float64(np.float32(1.0 / 255.0))) / Hh.BAND_ULPS
    assert (np.abs(k) <= 34).all() and (k == 0).sum() > 0.2 * len(k) and (np.abs(k) == 1).sum() > 0.4 * len(k)
    assert (np.abs(k) > 1).sum() > 0.15 * len(k)
