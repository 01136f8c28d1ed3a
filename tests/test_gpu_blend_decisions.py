"""The default blend's guarded decisions at their thresholds (gsr_blend.cu): the fast drain (ex2.approx alphas) must take every
skip and termination decision the exact drain takes, so n_contrib is identical and the backward replays the reference's
decisions.  Each case runs in both modes through the single pass with n_contrib (forward_raw(for_backward=True)), through
the drain that blends a second colour set (NX = 3; its n_contrib read from forward_raw(extra=...), the forward of the fused
autograd path), and through forward_multi (images and radii: it keeps no workspace).  Exact mode is bit-identical to the
compiled reference.  Cases (tests/helpers.py): 1080p termination stacks that put T (1 - alpha) of a deciding splat within
1e-4 relative of 1e-4 behind near-opaque unclamped fronts; far-edge skips (opacity >= 0.5, power <= -4, alpha within 34 ulp
of 1/255); config3 with half its opacities redrawn in [0.90, 0.99) from three cameras."""
import numpy as np
import pytest
import torch

from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _extra(P):
    return torch.rand(P, 3, generator=torch.Generator().manual_seed(149)).to(DEV)


def check_modes(a):
    """Asserts the default mode's decisions, radii and images against the exact mode's in the three paths, and the exact mode
    against the reference; returns (fast, exact) outputs of the single pass (images, n_contrib, stats)."""
    from autovfx_b200 import rasterizer as R
    out = {}
    for mode in (False, True):
        o = Hh.run_ours(a, for_backward=True, debug=False, exact=mode)
        out[mode] = {k: o[k].clone() for k in ("color", "depth", "alpha", "radii")} | {
            "n_contrib": o["views"]["n_contrib"].clone(), "stats": o["stats"]}
    fast, exact = out[False], out[True]
    assert torch.equal(fast["radii"], exact["radii"])
    nbad = int((fast["n_contrib"] != exact["n_contrib"]).sum())
    assert nbad == 0, "%d pixels where the default mode's n_contrib differs from the exact mode's" % nbad
    Hh.assert_images_close(fast, exact)
    P, W, H = a["means3D"].shape[0], a["W"], a["H"]
    extra, s = _extra(P), Hh.settings_from(a)
    multi = {}
    for mode in (False, True):
        e_out = torch.empty(3, H, W, device=DEV)
        c, d, al, radii, ws, _, _ = R.forward_raw(a["means3D"], a["shs"], a["colors_precomp"], a["opacities"], a["scales"], a["rotations"],
                                                  a["cov3D_precomp"], s, for_backward=True, sync=True, extra=extra, extra_out=e_out, exact=mode)
        multi[mode] = dict(color=c.clone(), depth=d.clone(), alpha=al.clone(), radii=radii.clone(), extra=e_out.clone(),
                           n_contrib=R.debug_views(ws, P, W, H)["n_contrib"].clone())
        f = R.forward_multi(a["means3D"], a["shs"], a["colors_precomp"], extra, a["opacities"], a["scales"], a["rotations"],
                            a["cov3D_precomp"], s, sync=True, exact=mode)
        multi[mode]["fm"] = dict(color=f[0].clone(), depth=f[1].clone(), alpha=f[2].clone(), extra=f[3].clone(), radii=f[4].clone())
    for mode in (False, True):
        m = multi[mode]
        assert torch.equal(m["n_contrib"], exact["n_contrib"]), "NX = 3 drain, exact=%s: n_contrib differs" % mode
        assert torch.equal(m["radii"], exact["radii"]) and torch.equal(m["fm"]["radii"], exact["radii"])
        Hh.assert_images_close(m, exact)
        Hh.assert_images_close(m["fm"], exact)
        assert Hh.maxabs(m["extra"], multi[True]["extra"]) <= Hh.FAST_TOL["color"]
        assert Hh.maxabs(m["fm"]["extra"], multi[True]["extra"]) <= Hh.FAST_TOL["color"]
    for k in ("color", "depth", "alpha", "radii"):  # the single pass and the fused forward blend the same decisions bit for bit
        assert torch.equal(multi[True][k], exact[k]) and torch.equal(multi[True]["fm"][k], exact[k]), k
    if Hh.have_ref():
        ref = Hh.run_ref(a)
        for k in ("color", "depth", "alpha", "radii"):
            assert Hh.ref_same(exact[k], lambda: ref[k]), k
    return fast, exact


@pytest.fixture(scope="module")
def stacks():
    return Hh.termination_stacks_case(device=DEV)


def test_termination_stacks(stacks):
    a, facts = stacks
    S = len(facts["r"])
    assert S >= 100_000
    fast, exact = check_modes(a)
    x, y = facts["pix"][:, 0], facts["pix"][:, 1]
    red_e = exact["color"][0].cpu().numpy()[y, x].astype(np.float64)
    red_f = fast["color"][0].cpu().numpy()[y, x].astype(np.float64)
    # the regime: every stack's exact test value T (1 - alpha_C) within STACK_WINDOW of the fp32 threshold, C blended where it is
    # above (red = T alpha_C > 0) and not where it is below.  The builder's exp is correctly rounded, CUDA's expf is within 2 ulp:
    # that moves T (1 - alpha_C) by up to alpha_C / (1 - alpha_C) <= 24 times 2.4e-7, so stacks within 1e-5 may go either way
    near = np.abs(facts["r"]) <= Hh.STACK_WINDOW * (1 + 1e-3)
    blended = red_e > 0
    off = blended != (facts["r"] >= 0)
    redos = fast["stats"]["exact_redos"]
    # T in front of C, fast against exact, where C is blended in both modes and the warp was not redone (a redone warp's images
    # are the exact ones): red carries T alpha_C, whose fast alpha_C differs from the exact one by ex2.approx's error alone
    both = blended & (red_f > 0) & (red_f != red_e)
    gap = np.abs(red_f[both] / red_e[both] - 1.0)
    print("termination stacks: %d of %d within +-%g of the threshold, %d terminate at C, exact_redos %d, largest fast-vs-exact "
          "relative gap of T alpha_C over %d stacks %.3g" % (int(near.sum()), S, Hh.STACK_WINDOW, S - int(blended.sum()), redos,
                                                              int(both.sum()), gap.max() if both.any() else 0.0))
    assert int(near.sum()) >= 100_000 and 0.4 * S < int(blended.sum()) < 0.6 * S
    assert (np.abs(facts["r"][off]) < 1e-5).all(), np.abs(facts["r"][off]).max()
    assert redos > 0 and int(both.sum()) > 100


def test_far_edge_skips():
    a, tpix = Hh.far_edge_skip_case(device=DEV)
    fast, exact = check_modes(a)
    hit = exact["n_contrib"].cpu().numpy()[tpix[:, 1], tpix[:, 0]] > 0
    redos = fast["stats"]["exact_redos"]
    print("far-edge skips: %d splats, %d blended at their target pixel, exact_redos %d" % (len(tpix), int(hit.sum()), redos))
    assert 0.2 * len(tpix) < int(hit.sum()) < 0.8 * len(tpix)
    assert redos > 0


@pytest.mark.parametrize("cam_index", [7, 150, 271])
def test_trained_like_frame(cam_index):
    a = Hh.trained_like_case(cam_index, DEV)
    fast, _ = check_modes(a)
    print("trained-like frame, camera %d: exact_redos %d" % (cam_index, fast["stats"]["exact_redos"]))
    assert fast["stats"]["exact_redos"] > 0
