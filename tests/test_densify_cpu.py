"""The one-pass densification plan (gsr_densify_plan's decisions and its four output streams, restated in torch by
tests/densify_ref.plan_map) against a literal clone -> split -> prune replay (densify_ref.sequential), on the CPU: the same final
row -> source map in every case the GPU tests run.  Also: the library exports the densification entry points."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402
import torch  # noqa: E402

from tests import densify_ref as DR  # noqa: E402

# name -> (max_grad, min_opacity, max_screen_size, scaling override, denom override)
CASES = {
    "default": (2e-4, 0.005, 20, None, None),
    "nothing": (1e9, 0.0, None, None, None),
    "clone_only": (2e-4, 0.005, 20, "small", None),
    "split_only": (2e-4, 0.005, 20, "medium", None),
    "all_pruned": (2e-4, 2.0, 20, None, None),
    "max_grad_zero": (0.0, 0.005, 20, None, None),
    "max_grad_negative": (-1.0, 0.005, 20, None, None),
    "screen_none": (2e-4, 0.005, None, None, None),
    "screen_zero": (2e-4, 0.005, 0, None, None),
    "screen_negative": (2e-4, 0.005, -1, None, None),
    "denom_zero": (2e-4, 0.005, 20, None, "zero"),
}


def make_case(name, P, M, seed, device="cpu"):
    """Seeded raw parameters of a GaussianModel ({group: tensor}) and densification statistics for case `name`."""
    max_grad, min_opacity, mss, scl, den = CASES[name]
    g = torch.Generator().manual_seed(seed)
    params = {"xyz": torch.randn(P, 3, generator=g) * 2, "f_dc": torch.randn(P, 1, 3, generator=g),
              "f_rest": torch.randn(P, M - 1, 3, generator=g), "opacity": torch.randn(P, 1, generator=g) * 3,
              "scaling": torch.rand(P, 3, generator=g) * 4.5 - 7.0, "rotation": torch.randn(P, 4, generator=g)}
    if scl == "small":
        params["scaling"] = torch.rand(P, 3, generator=g) * 2 - 8.0       # max(exp) < 0.01: never split
    elif scl == "medium":
        params["scaling"] = torch.rand(P, 3, generator=g) * 1.5 - 4.3     # 0.013 .. 0.06: never cloned, not pruned as big
    denom = torch.randint(0, 6, (P, 1), generator=g).float()
    accum = torch.rand(P, 1, generator=g) * 5e-4 * denom
    if den == "zero":
        denom = torch.zeros(P, 1)
        accum[::3] = torch.rand(accum[::3].shape, generator=g) * 1e-3      # accum / 0 = inf on a third, NaN -> 0 elsewhere
    out = {k: v.contiguous().to(device) for k, v in params.items()}
    return out, accum.to(device), denom.to(device), max_grad, min_opacity, mss


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("with_state", [False, True], ids=["no_state", "adam_state"])
def test_one_pass_plan_matches_sequential_replay(name, with_state):
    P, M, extent, pd = 600, 4, 1.0, 0.01
    params, accum, denom, max_grad, min_opacity, mss = make_case(name, P, M, seed=len(name))
    moments = {}
    if with_state:  # moments on some groups only: the others have no optimizer state yet
        g = torch.Generator().manual_seed(5)
        moments = {k: (torch.randn(v.shape, generator=g), torch.rand(v.shape, generator=g)) for k, v in params.items()
                   if k in ("xyz", "f_rest", "scaling")}
    torch.manual_seed(0)
    new, new_m, tags = DR.sequential(params, moments, accum, denom, max_grad, min_opacity, extent, mss, pd, DR.build_rotation)
    want, S = DR.plan_map(accum, denom, params["scaling"], params["opacity"], max_grad, min_opacity, extent, mss, pd)
    assert torch.equal(tags, want), name
    assert all(v.shape[0] == want.shape[0] for v in new.values())
    kind, src = tags // P, tags % P
    for k, v in new.items():
        base = params[k][src]
        same = kind <= 1 if k in ("xyz", "scaling") else torch.ones_like(kind, dtype=torch.bool)
        assert torch.equal(v[same], base[same]), k
        if k in new_m:  # kept originals carry their moments, every new row starts at zero
            for m_new, m_old in zip(new_m[k], moments[k]):
                assert torch.equal(m_new[kind == 0], m_old[src[kind == 0]])
                assert not m_new[kind > 0].any()
    # the case exercises what its name says
    if name == "nothing":
        assert torch.equal(tags, torch.arange(P))
    if name == "clone_only":
        assert S == 0 and (kind == 1).any()
    if name == "split_only":
        assert S > 0 and not (kind == 1).any()
    if name in ("all_pruned", "screen_negative"):
        assert tags.numel() == 0
    if name == "denom_zero":
        assert S > 0


def test_library_exports_the_densification_entry_points():
    from autovfx_b200 import _lib, densify
    for n in ("gsr_densify_stats", "gsr_densify_plan_bytes", "gsr_densify_plan", "gsr_densify_apply"):
        assert n in _lib.EXPORTS and hasattr(_lib.lib, n)
    assert set(densify.__all__) == {"add_densification_stats", "update_densification_stats", "densify_and_prune",
                                    "sugar_densify_and_prune"}


def test_cpu_tensors_raise():
    import types
    from autovfx_b200 import densify
    vs = torch.zeros(4, 3, requires_grad=True)
    vs.grad = torch.zeros(4, 3)
    m = types.SimpleNamespace(xyz_gradient_accum=torch.zeros(4, 1), denom=torch.zeros(4, 1))
    with pytest.raises(RuntimeError):
        densify.add_densification_stats(m, vs, torch.ones(4, dtype=torch.bool))
    vs.grad = None
    with pytest.raises(ValueError, match="grad"):
        densify.add_densification_stats(m, vs, torch.ones(4, dtype=torch.bool))
