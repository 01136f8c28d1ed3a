"""Torch restatements of densify_and_prune for the densification tests, written for them from the reference's documented steps
(GaussianModel.densify_and_prune, gaussian_model.py:359-413; SuGaRDensifier.densify_and_prune, sugar_densifier.py:186-244):

  * ``sequential`` replays the steps literally — clone (cat), split (normal draw, cat, prune), final prune — on a dict of raw
    parameters and Adam moments, with the same torch ops, and carries a source tag per row through every cat and mask;
  * ``plan_map`` restates gsr_densify_plan's one-pass decisions per original row and builds the final row -> source map from the
    four streams (surviving originals, clones, first split copies, second split copies).

A row's tag is kind * P + source row, kind 0 = original, 1 = clone, 2 = first split copy, 3 = second split copy.
"""
from __future__ import annotations

import torch


def build_rotation(r):
    """3DGS build_rotation: the quaternion over its norm, element-wise formulas (each op rounded on its own)."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)), -1)
    return R.reshape(-1, 3, 3)


def sugar_rotation(q):
    """SuGaR: pytorch3d quaternion_to_matrix of F.normalize(q)."""
    from autovfx_b200.renderer import quaternion_to_matrix
    return quaternion_to_matrix(torch.nn.functional.normalize(q, dim=-1))


def sequential(params, moments, accum, denom, max_grad, min_opacity, extent, max_screen_size, percent_dense, rotation,
               names=("xyz", "opacity", "scaling", "rotation")):
    """params: {group: raw tensor [P,...]}, moments: {group: (exp_avg, exp_avg_sq)} for the groups with state.  ``names`` gives the
    groups holding xyz, the raw opacity, the raw scaling and the raw rotation.  Returns (params, moments, tags)."""
    nx, no, ns, nr = names
    P = params[nx].shape[0]
    dev = params[nx].device
    params, moments = dict(params), dict(moments)
    tags = torch.arange(P, device=dev)
    grads = accum / denom
    grads[grads.isnan()] = 0.0

    def cat(ext, ext_tags):
        nonlocal tags
        for k in params:
            if k in moments:
                moments[k] = tuple(torch.cat((m, torch.zeros_like(ext[k])), dim=0) for m in moments[k])
            params[k] = torch.cat((params[k], ext[k]), dim=0)
        tags = torch.cat((tags, ext_tags))

    def keep(mask):
        nonlocal tags
        for k in params:
            if k in moments:
                moments[k] = tuple(m[mask] for m in moments[k])
            params[k] = params[k][mask]
        tags = tags[mask]

    # clone
    sel = torch.where(torch.norm(grads, dim=-1) >= max_grad, True, False)
    sel = torch.logical_and(sel, torch.max(torch.exp(params[ns]), dim=1).values <= percent_dense * extent)
    cat({k: v[sel] for k, v in params.items()}, tags[sel] + P)
    # split
    n_init = params[nx].shape[0]
    padded = torch.zeros((n_init), device=dev)
    padded[:grads.shape[0]] = grads.squeeze()
    sel = torch.where(padded >= max_grad, True, False)
    sel = torch.logical_and(sel, torch.max(torch.exp(params[ns]), dim=1).values > percent_dense * extent)
    stds = torch.exp(params[ns])[sel].repeat(2, 1)
    samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds)
    rots = rotation(params[nr][sel]).repeat(2, 1, 1)
    ext = {k: v[sel].repeat(2, *([1] * (v.dim() - 1))) for k, v in params.items()}
    ext[nx] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + params[nx][sel].repeat(2, 1)
    ext[ns] = torch.log(torch.exp(params[ns])[sel].repeat(2, 1) / (0.8 * 2))
    S = int(sel.sum())
    cat(ext, torch.cat((tags[sel] % P + 2 * P, tags[sel] % P + 3 * P)))
    keep(~torch.cat((sel, torch.zeros(2 * S, device=dev, dtype=bool))))
    # final prune: max_radii2D is all zeros after densification_postfix
    prune = (torch.sigmoid(params[no]) < min_opacity).squeeze()
    if max_screen_size:
        big_vs = torch.zeros(params[nx].shape[0], device=dev) > max_screen_size
        big_ws = torch.exp(params[ns]).max(dim=1).values > 0.1 * extent
        prune = torch.logical_or(torch.logical_or(prune, big_vs), big_ws)
    keep(~prune)
    return params, moments, tags


def plan_map(accum, denom, scaling, opacity, max_grad, min_opacity, extent, max_screen_size, percent_dense):
    """gsr_densify_plan's decisions per original row, restated in torch: returns (tags of the final rows, S)."""
    P = scaling.shape[0]
    dev = scaling.device
    g = (accum / denom).reshape(P)
    g = torch.where(g.isnan(), torch.zeros_like(g), g)
    mx = torch.exp(scaling).max(dim=1).values
    f32 = lambda x: torch.tensor(x, dtype=torch.float64).float().item()  # noqa: E731
    clone = (torch.norm(g[:, None], dim=-1) >= f32(max_grad)) & (mx <= f32(percent_dense * extent))
    split = (g >= f32(max_grad)) & (mx > f32(percent_dense * extent))
    low = torch.sigmoid(opacity.reshape(P)) < f32(min_opacity)
    child = torch.log(torch.exp(scaling) * (1.0 / torch.tensor(1.6, dtype=torch.float32)))
    mxc = torch.exp(child).max(dim=1).values
    if max_screen_size:
        vs = torch.tensor(0.0) > f32(max_screen_size)
        prune = low | vs | (mx > f32(0.1 * extent))
        prune_child = low | vs | (mxc > f32(0.1 * extent))
    else:
        prune, prune_child = low, low
    rows = torch.arange(P, device=dev)
    streams = [rows[~split & ~prune], rows[clone & ~prune] + P, rows[split & ~prune_child] + 2 * P, rows[split & ~prune_child] + 3 * P]
    return torch.cat(streams), int(split.sum())
