"""Shared helpers for the parity tests and tools: run the same seeded inputs through (a) the product CUDA path
(autovfx_b200, via the C ABI), (b) the compiled reference (oracle/_ref, GPU) and (c) the CPU oracle."""
from __future__ import annotations

import math
import os
import sys
from typing import Dict, Optional

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from autovfx_b200 import scene  # noqa: E402


def case_inputs(name: str) -> Dict:
    """Named deterministic cases.  Returns dict(g=gaussians (cpu tensors), cam=Camera, kw=extra settings)."""
    if name == "config1":  # BASELINE configs[0]: 10k Gaussians, 256x256
        g, cam = scene.config1_scene()
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "small_sh":  # tiny, non-multiple-of-16 image, coloured background
        g = scene.synthetic_gaussians(600, seed=3, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.6)
        cam = scene.lookat_camera((0.3, -3.0, 0.4), (0, 0, 0), 100, 75, 55.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.2, 0.5, 0.9), scale_modifier=1.0)
    if name == "small_deg1_m25":  # SuGaR-style storage: M=25 (stride 300 B), active degree 1, scale modifier
        g = scene.synthetic_gaussians(500, seed=5, extent=(1, 1, 1), log_scale_mean=math.log(0.06), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((-2.0, -2.0, 1.0), (0, 0, 0), 96, 64, 70.0)
        return dict(g=g, cam=cam, sh_degree=1, bg=(1.0, 1.0, 1.0), scale_modifier=0.8)
    if name == "deg3_m25":  # SuGaR storage (M=25, 300-byte rows: only 4-byte aligned) rendered at degree 3 and 2: windowed SH staging
        g = scene.synthetic_gaussians(3000, seed=23, extent=(1, 1, 1), log_scale_mean=math.log(0.04), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((1.5, -2.5, 0.8), (0, 0, 0), 144, 96, 65.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.3, 0.3, 0.3), scale_modifier=1.0)
    if name == "deg2_m25":
        g = scene.synthetic_gaussians(2000, seed=29, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.5, sh_degree=4)
        cam = scene.lookat_camera((-1.0, -2.8, 0.5), (0, 0, 0), 112, 80, 65.0)
        return dict(g=g, cam=cam, sh_degree=2, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "small_precomp":  # colors_precomp + cov3D_precomp mode
        g = scene.synthetic_gaussians(700, seed=7, extent=(1, 1, 1), log_scale_mean=math.log(0.05), log_scale_std=0.5)
        cam = scene.lookat_camera((0.0, -2.5, 1.5), (0, 0, 0), 80, 80, 60.0)
        return dict(g=g, cam=cam, sh_degree=0, bg=(0.0, 0.0, 0.0), scale_modifier=1.0, precomp=True)
    if name == "big_splats":  # few huge splats (warp-cooperative tile walk) + a camera inside the cloud (near culling)
        g = scene.synthetic_gaussians(300, seed=11, extent=(1.5, 1.5, 1.5), log_scale_mean=math.log(0.4), log_scale_std=0.7)
        cam = scene.lookat_camera((0.2, -0.6, 0.1), (0, 0.5, 0), 128, 112, 80.0)
        return dict(g=g, cam=cam, sh_degree=2, bg=(0.1, 0.1, 0.1), scale_modifier=1.0)
    if name == "dense_tile":  # > 4096 splats on single tiles: exercises the large-bucket sort path
        g = scene.synthetic_gaussians(30000, seed=13, extent=(0.05, 0.05, 1.0), log_scale_mean=math.log(0.004), log_scale_std=0.3,
                                      opacity_mean=-3.0, opacity_std=1.0)
        cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 64, 64, 40.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if name == "coplanar":  # thousands of exactly equal depths: sort ties resolve by Gaussian id; degenerate depth range
        g = scene.synthetic_gaussians(6000, seed=17, extent=(0.6, 0.0, 0.6), log_scale_mean=math.log(0.02), log_scale_std=0.3,
                                      opacity_mean=-2.0, opacity_std=1.0)
        cam = scene.lookat_camera((0.0, -2.0, 0.0), (0, 0, 0), 96, 96, 50.0)
        return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.2, 0.0), scale_modifier=1.0)
    raise KeyError(name)


def sh_layout(shs: torch.Tensor, M: int, D: int, offset: bool, tail_seed: int, device=None) -> torch.Tensor:
    """shs [P,>=16,3] restored in a [P,M,3] layout: the (min(D,3)+1)^2 coefficients degree D reads, then a seeded random tail
    the rasterizer must ignore.  offset: the rows start 4 bytes past a 16-byte boundary (a [1:] view of a flat buffer of
    P*M*3+1 floats), the alignment a sliced or concatenated parameter tensor can have."""
    P = shs.shape[0]
    n = (min(D, 3) + 1) ** 2
    out = torch.randn(P, M, 3, generator=torch.Generator().manual_seed(tail_seed)) * 0.3
    out[:, :n] = shs[:, :n]
    buf = torch.empty(P * M * 3 + 1, device=device)
    base = buf[1:] if offset else buf[:-1]
    base.copy_(out.reshape(-1).to(base.device))
    return base.view(P, M, 3)


def layout_case() -> Dict:
    """Scene of the SH layout matrix: 3000 Gaussians with 25 stored coefficients, a ragged 123x85 image, DC terms wide enough
    that about a fifth of the colour channels are clamped at 0."""
    g = scene.synthetic_gaussians(3000, seed=41, extent=(1, 1, 1), log_scale_mean=math.log(0.035), log_scale_std=0.5, sh_degree=4)
    g["shs"][:, 0] *= 4.0
    cam = scene.lookat_camera((0.8, -2.6, 0.9), (0, 0, 0), 123, 85, 62.0)
    return dict(g=g, cam=cam, sh_degree=3, bg=(0.2, 0.4, 0.1), scale_modifier=1.0)


def sort_regimes_case() -> Dict:
    """16,000 Gaussians in a thin column seen end-on (80x72 image, 25 tiles): tiles of <= 2048 instances (single-pass sort),
    one of 2048..4096 (one shared-memory sort) and four of > 4096 (chunked sort through global memory)."""
    g = scene.synthetic_gaussians(16000, seed=13, extent=(0.08, 0.08, 1.0), log_scale_mean=math.log(0.004), log_scale_std=0.3,
                                  opacity_mean=-3.0, opacity_std=1.0)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 80, 72, 40.0)
    return dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)


def faint_slab_case(device=None) -> Dict:
    """5,000 faint splats (opacity 0.02..0.05) in a slab in front of a wall of 1,400 larger, nearly opaque ones (0.85..0.95), on a
    ragged 100x74 image.  The wall has a gap on the right, so in the footprints along its edge some pixels terminate at the wall
    (T < 1e-4) while their neighbours blend to the end of the list; the slab puts over 1,024 entries in front of the wall on the
    centre tiles.  Stored as SuGaR SH rows (M = 25) 4 bytes off 16-byte alignment, rendered at degree 3 with scale_modifier 1.15.
    Returns resolved arguments."""
    gen = torch.Generator().manual_seed(85)
    slab = scene.synthetic_gaussians(5000, seed=83, extent=(0.45, 0.25, 0.35), log_scale_mean=math.log(0.022), log_scale_std=0.4, sh_degree=4)
    slab["opacities"] = 0.02 + 0.03 * torch.rand(5000, 1, generator=gen)
    wall = scene.synthetic_gaussians(2000, seed=89, extent=(1.3, 0.02, 1.0), log_scale_mean=math.log(0.06), log_scale_std=0.3, sh_degree=4)
    wall["means3D"][:, 1] += 0.7
    wall["opacities"] = 0.85 + 0.1 * torch.rand(2000, 1, generator=gen)
    keep = wall["means3D"][:, 0] < 0.25 + 0.2 * wall["means3D"][:, 2]  # the gap: a slanted edge, so it crosses footprints at all offsets
    g = {k: torch.cat([slab[k], wall[k][keep]]).contiguous() for k in slab}
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 100, 74, 50.0)
    a = resolve(dict(g=g, cam=cam, sh_degree=3, bg=(0.1, 0.3, 0.2), scale_modifier=1.15), device)
    a["shs"] = sh_layout(g["shs"], 25, 3, True, tail_seed=87, device=device)
    return a


BAND_ULPS = 2.0 ** -31  # one ulp of fp32 at 1/255
BAND_SPLATS = 240


def skip_band_case(device=None) -> Dict:
    """Small splats (their screen footprint is the 0.3-pixel low-pass filter) whose centres lie within 0.3 pixel of a pixel
    centre on both axes, at least 2 pixels apart, each with the opacity that puts opacity * exp(power) at that pixel on 1/255
    (fp32), or 1 ulp above or below it, for three in four of them, and 2..34 ulp (up to 4e-6 relative) above or below for the
    rest.  Every other pixel is at least 0.7 pixel from the centre and far below 1/255, so each splat contributes at its one
    pixel or nowhere, and no other splat reaches that pixel.  power is evaluated with the GPU forward's rounding sequence
    (forward_power) on the records the forward computes: the GPU's own (debug_views) when device is a CUDA device, else the
    oracle's, and exp(power) correctly rounded.  At 0 and 1 ulp the backward's first evaluation (ex2.approx, about 1.5 ulp) often
    reaches the other decision than expf; its redo with expf must restore the forward's.
    The first tile holds none of them but a stack of 1,030 faint splats (opacity 0.006) around one pixel, so that one footprint's
    last contributor is at list position 1,025..1,056: its ballot column ends on a 32-row block of exactly 32 rows.
    The band splats are the first BAND_SPLATS Gaussians.  Returns resolved arguments."""
    g = scene.synthetic_gaussians(4000, seed=97, extent=(1.0, 0.3, 0.75), log_scale_mean=math.log(0.002), log_scale_std=0.2, sh_degree=3)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), 72, 56, 50.0)
    case = dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0)
    if device is not None and torch.device(device).type == "cuda":
        o = run_ours(resolve(case, device), for_backward=True)
        rec, vis = o["views"]["records"].cpu().numpy()[:, :6], o["radii"].cpu().numpy() > 0
    else:
        pre = run_oracle(resolve(case), stop_after="preprocess")
        rec, vis = np.concatenate([pre["means2D"], pre["conic_opacity"]], axis=1), pre["radii"] > 0
    m2 = rec[:, :2]
    pix = np.rint(m2)
    cand = np.flatnonzero(vis & (np.abs(m2 - pix) < 0.3).all(axis=1) & (pix >= 1).all(axis=1) & (pix[:, 0] <= 70) &
                          (pix[:, 1] <= 54) & (pix > 19).any(axis=1))
    taken, sel = set(), []
    for i in cand:  # no two centres within one pixel of each other's pixel
        x, y = int(pix[i, 0]), int(pix[i, 1])
        if any((x + u, y + v) in taken for u in (-1, 0, 1) for v in (-1, 0, 1)):
            continue
        taken.add((x, y))
        sel.append(i)
        if len(sel) == BAND_SPLATS:
            break
    sel = np.asarray(sel)
    assert len(sel) == BAND_SPLATS, len(sel)
    g = {k: v[torch.from_numpy(sel)].contiguous() for k, v in g.items()}
    E = np.exp(forward_power(rec[sel], pix[sel].astype(np.float32)).astype(np.float64)).astype(np.float32)
    n = np.arange(BAND_SPLATS)
    k = np.where(n % 4 < 3, (n % 4) - 1, (2 + (n * 7) % 33) * np.where((n // 4) % 2 == 0, 1, -1)).astype(np.float64)
    target = np.float32(1.0 / 255.0).astype(np.float64) + k * BAND_ULPS
    o = (target / E.astype(np.float64)).astype(np.float32)
    for _ in range(4):  # nudge each opacity until the fp32 product is the target exactly
        got = (o.astype(np.float64) * E).astype(np.float32).astype(np.float64)
        o = np.where(got < target, np.nextafter(o, np.float32(1)), np.where(got > target, np.nextafter(o, np.float32(0)), o))
    g["opacities"] = torch.from_numpy(o.reshape(-1, 1))
    stack = scene.synthetic_gaussians(1030, seed=101, extent=(0.004, 0.2, 0.004), log_scale_mean=math.log(0.003), log_scale_std=0.2,
                                      sh_degree=3)
    stack["means3D"] += torch.tensor([-1.2, 0.0, 0.85])  # near pixel (5, 6)
    stack["opacities"] = torch.full((1030, 1), 0.006)
    g = {k: torch.cat([g[k], stack[k]]).contiguous() for k in g}
    return resolve(dict(case, g=g), device)


def _records(a: Dict, device=None):
    """[P, 6] fp32 {x, y, a, b, c, opacity} records and the visibility of a case's splats: the GPU forward's own (debug_views) when
    device is a CUDA device, else the oracle's preprocess."""
    if device is not None and torch.device(device).type == "cuda":
        o = run_ours(a, for_backward=True)
        return o["views"]["records"].cpu().numpy()[:, :6].copy(), o["radii"].cpu().numpy() > 0
    pre = run_oracle({k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in a.items()}, stop_after="preprocess")
    return np.concatenate([pre["means2D"], pre["conic_opacity"]], axis=1), pre["radii"] > 0


def _points_at_pixels(cam, pix: np.ndarray, z: np.ndarray) -> torch.Tensor:
    """World points that project to pixel coordinates pix [N, 2] at view-space depth z [N] (float64 inverse of the projection)."""
    ndc = (2.0 * pix + 1.0) / np.array([cam.image_width, cam.image_height]) - 1.0
    pv = np.stack([ndc[:, 0] * cam.tanfovx * z, ndc[:, 1] * cam.tanfovy * z, z, np.ones_like(z)], axis=1)
    pw = pv @ np.linalg.inv(cam.world_view_transform.double().numpy())
    return torch.from_numpy(pw[:, :3]).float().contiguous()


def _point_splats(cam, pix: np.ndarray, z: np.ndarray, colors: np.ndarray, device=None) -> Dict:
    """Resolved arguments of tiny isotropic splats (scale 1e-5: the 0.3-pixel low-pass sets the footprint) centred on pix at
    depth z, with colours precomputed; the opacities are placeholders until the records are known."""
    n = len(pix)
    g = dict(means3D=_points_at_pixels(cam, pix, z), scales=torch.full((n, 3), 1e-5), opacities=torch.full((n, 1), 0.5),
             rotations=torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(n, 1), shs=None)
    a = resolve(dict(g=g, cam=cam, sh_degree=0, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), device)
    a["colors_precomp"] = torch.from_numpy(np.ascontiguousarray(colors, dtype=np.float32)).to(a["means3D"].device)
    return a


def _alpha_window(rec: np.ndarray, o: np.ndarray, centre: np.ndarray, R: int = 4):
    """alpha = o * exp(power) in float64 (power with the GPU forward's rounding) at every pixel centre + (u, v), |u|, |v| <= R:
    ([N, (2R+1)^2] alphas, [(2R+1)^2, 2] offsets).  Evaluated in chunks."""
    off = np.stack(np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="xy"), -1).reshape(-1, 2)
    out = np.empty((len(rec), len(off)))
    for s in range(0, len(rec), 65536):
        r, c = rec[s:s + 65536, None, :], centre[s:s + 65536, None, :] + off[None]
        out[s:s + 65536] = o[s:s + 65536, None].astype(np.float64) * np.exp(forward_power(r, c.astype(np.float32)).astype(np.float64))
    return out, off


def exact_alpha(o: np.ndarray, power: np.ndarray) -> np.ndarray:
    """The exact drain's alpha in fp32: min(0.99, opacity * exp(power)), exp correctly rounded."""
    e = np.exp(power.astype(np.float64)).astype(np.float32)
    return np.minimum(np.float32(0.99), (o.astype(np.float32) * e).astype(np.float32))


def exact_step(T: np.ndarray, alpha: np.ndarray) -> np.ndarray:
    """The exact drain's termination test value T * (1 - alpha) in fp32."""
    return (T * (np.float32(1) - alpha).astype(np.float32)).astype(np.float32)


# Termination stacks: roles in depth order.  One-hot colours on a zero background: green carries the fronts and the clamped
# control, red the deciding splat C alone (so red = T in front of C times alpha_C), blue the splat after C.
ST_FRONT, ST_CTRL, ST_C, ST_AFTER = 0, 1, 2, 3
STACK_WINDOW = 1e-4  # C's exact T (1 - alpha) is swept over 1e-4 * (1 +- STACK_WINDOW) ...
STACK_FAR = (6e-4, 2e-3)  # ... or, for a fifth of the stacks, 1e-4 * (1 +- r) with r in this range


def termination_stacks_case(W: int = 1920, H: int = 1080, seed: int = 131, device=None):
    """Independent stacks of tiny splats on a 4-pixel grid, each centred within 0.04 pixel of its pixel centre, that put the
    termination decision T (1 - alpha) < 1e-4 of a deciding splat C at its threshold.  In front of C: one front splat with
    unclamped alpha in [0.90, 0.983] and a clamped control (alpha 0.99 in both drains), in either order; or two fronts with
    alpha in [0.90, 0.989]; or three in [0.90, 0.944].  C's opacity is chosen so that the exact drain's fp32 T (1 - alpha_C) at
    the stack's pixel is 1e-4 * (1 + r), r uniform in +-STACK_WINDOW (or +-STACK_FAR for one in five, outside the default blend's
    termination band); every other stack is followed by one more splat (alpha
    0.5..0.8).  The fronts' fast alphas drift from the exact ones by ~a / (1 - a) of ex2.approx's relative error each, so the
    two drains' T in front of C can differ by more than the default blend's 1e-5 termination band.  No (pixel, splat) pair
    comes within 2 % of alpha = 1/255, and at every stack's pixel the other stacks' splats stay below 1/510.
    Returns (resolved arguments, facts): facts holds each stack's pixel, kind (1..3 fronts), whether a splat follows C, the
    index of C, the exact fp32 T in front of C, the relative position r of its test value to the fp32 threshold and which
    stacks are the far ones."""
    rng = np.random.default_rng(seed)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), W, H, 60.0)
    gx, gy = np.meshgrid(2 + 4 * np.arange((W - 1) // 4), 2 + 4 * np.arange((H - 1) // 4), indexing="xy")
    spix = np.stack([gx.reshape(-1), gy.reshape(-1)], 1).astype(np.float64)
    S = len(spix)
    kind = rng.integers(1, 4, S)
    after = rng.random(S) < 0.5
    ctrl_first = rng.random(S) < 0.5
    # 1 - alpha of the fronts, log-uniform so that alphas near the top of their range are well represented
    lu = lambda lo, hi, n: np.exp(rng.uniform(np.log(lo), np.log(hi), n))  # noqa: E731
    om = np.zeros((S, 3))
    om[:, 0] = np.where(kind == 3, lu(0.056, 0.1, S), np.where(kind == 1, lu(0.017, 0.1, S), lu(0.011, 0.1, S)))
    lo2, hi2 = np.maximum(0.011, 1.7e-4 / om[:, 0]), np.minimum(0.1, 2e-3 / om[:, 0])
    om[:, 1] = np.where(kind == 3, lu(0.056, 0.1, S), np.exp(rng.uniform(np.log(lo2), np.log(hi2))))
    om[:, 2] = lu(0.056, 0.1, S)
    # one stack in five lies outside the default blend's termination band (STACK_FAR): there the fast T in front of C is not
    # replaced by a redo and can be compared with the exact one
    far = rng.random(S) < 0.2
    r = np.where(far, rng.uniform(*STACK_FAR, S) * rng.choice([-1.0, 1.0], S), rng.uniform(-STACK_WINDOW, STACK_WINDOW, S))
    roles, stack, target, depth_rank = [], [], [], []
    for s in range(S):
        k = int(kind[s])
        seq = [(ST_FRONT, 1 - om[s, 0])] + ([(ST_CTRL, 0.99)] if k == 1 else [(ST_FRONT, 1 - om[s, i]) for i in range(1, k)])
        if k == 1 and ctrl_first[s]:
            seq = seq[::-1]
        seq += [(ST_C, 0.0)] + ([(ST_AFTER, rng.uniform(0.5, 0.8))] if after[s] else [])
        roles += [q[0] for q in seq]
        target += [q[1] for q in seq]
        stack += [s] * len(seq)
        depth_rank += list(range(len(seq)))
    roles, stack, target, depth_rank = (np.asarray(v) for v in (roles, stack, target, depth_rank))
    pix = spix[stack]
    colors = np.zeros((len(roles), 3))
    colors[roles == ST_C, 0] = 1.0
    colors[(roles == ST_FRONT) | (roles == ST_CTRL), 1] = 1.0
    colors[roles == ST_AFTER, 2] = 1.0
    a = _point_splats(cam, pix + rng.uniform(-0.04, 0.04, pix.shape), 3.0 + 0.05 * depth_rank, colors, device)
    rec, vis = _records(a, device)
    assert vis.all() and (np.abs(rec[:, :2] - pix) <= 0.05).all()
    E = np.exp(forward_power(rec, pix.astype(np.float32)).astype(np.float64))
    o = (target / E).astype(np.float32)
    o[roles == ST_CTRL] = np.float32(0.99 * 1.001) / E[roles == ST_CTRL].astype(np.float32)
    # the exact drain's T in front of C, replayed in fp32, then C's opacity for T (1 - alpha_C) = 1e-4 (1 + r)
    power = forward_power(rec, pix.astype(np.float32))
    T = np.ones(S, np.float32)
    for d in range(int(depth_rank.max()) + 1):
        sel = (depth_rank == d) & ((roles == ST_FRONT) | (roles == ST_CTRL))
        s = stack[sel]
        al = exact_alpha(o[sel], power[sel])
        T[s] = exact_step(T[s], al)
    c_idx = np.flatnonzero(roles == ST_C)
    assert (stack[c_idx] == np.arange(S)).all()
    a_c = 1.0 - 1e-4 * (1.0 + r) / T.astype(np.float64)
    o[c_idx] = (a_c / E[c_idx]).astype(np.float32)
    test = exact_step(T, exact_alpha(o[c_idx], power[c_idx]))
    assert (o > 0.3).all() and (o < 1.0).all(), (o.min(), o.max())
    # no pair near the skip threshold; the other stacks' splats far below it at a stack's pixel
    aw, off = _alpha_window(rec, o, pix)
    assert (np.abs(255.0 * aw - 1.0) > 0.02).all()
    other = ((off % 4) == 0).all(axis=1) & (off != 0).any(axis=1)
    assert (aw[:, other] < 0.5 / 255.0).all()
    a["opacities"] = torch.from_numpy(o.reshape(-1, 1)).to(a["means3D"].device)
    facts = dict(pix=spix.astype(np.int64), kind=kind, after=after, c_idx=c_idx, T_front=T, far=far,
                 r=test.astype(np.float64) / np.float64(np.float32(1e-4)) - 1.0)
    return a, facts


def far_edge_skip_case(W: int = 1920, H: int = 1080, seed: int = 137, device=None):
    """Tiny splats on an 8-pixel grid with opacities in [0.5, 1), each placed so that at one pixel 1.6..1.9 pixel from its centre
    (power <= -4, power * log2e about -7.5) opacity * exp(power) is 1/255 in fp32, or 1 ulp above or below it, for three in four
    of them, and 2..34 ulp above or below for the rest (skip_band_case's pattern and nudge loop).  There log2(opacity) is small
    and power carries q's rounding error, the other end of the skip decision's error budget from skip_band_case.  Every other
    (pixel, splat) pair is at least 0.2 % from 1/255 (splats for which one is not are left out).  Returns (resolved arguments,
    the [N, 2] target pixel of each splat)."""
    rng = np.random.default_rng(seed)
    cam = scene.lookat_camera((0.0, -3.0, 0.0), (0, 0, 0), W, H, 60.0)
    gx, gy = np.meshgrid(4 + 8 * np.arange((W - 8) // 8), 4 + 8 * np.arange((H - 8) // 8), indexing="xy")
    tpix = np.stack([gx.reshape(-1), gy.reshape(-1)], 1).astype(np.float64)
    N = len(tpix)
    o0 = rng.uniform(0.55, 0.95, N)
    d = np.sqrt(np.log(255.0 * o0) / (0.5 / 0.3))  # distance at which o0 exp(-d^2 / 0.6) = 1/255 under the low-pass alone
    th = rng.uniform(0, 2 * np.pi, N)
    centre = tpix + np.stack([d * np.cos(th), d * np.sin(th)], 1)
    a = _point_splats(cam, centre, np.full(N, 3.0), rng.uniform(0.0, 1.0, (N, 3)), device)
    rec, vis = _records(a, device)
    assert vis.all()
    power = forward_power(rec, tpix.astype(np.float32))
    assert (power <= -4.0).all(), power.max()
    E = np.exp(power.astype(np.float64)).astype(np.float32)
    n = np.arange(N)
    k = np.where(n % 4 < 3, (n % 4) - 1, (2 + (n * 7) % 33) * np.where((n // 4) % 2 == 0, 1, -1)).astype(np.float64)
    target = np.float32(1.0 / 255.0).astype(np.float64) + k * BAND_ULPS
    o = (target / E.astype(np.float64)).astype(np.float32)
    for _ in range(4):  # nudge each opacity until the fp32 product is the target exactly
        got = (o.astype(np.float64) * E).astype(np.float32).astype(np.float64)
        o = np.where(got < target, np.nextafter(o, np.float32(1)), np.where(got > target, np.nextafter(o, np.float32(0)), o))
    assert ((o.astype(np.float64) * E).astype(np.float32).astype(np.float64) == target).all()
    assert (o >= 0.5).all() and (o < 1.0).all()
    aw, off = _alpha_window(rec, o, tpix)
    aw[:, (off == 0).all(axis=1)] = 0.0
    keep = (np.abs(255.0 * aw - 1.0) > 2e-3).all(axis=1)
    assert keep.mean() > 0.95, keep.mean()
    a["opacities"] = torch.from_numpy(o.reshape(-1, 1)).to(a["means3D"].device)
    kt = torch.from_numpy(keep).to(a["means3D"].device)
    for key in ("means3D", "scales", "rotations", "opacities", "colors_precomp"):
        a[key] = a[key][kt].contiguous()
    return a, tpix[keep].astype(np.int64)


def trained_like_case(cam_index: int, device=None) -> Dict:
    """config3's 3M Gaussians with every second opacity redrawn in [0.90, 0.99) (a trained scene's opaque surfaces: fronts whose
    fast alpha drifts from the exact one by up to ~a / (1 - a) of ex2.approx's error), at 1920x1080 from a trajectory camera."""
    g = scene.config3_scene()
    g["opacities"][::2] = 0.90 + 0.09 * torch.rand(g["opacities"][::2].shape, generator=torch.Generator().manual_seed(139))
    cam = scene.cameras_from_trajectory(scene.trajectory_dict(num_views=300))[cam_index]
    return resolve(dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), device)


def band_pixels(a: Dict) -> np.ndarray:
    """[BAND_SPLATS, 2] (x, y) pixel of each band splat of skip_band_case: the nearest to its projected centre."""
    from oracle import gsr_oracle  # noqa: F401
    pre = run_oracle({k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in a.items()}, stop_after="preprocess")
    return np.rint(pre["means2D"][:BAND_SPLATS]).astype(np.int64)


def oracle_power(m2d: np.ndarray, co: np.ndarray, pix: np.ndarray) -> np.ndarray:
    """power = -0.5 (a dx^2 + c dy^2) - b dx dy in fp32, the oracle's rounding sequence (no fused multiply-add)."""
    f = np.float32
    dx = (m2d[..., 0] - pix[..., 0]).astype(f)
    dy = (m2d[..., 1] - pix[..., 1]).astype(f)
    return (f(-0.5) * (co[..., 0] * dx * dx + co[..., 2] * dy * dy) - co[..., 1] * dx * dy).astype(f)


def forward_power(rec: np.ndarray, pix: np.ndarray) -> np.ndarray:
    """power in fp32 with the GPU forward's rounding sequence (gsr_blend.cu: products, then two fused multiply-adds), from
    records [.., {x, y, a, b, c}]; each fma is evaluated exactly in float64 and rounded once."""
    f, d = np.float32, np.float64
    dx = (rec[..., 0] - pix[..., 0]).astype(f)
    dy = (rec[..., 1] - pix[..., 1]).astype(f)
    t1, t3, t2 = (rec[..., 4] * dy).astype(f), (rec[..., 2] * dx).astype(f), ((-rec[..., 3]) * dx).astype(f)
    t4, t5 = (dy * t1).astype(f), (dy * t2).astype(f)
    t6 = (dx.astype(d) * t3 + t4).astype(f)
    return (t6.astype(d) * -0.5 + t5).astype(f)


def band_pairs(rec: np.ndarray, W: int, H: int) -> int:
    """(pixel, splat) pairs, at the pixel nearest each centre inside the image, where the backward's first evaluation of
    opacity * exp(power) lands within its redo band |255 alpha - 1| < 8e-6 (checked with a margin: 7e-6).  rec: [P, >= 6]
    fp32 records {x, y, a, b, c, opacity} of the rendered splats."""
    pix = np.rint(rec[:, :2]).astype(np.float32)
    inside = (pix[:, 0] >= 0) & (pix[:, 0] < W) & (pix[:, 1] >= 0) & (pix[:, 1] < H)
    oG = rec[:, 5].astype(np.float64) * np.exp(forward_power(rec, pix).astype(np.float64))
    return int((inside & (np.abs(oG * 255.0 - 1.0) < 7e-6)).sum())


def footprint_coverage(fw: Dict, W: int, H: int) -> Dict[str, np.ndarray]:
    """Per 8x4-pixel footprint of the blend backward (16x16 tiles, footprint f at x + 8 (f & 1), y + 4 (f >> 1)), from the oracle's
    forward: `last`, the list position (1-based) of the furthest last contributor of its pixels; `survivors`, the list entries
    before it that reach power <= 0 and alpha >= 1/255 at one of its pixels; `mixed`, whether its pixels inside the image have
    different last contributors; `partial`, whether it has pixels outside the image; `terminated` and `through`, whether one of
    its pixels stopped at T < 1e-4 (the first list entry it would blend after its last contributor takes T_final (1 - alpha) below
    1e-4) and whether one blended to the end of its list."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    m2, co, nc = fw["means2D"], fw["conic_opacity"], fw["n_contrib"].astype(np.int64)
    out = {k: [] for k in ("last", "survivors", "mixed", "partial", "terminated", "through")}
    T_final = (np.float32(1) - fw["alpha"].reshape(H, W)).astype(np.float32)
    fx, fy = np.arange(32) % 8, np.arange(32) // 8
    for tile in range(gx * gy):
        r0, r1 = (int(v) for v in fw["ranges"][tile])
        ty, tx = divmod(tile, gx)
        for f in range(8):
            px, py = tx * 16 + (f & 1) * 8 + fx, ty * 16 + (f >> 1) * 4 + fy
            inside = (px < W) & (py < H)
            lanes = nc[py[inside], px[inside]]
            last = int(lanes.max()) if lanes.size else 0
            g = fw["point_list"][r0:r1].astype(np.int64)
            pix = np.stack([px[inside], py[inside]], axis=-1).astype(np.float32)[None]
            power = oracle_power(m2[g][:, None], co[g][:, None], pix)
            alpha = np.minimum(np.float32(0.99), co[g][:, None, 3] * np.exp(power.astype(np.float64)).astype(np.float32))
            hit = (power <= 0) & (alpha >= np.float32(1.0 / 255.0))
            # per pixel, the first entry it would blend after its last contributor (index n_contrib), if any
            after = hit & (np.arange(len(g))[:, None] >= lanes[None])
            has = after.any(axis=0)
            first = np.argmax(after, axis=0) if len(g) else np.zeros(len(lanes), np.int64)
            a_next = alpha[first, np.arange(len(lanes))] if len(g) else np.ones(len(lanes), np.float32)
            stop = has & (T_final[py[inside], px[inside]] * (np.float32(1) - a_next) < np.float32(1e-4))
            out["terminated"].append(bool(stop.any()))
            out["through"].append(bool((~has).any()))
            out["last"].append(last)
            out["survivors"].append(int(hit[:last].any(axis=1).sum()) if last else 0)
            out["mixed"].append(bool(lanes.size and lanes.min() != lanes.max()))
            out["partial"].append(bool((~inside).any()) and r1 > r0)
    return {k: np.asarray(v) for k, v in out.items()}


# The dense gradient cases (tests/test_gpu_dense_grads.py, pinned on the CPU by tests/test_dense_grads_cpu.py) and the regimes of
# the blend backward each must reach (coverage_facts): the survivor ring (128 entries) wraps, and wraps twice; a footprint's last
# contributor lies beyond list position 1024 (more than one 32-row ballot block) or 4096, or at 1025..1056 (+ 1024 k), where the
# last block holds exactly 32 rows; a footprint beyond position 1024 with a pixel that terminates (T < 1e-4) next to one that
# blends to the end of its list; footprints with pixels outside the image; (skip_band) splats in the backward's redo band.
DENSE_CASES = {"skip_band": ("ring", "ring2", "blocks", "block_edge", "band"),
               "dense_tile": ("ring", "ring2", "blocks", "blocks4096"), "sort_regimes": ("ring", "ring2", "blocks", "blocks4096"),
               "coplanar": ("ring",), "config1": ("ring", "mixed"),
               "faint_slab": ("ring", "ring2", "blocks", "mixed", "partial", "terminate_deep")}
BAND_MIN_PAIRS = 200  # of BAND_SPLATS, each with one candidate pixel


def dense_case(name: str, device=None) -> Dict:
    if name == "faint_slab":
        return faint_slab_case(device)
    if name == "skip_band":
        return skip_band_case(device)
    return resolve(sort_regimes_case() if name == "sort_regimes" else case_inputs(name), device)


def coverage_facts(a: Dict, fw: Dict, records: Optional[np.ndarray] = None) -> Dict[str, bool]:
    """Which regimes of the blend backward the oracle's forward of a case reaches (see DENSE_CASES).  records: [P, >= 6] fp32
    {x, y, a, b, c, opacity} of the rendered splats for the redo-band count (default: the oracle's)."""
    c = footprint_coverage(fw, a["W"], a["H"])
    if records is None:
        records = np.concatenate([fw["means2D"], fw["conic_opacity"]], axis=1)[fw["radii"] > 0]
    return {"ring": bool((c["survivors"] > 128).any()), "ring2": bool((c["survivors"] > 256).any()),
            "blocks": bool((c["last"] > 1024).any()), "blocks4096": bool((c["last"] > 4096).any()),
            "block_edge": bool(((c["last"] > 1024) & (((c["last"] - 1) >> 5) % 32 == 0)).any()),
            "mixed": bool(c["mixed"].any()), "partial": bool((c["partial"] & (c["last"] > 0)).any()),
            "terminate_deep": bool((c["terminated"] & c["through"] & (c["last"] > 1024)).any()),
            "band": band_pairs(records, a["W"], a["H"]) >= BAND_MIN_PAIRS}


def assert_dense_coverage(name: str, a: Dict, fw: Dict, records: Optional[np.ndarray] = None):
    facts = coverage_facts(a, fw, records)
    missing = [k for k in DENSE_CASES[name] if not facts[k]]
    assert not missing, "%s does not reach %s" % (name, missing)


def layout_args(M: Optional[int], D: int, offset: bool, device=None) -> Dict:
    """The layout case rendered from shs [P,M,3] at degree D (M None: colours precomputed from the degree-3 SH, with scales and
    rotations)."""
    a = resolve(layout_case(), device)
    a["sh_degree"] = D
    if M is None:
        gen = torch.Generator().manual_seed(43)
        a["colors_precomp"] = (torch.rand(a["means3D"].shape[0], 3, generator=gen) * 1.2 - 0.1).to(a["means3D"].device)
        a["shs"] = None
    else:
        a["shs"] = sh_layout(a["shs"].cpu(), M, D, offset, tail_seed=1000 + 31 * M + D + (7 if offset else 0), device=device)
    return a


# Small cases of the per-Gaussian gradient checks, one per SH storage family: (M, D, shs offset by 4 bytes, scale_modifier);
# "precomp" renders colors_precomp + cov3D_precomp.  Opacity is capped at 0.95 so alpha stays below the 0.99 clamp, whose
# derivative the reference drops by design.
GRAD_FAMILIES = {"M1_D0": (1, 0, False, 1.0), "M4_D1": (4, 1, False, 0.9), "M9_D2": (9, 2, False, 1.0), "M16_D3": (16, 3, False, 1.1),
                 "M25_D3": (25, 3, False, 1.0), "M25_D2_off": (25, 2, True, 1.0), "precomp": (None, 0, False, 1.0)}


def grad_args(family: str, device=None, opacity_cap: float = 0.95) -> Dict:
    M, D, offset, mod = GRAD_FAMILIES[family]
    g = scene.synthetic_gaussians(400, seed=61 + len(family), extent=(1.6, 1.6, 1), log_scale_mean=math.log(0.07), log_scale_std=0.5,
                                  sh_degree=4, opacity_mean=0.0, opacity_std=1.5)
    g["shs"][:, 0] *= 4.0
    g["opacities"] = g["opacities"].clamp(max=opacity_cap)
    cam = scene.lookat_camera((0.5, -2.4, 0.7), (0, 0, 0), 70, 54, 50.0)  # a fifth of the Gaussians fall outside the view
    case = dict(g=g, cam=cam, sh_degree=D, bg=(0.3, 0.1, 0.6), scale_modifier=mod, precomp=M is None)
    a = resolve(case, device)
    if M is None:
        a["colors_precomp"] = (a["colors_precomp"] * 1.2 - 0.1).contiguous()
    else:
        a["shs"] = sh_layout(g["shs"], M, D, offset, tail_seed=77, device=device)
    return a


def isolated_image_grads(a: Dict, term: str, device=None):
    """image_grads with all but one of dL/dcolor, dL/ddepth, dL/dalpha set to zero (term "all" keeps the three, "extra", the loss
    on the second colour set's image alone, none)."""
    dc, dd, da = image_grads(a, device=device)
    keep = {"color": (1, 0, 0), "depth": (0, 1, 0), "alpha": (0, 0, 1), "all": (1, 1, 1), "extra": (0, 0, 0)}[term]
    return dc * keep[0], dd * keep[1], da * keep[2]


def extra_pass(a: Dict, extra: torch.Tensor) -> Dict:
    """The arguments of the pass that blends a second colour set extra [P,3] (the normals of render()) with the same weights: a's
    geometry with colors_precomp = extra."""
    return dict(a, shs=None, colors_precomp=extra)


def extra_image_grad(a: Dict, term: str, device=None) -> torch.Tensor:
    """dL/dE of the second colour set's image, ~ N(0,1) with seed 8, under the terms "extra" and "all"; zeros under the others."""
    de = torch.randn(3, a["H"], a["W"], generator=torch.Generator().manual_seed(8))
    de = de if term in ("extra", "all") else torch.zeros_like(de)
    return de if device is None else de.to(device)


def row_errors(g, g64) -> np.ndarray:
    """Per-Gaussian relative error ||g - g64|| / ||g64|| over the rows whose ||g64|| exceeds 1e-6 of the largest row."""
    g = torch.as_tensor(g).detach().double().cpu().reshape(g64.shape[0], -1)
    g64 = torch.as_tensor(g64).detach().double().cpu().reshape(g64.shape[0], -1)
    n = g64.norm(dim=1)
    keep = n > 1e-6 * n.max()
    return ((g - g64).norm(dim=1)[keep] / n[keep]).numpy()


def fp64_grads(a: Dict, fw, terms, oracle_decisions=False, extra=None) -> Dict:
    """{term: {name: fp64 autograd gradient}} of torch_ref.render on the oracle's tile lists, for each isolated loss term.  Names
    follow the oracle's dL_d* keys; dL_dmeans2D holds the pixel gradient scaled to the reference's units (0.5 W, 0.5 H).  The
    frustum clamp is differentiated as the reference does (Gaussians near the image border differ from the true gradient).
    oracle_decisions: the skip / terminate decisions are the oracle's fp32 ones, so that a row differs only by arithmetic (else
    they are taken on the fp64 values).
    extra: (b, fb), the extra_pass arguments of a second colour set and the oracle's forward of them.  Each term's gradients are
    then those of both passes summed, the second's loss being dL/dE (extra_image_grad) . E, and its dL/dcolors is dL_dextra."""
    from tests import torch_ref
    names = {"means3D": "dL_dmeans3D", "opacities": "dL_dopacity", "shs": "dL_dsh", "scales": "dL_dscales", "rotations": "dL_drotations",
             "colors_precomp": "dL_dcolors", "cov3D_precomp": "dL_dcov3D"}
    passes = [(a, fw, False)] + ([(extra[0], extra[1], True)] if extra is not None else [])
    graphs = [torch_ref.render(p, f, reference_clamp_grad=True, oracle_decisions=oracle_decisions) + (second,) for p, f, second in passes]
    out = {}
    for term in terms:
        res = {}
        for color, depth, alpha, leaves, m2d, second in graphs:
            weights = (extra_image_grad(a, term),) if second else isolated_image_grads(a, term)
            loss = sum((img * w.double()).sum() for img, w in zip((color, depth, alpha), weights))
            inputs = [(k, v) for k, v in leaves.items() if v is not None] + [("means2D", m2d)]
            if any(bool(w.any()) for w in weights):
                gs = torch.autograd.grad(loss, [v for _, v in inputs], retain_graph=True, allow_unused=True)
            else:  # a pass the term leaves out of the loss: zero gradients without an autograd pass
                gs = [None] * len(inputs)
            for (k, v), gr in zip(inputs, gs):
                gr = torch.zeros_like(v) if gr is None else gr
                if k == "means2D":
                    key, gr = "dL_dmeans2D", gr * torch.tensor([0.5 * a["W"], 0.5 * a["H"]], dtype=torch.float64)
                else:
                    key = "dL_dextra" if (second and k == "colors_precomp") else names[k]
                res[key] = res[key] + gr if key in res else gr
        out[term] = res
    return out


def oracle_two_pass_grads(a: Dict, fw, b: Dict, fb, dc, dd, da, de) -> Dict:
    """comparable_grads of the oracle's backward of the colour pass a (loss dc, dd, da) plus that of the extra pass b (loss de on its
    colour image): the gradients of a frame that blends both colour sets with the same weights, dL_dextra the second's dL/dcolors."""
    o1 = comparable_grads(oracle_backward(a, fw, dc, dd, da), a)
    o2 = comparable_grads(oracle_backward(b, fb, de, 0 * dd, 0 * da), b)
    o = {k: (v + o2[k] if k in o2 and o2[k].shape == v.shape else v) for k, v in o1.items() if k != "dL_dcolors"}
    o["dL_dextra"] = o2["dL_dcolors"]
    if a["colors_precomp"] is not None:
        o["dL_dcolors"] = o1["dL_dcolors"]
    return o


def comparable_grads(g: Dict, a: Dict) -> Dict:
    """An oracle-style gradient dict (dL_d* keys) reduced to what fp64_grads holds: dL_dmeans2D without its unused third column, and
    dL_dscales times scale_modifier (the reference reports the gradient w.r.t. scale_modifier * scale, backward.cu:318-321)."""
    out = {}
    for k, v in g.items():
        v = torch.as_tensor(v).detach().double().cpu()
        if k == "dL_dmeans2D":
            v = v[:, :2]
        elif k == "dL_dscales":
            v = v * a["scale_modifier"]
        out[k] = v
    return out


def load_golden(path: str) -> Dict:
    """A golden case; the gradients of the larger cases are stored beside it under golden/grads/ (same file name)."""
    gold = dict(np.load(path))
    grads = os.path.join(os.path.dirname(path), "grads", os.path.basename(path))
    if os.path.exists(grads):
        gold.update(np.load(grads))
    return gold


def cov3d_from(scales: torch.Tensor, rotations: torch.Tensor, mod: float) -> torch.Tensor:
    """Python-side precomputed covariance (what gaussian_model.get_covariance builds, gaussian_model.py:47-52,117-118)."""
    r, x, y, z = rotations.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).view(-1, 3, 3)
    L = R * (scales * mod).unsqueeze(1)  # R @ diag(s)
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=-1).contiguous()


def resolve(case: Dict, device=None) -> Dict:
    """Flatten a case into the exact argument set of one rasterizer call."""
    g, cam = case["g"], case["cam"]
    a = dict(means3D=g["means3D"], opacities=g["opacities"], view=cam.world_view_transform, proj=cam.full_proj_transform,
             campos=cam.camera_center, W=cam.image_width, H=cam.image_height, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
             sh_degree=case["sh_degree"], scale_modifier=case["scale_modifier"], bg=torch.tensor(case["bg"], dtype=torch.float32),
             shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None)
    if case.get("precomp"):
        gen = torch.Generator().manual_seed(99)
        a["colors_precomp"] = torch.rand(g["means3D"].shape[0], 3, generator=gen)
        a["cov3D_precomp"] = cov3d_from(g["scales"], g["rotations"], case["scale_modifier"])
    else:
        a["shs"], a["scales"], a["rotations"] = g["shs"], g["scales"], g["rotations"]
    if device is not None:
        a = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in a.items()}
    return a


def settings_from(a: Dict, debug=False, prefiltered=False):
    from autovfx_b200.rasterizer import GaussianRasterizationSettings
    return GaussianRasterizationSettings(image_height=a["H"], image_width=a["W"], tanfovx=a["tanfovx"], tanfovy=a["tanfovy"], bg=a["bg"],
                                         scale_modifier=a["scale_modifier"], viewmatrix=a["view"], projmatrix=a["proj"],
                                         sh_degree=a["sh_degree"], campos=a["campos"], prefiltered=prefiltered, debug=debug)


def run_ours(a: Dict, for_backward=False, sorted_keys=False, debug=True, tight=None, exact=None):
    from autovfx_b200 import rasterizer as R
    s = settings_from(a, debug=debug)
    color, depth, alpha, radii, ws, ticket, keep = R.forward_raw(a["means3D"], a["shs"], a["colors_precomp"], a["opacities"], a["scales"],
                                                                 a["rotations"], a["cov3D_precomp"], s, for_backward=for_backward,
                                                                 sorted_keys=sorted_keys, sync=True, tight=tight, exact=exact)
    views = R.debug_views(ws, a["means3D"].shape[0], a["W"], a["H"])
    return dict(color=color, depth=depth, alpha=alpha, radii=radii, views=views, stats=ticket.stats(), ws=ws, keep=keep)


def run_ref(a: Dict):
    """The compiled reference's forward on the same tensors, or None where it is not built: comparisons against its outputs
    go through the ref_* helpers below, which replay stored digests of them in that case."""
    from oracle import ref_cuda
    if not ref_cuda.available():
        return None
    fw = ref_cuda.forward(a["means3D"], a["opacities"], a["view"], a["proj"], a["campos"], a["W"], a["H"], a["tanfovx"], a["tanfovy"],
                          shs=a["shs"], colors_precomp=a["colors_precomp"], scales=a["scales"], rotations=a["rotations"],
                          cov3D_precomp=a["cov3D_precomp"], sh_degree=a["sh_degree"], scale_modifier=a["scale_modifier"], bg=a["bg"])
    return fw


def ref_state(device):
    """ref_cuda.state() after run_ref, or None where the reference is not built."""
    from oracle import ref_cuda
    return ref_cuda.state(device) if ref_cuda.available() else None


def ref_backward(a: Dict, dc, dd, da):
    """The reference's gradients for run_ref(a), or None where the reference is not built."""
    from oracle import ref_cuda
    return ref_cuda.backward(run_ref(a), dc, dd, da) if ref_cuda.available() else None


def run_oracle(a: Dict, stop_after="render"):
    from oracle import gsr_oracle as O
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    return O.forward(n(a["means3D"]), n(a["opacities"]), n(a["view"]), n(a["proj"]), n(a["campos"]), a["W"], a["H"], a["tanfovx"],
                     a["tanfovy"], shs=n(a["shs"]), colors_precomp=n(a["colors_precomp"]), scales=n(a["scales"]), rotations=n(a["rotations"]),
                     cov3D_precomp=n(a["cov3D_precomp"]), sh_degree=a["sh_degree"], scale_modifier=a["scale_modifier"],
                     bg=tuple(float(v) for v in a["bg"].cpu()), stop_after=stop_after)


def oracle_backward(a: Dict, fw, dc, dd, da):
    from oracle import gsr_oracle as O
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    return O.backward(fw, n(a["means3D"]), n(a["view"]), n(a["proj"]), n(a["campos"]), a["W"], a["H"], a["tanfovx"], a["tanfovy"],
                      n(dc), n(dd), n(da), shs=n(a["shs"]), colors_precomp=n(a["colors_precomp"]), scales=n(a["scales"]),
                      rotations=n(a["rotations"]), cov3D_precomp=n(a["cov3D_precomp"]), sh_degree=a["sh_degree"],
                      scale_modifier=a["scale_modifier"], bg=tuple(float(v) for v in a["bg"].cpu()))


def image_grads(a: Dict, seed=7, device=None):
    """dL/dcolor, dL/ddepth, dL/dalpha ~ N(0,1), seed 7 (SURVEY §8d config 3)."""
    g = torch.Generator().manual_seed(seed)
    H, W = a["H"], a["W"]
    dc, dd, da = torch.randn(3, H, W, generator=g), torch.randn(1, H, W, generator=g), torch.randn(1, H, W, generator=g)
    if device is not None:
        dc, dd, da = dc.to(device), dd.to(device), da.to(device)
    return dc, dd, da


def ours_backward(a: Dict, dc, dd, da):
    """Forward+backward through the public GaussianRasterizer API; returns (outputs, grads dict)."""
    from autovfx_b200.rasterizer import GaussianRasterizer
    leaves = {}
    for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"):
        leaves[k] = None if a[k] is None else a[k].detach().clone().requires_grad_(True)
    means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
    rast = GaussianRasterizer(settings_from(a))
    color, depth, alpha, radii = rast(leaves["means3D"], means2D, leaves["opacities"], shs=leaves["shs"], colors_precomp=leaves["colors_precomp"],
                                      scales=leaves["scales"], rotations=leaves["rotations"], cov3D_precomp=leaves["cov3D_precomp"])
    loss = (color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()
    loss.backward()
    grads = {k: (None if v is None else v.grad) for k, v in leaves.items()}
    grads["means2D"] = means2D.grad
    return (color, depth, alpha, radii), grads


# default (fast-alpha) blend against exact images: the measured differences are ~1e-6 of the value; BASELINE allows 1e-4
FAST_TOL = {"color": 1e-5, "alpha": 1e-5, "depth": 5e-5}


def assert_images_close(got: Dict, want: Dict, tol=None):
    for k in ("color", "depth", "alpha"):
        t = FAST_TOL[k] if tol is None else tol
        e = maxabs(got[k], want[k])
        assert e <= t, "%s: max abs %.3g > %.3g" % (k, e, t)


def maxabs(a, b) -> float:
    a = torch.as_tensor(a).float().cpu()
    b = torch.as_tensor(b).float().cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max())


def relerr(a, b) -> float:
    """max |a-b| / (max|b| + tiny): scale-aware error for gradient tensors."""
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ---- comparisons against the compiled reference (oracle/_ref), live or replayed ---------------------------------------------
# Each ref_* call compares one of our tensors with a value of the reference, passed as a function that computes it.  Where the
# reference library is built the function runs and the comparison is exact, and with GSR_REF_RECORD=<dir> every value is also
# stored, in call order, as <dir>/<test id>.npz: a SHA-256 of its bytes for bit-identity checks, a seeded sample of REF_SAMPLE
# elements (plus its max |value|) for tolerance checks: one per block of the flattened tensor.  Where
# an exact-mode image is shown bit-identical to the reference, tests also compare the default-mode image with it in full.  Where the library is absent the functions are never called and the same
# comparisons run against tests/golden/ref/<test id>.npz, recorded by the reference on an H100.
REF_GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")
REF_SAMPLE = 2048
_ref_log: Dict = {"test": None, "i": 0, "rec": {}}


def _test_id() -> str:
    tid = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    return "".join(c if c.isalnum() or c in "-_." else "_" for c in tid.replace("tests/", "", 1))


def use_ref_python():
    """Declares that the running test's reference values come from the reference's Python code (oracle/ref_py): its comparisons
    run live only where that code is staged (not merely the compiled library) and replay the stored values elsewhere."""
    _ref_log["py_test"] = _test_id()


def ref_live() -> bool:
    """Whether the running test's reference values are computed here (else they are replayed)."""
    from oracle import ref_cuda, ref_py
    return ref_py.available() if _ref_log.get("py_test") == _test_id() else ref_cuda.available()


def have_ref() -> bool:
    """The reference is built here, or its values are stored for the running test."""
    return ref_live() or os.path.exists(os.path.join(REF_GOLDEN, _test_id() + ".npz"))


def _canon(t) -> torch.Tensor:
    t = torch.as_tensor(t).detach()
    t = t.float() if t.is_floating_point() else t.long()
    return t.contiguous().cpu()


def _digest(t: torch.Tensor) -> str:
    import hashlib
    return hashlib.sha256(str(tuple(t.shape)).encode() + t.numpy().tobytes()).hexdigest()


def _sample_idx(n: int) -> np.ndarray:
    """Stratified: one seeded element from each of REF_SAMPLE equal blocks of the flattened tensor, so every region is covered."""
    if n <= REF_SAMPLE:
        return np.arange(n)
    edges = (np.arange(REF_SAMPLE + 1, dtype=np.int64) * n) // REF_SAMPLE
    return edges[:-1] + np.random.default_rng(n).integers(0, edges[1:] - edges[:-1])


def _ref_entry(kind: str, fn):
    """The reference's record for the next comparison of the running test: computed by fn (and stored when recording) or replayed."""
    tid = _test_id()
    if _ref_log["test"] != tid:
        _ref_log.update(test=tid, i=0, rec={})
    i = _ref_log["i"]
    _ref_log["i"] += 1
    if not ref_live():
        path = os.path.join(REF_GOLDEN, tid + ".npz")
        if tid not in _ref_log["rec"]:
            assert os.path.exists(path), "no compiled reference and no stored reference values (%s)" % path
            _ref_log["rec"][tid] = dict(np.load(path))
        rec = _ref_log["rec"][tid]
        assert "%d_kind" % i in rec and str(rec["%d_kind" % i]) == kind, "stored reference values do not match comparison %d" % i
        return None, {k.split("_", 1)[1]: v for k, v in rec.items() if k.split("_", 1)[0] == str(i)}
    v = fn()
    out = os.environ.get("GSR_REF_RECORD")
    if out:
        e = {"kind": np.str_(kind)}
        if kind == "value":
            e["value"] = np.asarray(v)
        else:
            c = _canon(v)
            e["shape"] = np.asarray(c.shape, dtype=np.int64)
            if kind == "same":
                e["sha"] = np.str_(_digest(c))
            else:
                flat = c.double().reshape(-1)
                e["sample"] = flat[torch.from_numpy(_sample_idx(flat.numel()))].float().numpy()
                e["absmax"] = np.asarray(float(flat.abs().max()) if flat.numel() else 0.0)
        rec = _ref_log["rec"].setdefault(tid, {})
        rec.update({"%d_%s" % (i, k): x for k, x in e.items()})
        os.makedirs(out, exist_ok=True)
        np.savez_compressed(os.path.join(out, tid + ".npz"), **rec)
    return v, None


def ref_value(fn):
    """A scalar of the reference (e.g. num_rendered)."""
    v, rec = _ref_entry("value", fn)
    return v if rec is None else rec["value"].item()


def ref_same(x, fn) -> bool:
    """Bit identity with a tensor of the reference (integers compared as int64, floats as float32)."""
    v, rec = _ref_entry("same", fn)
    if rec is None:
        a, b = _canon(x), _canon(v)
        return a.shape == b.shape and torch.equal(a, b)
    c = _canon(x)
    return list(c.shape) == rec["shape"].tolist() and _digest(c) == str(rec["sha"])


def _ref_pair(x, fn):
    v, rec = _ref_entry("sample", fn)
    a = _canon(x).double().reshape(-1)
    if rec is None:
        return a, _canon(v).double().reshape(-1), None
    assert a.numel() == int(np.prod(rec["shape"])), "shape differs from the stored reference values"
    return a[torch.from_numpy(_sample_idx(a.numel()))], torch.from_numpy(rec["sample"]).double(), float(rec["absmax"])


def ref_maxabs(x, fn) -> float:
    a, b, _ = _ref_pair(x, fn)
    return float((a - b).abs().max()) if a.numel() else 0.0


def ref_meanabs(x, fn) -> float:
    a, b, _ = _ref_pair(x, fn)
    return float((a - b).abs().mean()) if a.numel() else 0.0


def ref_allclose(x, fn, rtol: float) -> bool:
    a, b, _ = _ref_pair(x, fn)
    return bool(((a - b).abs() <= rtol * b.abs()).all())


def ref_relerr(x, fn) -> float:
    a, b, bmax = _ref_pair(x, fn)
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / ((float(b.abs().max()) if bmax is None else bmax) + 1e-30))


def ref_images_close(got: Dict, ref, tol=None):
    """assert_images_close against the reference's forward (run_ref's result, None where replayed)."""
    for k in ("color", "depth", "alpha"):
        t = FAST_TOL[k] if tol is None else tol
        e = ref_maxabs(got[k], lambda: ref[k])
        assert e <= t, "%s: max abs %.3g > %.3g" % (k, e, t)
