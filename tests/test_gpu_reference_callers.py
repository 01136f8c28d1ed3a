"""The reference's OWN Python callers of the hot path against the drop-in (SURVEY §8 rows a17, a19, b, f-1..f-4).

``make -C oracle ref refpy`` stages unmodified copies of the reference's ``render()`` (gaussian_renderer/__init__.py:83-218),
``GaussianModel`` (scene/gaussian_model.py), ``Camera`` (scene/cameras.py), ``transform_gaussians`` / ``merge_two_gaussians``
(gaussians_utils.py:71-125) and its Python autograd front end into the git-ignored ``oracle/_ref_py`` where the reference sources are
available; ``oracle/ref_py.py`` binds them either to this repository's drop-in packages or to the reference's own CUDA (oracle/_ref).
Tests taking ``ref_ns`` compare our code with values the reference code computes, through the Hh.ref_* helpers: live where the
reference is staged, replayed from tests/golden/ref/ elsewhere.  Tests taking ``rp`` execute the reference's code ON the drop-in and
need it staged.
"""
import math
import os
import types

import numpy as np
import pytest
import torch

from tests import helpers as Hh
from tests import wrapper_ref as WR
from tests.test_wrapper_cpu import _raw, _rot
from autovfx_b200 import scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ref():
    from oracle import ref_py
    if not ref_py.available():
        pytest.skip("oracle/_ref_py or oracle/_ref not staged (make -C oracle ref refpy REF=<reference checkout>)")
    return ref_py


@pytest.fixture(scope="module")
def rp():
    """For the tests that execute the reference's Python code on the drop-in: they need that code staged."""
    return _ref()


@pytest.fixture
def ref_ns():
    """The reference's Python modules, loaded on first use.  The tests taking this fixture only call it inside the functions
    they pass to the Hh.ref_* comparisons, which replay stored reference values where the reference is not staged."""
    Hh.use_ref_python()
    if not Hh.have_ref():
        pytest.skip("no staged reference and no stored reference values")
    cache = {}

    def load():
        from oracle import ref_py
        if "ns" not in cache:
            cache["rp"], cache["ns"] = ref_py, ref_py.load("ref")
        return cache["rp"], cache["ns"]
    return load


def _once(fn):
    """fn() evaluated at most once (a reference computation several comparisons read from)."""
    box = []
    return lambda: box[0] if box else (box.append(fn()) or box[0])


class _Model:
    """What the reference's GaussianModel exposes to render(): its get_* activations (tests/wrapper_ref.activate, the same torch
    ops on the same device, hence the same bits) and get_normal (gaussian_model.py:120-128)."""

    def __init__(self, raw, max_sh_degree, active_sh_degree):
        a = WR.activate({k: v.to(DEV).float().contiguous() for k, v in raw.items()})
        self.get_xyz, self.get_features, self.get_opacity = a["means3D"], a["shs"], a["opacities"]
        self.get_scaling, self.get_rotation = a["scales"], a["rotations"]
        self.max_sh_degree, self.active_sh_degree = max_sh_degree, active_sh_degree

    def get_normal(self, dir_pp_normalized=None):
        n, _ = WR.flip_align_view(WR.get_minimum_axis(self.get_scaling, self.get_rotation), dir_pp_normalized)
        return n / n.norm(dim=1, keepdim=True)


def _camera(c2w, fx, W, H):
    """The reference Camera's fields for a c2w pose: matrices from scene.camera_from_c2w (identical, see the camera test) and
    camera_center = world_view_transform.inverse()[3, :3] on the GPU, as scene/cameras.py computes it."""
    cam = scene.camera_from_c2w(c2w, fx, fx, W, H)
    view = cam.world_view_transform.to(DEV)
    return types.SimpleNamespace(FoVx=cam.FoVx, FoVy=cam.FoVy, image_width=W, image_height=H, world_view_transform=view,
                                 full_proj_transform=cam.full_proj_transform.to(DEV), camera_center=view.inverse()[3, :3])


PIPE = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)


def _scene_raw(N, M, seed, spread=1.0, log_scale=-3.3):
    r = _raw(N, M, seed)
    r["xyz"] = r["xyz"] * spread
    r["scaling"] = r["scaling"] * 0.6 + (log_scale + 3.0)
    r["f_dc"] = r["f_dc"] * 0.5
    return r


def _cam_args(eye=(0.4, -3.2, 0.6), target=(0, 0, 0), W=160, H=112, fovx_deg=58.0):
    """R, T, FoVx, FoVy exactly as scene_representation.py:144-156 derives them from a c2w."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    Rc = scene.rotm_from_lookat(target - eye, np.asarray((0.0, 0.0, 1.0)))
    c2w = np.vstack((np.hstack((Rc, eye.reshape(3, 1))), np.array([0, 0, 0, 1])))
    w2c = np.linalg.inv(c2w)
    fx = W / (2 * math.tan(math.radians(fovx_deg) / 2))
    return np.transpose(w2c[:3, :3]), w2c[:3, 3], scene.focal2fov(fx, W), scene.focal2fov(fx, H), W, H, c2w, fx


def test_reference_camera_class_matches_scene_helpers(rp):
    """scene/cameras.py Camera (the reference's own class) vs autovfx_b200.scene.camera_from_c2w: identical matrices."""
    ns = rp.load("ours")
    R, T, fovx, fovy, W, H, c2w, fx = _cam_args()
    cam = rp.make_camera(ns, R, T, fovx, fovy, W, H)
    mine = scene.camera_from_c2w(c2w, fx, fx, W, H)
    assert torch.equal(cam.world_view_transform.cpu(), mine.world_view_transform)
    assert torch.equal(cam.full_proj_transform.cpu(), mine.full_proj_transform)
    # the reference inverts the view matrix on the GPU (cuSOLVER), scene.py on the CPU (LAPACK): last-bit differences only
    assert torch.allclose(cam.camera_center.cpu(), mine.camera_center, rtol=0, atol=1e-6)
    assert cam.image_width == W and cam.image_height == H and cam.FoVx == mine.FoVx and cam.FoVy == mine.FoVy


@pytest.mark.parametrize("M,deg", [(16, 3), (25, 1), (25, 3)])
def test_reference_render_on_dropin_equals_reference_render_on_reference(rp, M, deg):
    """The reference's render() with `diff_gaussian_rasterization` = this repo's drop-in, against the same render() on the
    reference's Python + CUDA rasterizer.  Exact image mode: every output bit-identical (the torch post-processing is the same
    code fed identical rasterizer outputs).  Default mode: within the 1e-4 image tolerance."""
    from autovfx_b200 import rasterizer as R
    ours, ref = rp.load("ours"), rp.load("ref")
    raw = _scene_raw(5000, M, 11)
    Rm, T, fovx, fovy, W, H, _, _ = _cam_args()
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    outs = {}
    for tag, ns in (("ours", ours), ("ref", ref)):
        pc = rp.make_model(ns, raw, int(math.isqrt(M)) - 1, deg)
        cam = rp.make_camera(ns, Rm, T, fovx, fovy, W, H)
        modes = (True, False) if tag == "ours" else (None,)
        for exact in modes:
            if exact is not None:
                R.set_exact_images(exact)
            try:
                with torch.no_grad():
                    o = ns.renderer.render(cam, pc, rp.Pipe(), bg)
            finally:
                R.set_exact_images(False)
            outs[(tag, exact)] = {k: v.detach().clone() for k, v in o.items() if isinstance(v, torch.Tensor)}
    want = outs[("ref", None)]
    ex = outs[("ours", True)]
    for k in ("render", "depth", "normal", "pseudo_normal", "radii", "visibility_filter"):
        assert torch.equal(ex[k], want[k]), k
    fast = outs[("ours", False)]
    assert torch.equal(fast["radii"], want["radii"])
    assert Hh.maxabs(fast["render"], want["render"]) <= 1e-5 and Hh.maxabs(fast["depth"], want["depth"]) <= 5e-5
    assert Hh.maxabs(fast["normal"], want["normal"]) <= 1e-4


@pytest.mark.parametrize("M,deg", [(16, 3), (25, 2)])
def test_fused_render_matches_reference_render(ref_ns, M, deg):
    """autovfx_b200.renderer.render (axis normals + ONE 6-channel pass + normal-map kernel) on the parameters and camera of a
    reference GaussianModel / Camera, against the reference's render() on the reference rasterizer."""
    from autovfx_b200 import rasterizer as R, renderer as RD
    raw = _scene_raw(6000, M, 5)
    Rm, T, fovx, fovy, W, H, c2w, fx = _cam_args(eye=(-2.0, -2.4, 1.1), W=176, H=96)
    bg = torch.tensor([0.0, 0.0, 0.0], device=DEV)
    pc, cam = _Model(raw, int(math.isqrt(M)) - 1, deg), _camera(c2w, fx, W, H)

    @_once
    def want():
        rp, ns = ref_ns()
        with torch.no_grad():
            return ns.renderer.render(rp.make_camera(ns, Rm, T, fovx, fovy, W, H), rp.make_model(ns, raw, int(math.isqrt(M)) - 1, deg), rp.Pipe(), bg)
    with torch.no_grad():
        R.set_exact_images(True)
        try:
            got = RD.render(cam, pc, PIPE, bg)
        finally:
            R.set_exact_images(False)
        fast = RD.render(cam, pc, PIPE, bg)
    for k in ("render", "depth", "radii", "visibility_filter"):
        assert Hh.ref_same(got[k], lambda: want()[k]), k
    assert Hh.ref_maxabs(got["normal"], lambda: want()["normal"]) <= 1e-4  # blended normal image: per-Gaussian normals differ in the last bit
    # pseudo normal: normalised cross product of depth differences (cancellation): compare directions where the normal is defined,
    # against the reference's expression (tests/wrapper_ref.pseudo_normal) on the depth image, which equals the reference's bit for bit
    a = got["pseudo_normal"]
    b = WR.pseudo_normal(got["depth"].reshape(H, W), cam.world_view_transform, cam.FoVx, cam.FoVy)
    defined = (b.norm(dim=-1) > 0.5) & (a.norm(dim=-1) > 0.5)
    cos = (a * b).sum(-1)[defined]
    assert defined.float().mean() > 0.5 and float((cos > 1 - 5e-3).float().mean()) > 0.999
    assert Hh.ref_maxabs(fast["render"], lambda: want()["render"]) <= 1e-5 and Hh.ref_maxabs(fast["depth"], lambda: want()["depth"]) <= 5e-5
    assert Hh.maxabs(fast["render"], got["render"]) <= 1e-5 and Hh.maxabs(fast["depth"], got["depth"]) <= 5e-5  # every pixel


def test_training_step_through_reference_render_gradients(rp):
    """Backward through the reference's render() (two rasterizer passes, gradients w.r.t. the raw GaussianModel parameters) on the
    drop-in vs on the reference's autograd front end + CUDA backward."""
    ours, ref = rp.load("ours"), rp.load("ref")
    raw = _scene_raw(3000, 16, 23)
    Rm, T, fovx, fovy, W, H, _, _ = _cam_args(W=128, H=96)
    bg = torch.tensor([0.2, 0.2, 0.2], device=DEV)
    gen = torch.Generator().manual_seed(3)
    w_img, w_d, w_n = torch.randn(4, H, W, generator=gen).to(DEV), torch.randn(H, W, generator=gen).to(DEV), torch.randn(H, W, 3, generator=gen).to(DEV)
    grads = {}
    for tag, ns in (("ours", ours), ("ref", ref)):
        pc = rp.make_model(ns, raw, 3, 3)
        cam = rp.make_camera(ns, Rm, T, fovx, fovy, W, H)
        o = ns.renderer.render(cam, pc, rp.Pipe(), bg)
        loss = (o["render"] * w_img).sum() + (o["depth"] * w_d).sum() + (o["normal"] * w_n).sum()
        loss.backward()
        grads[tag] = {"xyz": pc._xyz.grad, "f_dc": pc._features_dc.grad, "f_rest": pc._features_rest.grad, "opacity": pc._opacity.grad,
                      "scaling": pc._scaling.grad, "rotation": pc._rotation.grad, "screen": o["viewspace_points"].grad}
    for k, g in grads["ours"].items():
        assert g is not None and grads["ref"][k] is not None, k
        assert Hh.relerr(g, grads["ref"][k]) < 3e-4, k


def test_create_from_pcd_uses_distcuda2(rp):
    """GaussianModel.create_from_pcd (gaussian_model.py:134-157), the only real distCUDA2 call site: initial log-scales from the
    drop-in simple_knn._C vs the reference's simple-knn CUDA."""
    ours, ref = rp.load("ours"), rp.load("ref")
    gen = np.random.default_rng(4)
    pts = (gen.standard_normal((20000, 3)) * np.array([2.0, 1.0, 0.4])).astype(np.float32)
    cols = gen.random((20000, 3)).astype(np.float32)
    models = {}
    for tag, ns in (("ours", ours), ("ref", ref)):
        pcd = ns.graphics_utils.BasicPointCloud(points=pts, colors=cols, normals=np.zeros_like(pts))
        m = ns.gaussian_model.GaussianModel(3)
        m.create_from_pcd(pcd, 1.0)
        models[tag] = m
    a, b = models["ours"], models["ref"]
    assert torch.allclose(a._scaling, b._scaling, rtol=0, atol=2e-6) and torch.equal(a._xyz, b._xyz)
    assert torch.equal(a._features_dc, b._features_dc) and torch.equal(a._opacity, b._opacity) and torch.equal(a._rotation, b._rotation)


@pytest.mark.parametrize("M", [16, 25])
def test_activations_match_reference_gaussian_model(ref_ns, M):
    """edit.activate (gsr_activate_gaussians) vs the reference GaussianModel's get_* properties (gaussian_model.py:95-115)."""
    from autovfx_b200 import edit
    raw = _scene_raw(40000, M, 9)

    @_once
    def pc():
        rp, ns = ref_ns()
        return rp.make_model(ns, raw, int(math.isqrt(M)) - 1, 0)
    got = edit.activate({k: v.to(DEV) for k, v in raw.items()}, DEV)
    with torch.no_grad():
        assert Hh.ref_same(got["means3D"], lambda: pc().get_xyz) and Hh.ref_same(got["shs"], lambda: pc().get_features)
        assert Hh.ref_same(got["scales"], lambda: pc().get_scaling)
        assert Hh.ref_maxabs(got["opacities"], lambda: pc().get_opacity) <= 1.2e-7
        assert Hh.ref_maxabs(got["rotations"], lambda: pc().get_rotation) <= 2.4e-7


def test_get_normal_matches_reference(ref_ns):
    """renderer.axis_normals (gsr_axis_normals) vs GaussianModel.get_normal (gaussian_model.py:120-128), on the model's activations."""
    from autovfx_b200 import renderer as RD
    raw = _scene_raw(50000, 16, 13)
    campos = torch.tensor([0.3, -2.0, 0.7], device=DEV)

    def want():
        rp, ns = ref_ns()
        pc = rp.make_model(ns, raw, 3, 3)
        with torch.no_grad():
            d = pc.get_xyz - campos
            return pc.get_normal(dir_pp_normalized=d / d.norm(dim=1, keepdim=True))
    pc = _Model(raw, 3, 3)
    with torch.no_grad():
        got = RD.axis_normals(pc.get_xyz, pc.get_scaling, pc.get_rotation, campos, remap01=False)
    assert Hh.ref_maxabs(got, want) <= 5e-7


def test_transform_and_merge_match_reference(ref_ns):
    """edit.ResidentScene.compose vs the reference's transform_gaussians + merge_two_gaussians executed from gaussians_utils.py
    (:71-125), then both scenes through the rasterizer."""
    from autovfx_b200 import edit
    M = 25
    scene_raw, obj_raw = _scene_raw(8000, M, 1), _scene_raw(1500, M, 2, spread=0.3)
    Rot = _rot(5)
    center, init_c, scaling = torch.tensor([0.4, -0.2, 0.3]), torch.tensor([0.05, 0.02, -0.01]), 1.7

    @_once
    def want():
        rp, ns = ref_ns()
        bg_model, obj_model = rp.make_model(ns, scene_raw, 4, 0), rp.make_model(ns, obj_raw, 4, 0)
        with torch.no_grad():
            moved = ns.gaussians_utils.transform_gaussians(obj_model, center.to(DEV), Rot.to(DEV), scaling, init_c.to(DEV))
            merged = ns.gaussians_utils.merge_two_gaussians(bg_model, moved)
            assert merged.active_sh_degree == 0
            return {"means3D": merged.get_xyz, "shs": merged.get_features, "opacities": merged.get_opacity, "scales": merged.get_scaling,
                    "rotations": merged.get_rotation}
    rs = edit.ResidentScene({k: v.to(DEV) for k, v in scene_raw.items()}, {"obj": {k: v.to(DEV) for k, v in obj_raw.items()}}, DEV)
    got = rs.compose({"obj": (center, Rot, scaling, init_c)})
    assert Hh.ref_maxabs(got["means3D"], lambda: want()["means3D"]) <= 2e-6 and Hh.ref_same(got["shs"], lambda: want()["shs"])
    smax = Hh.ref_value(lambda: float(want()["scales"].max()))
    assert Hh.ref_maxabs(got["scales"], lambda: want()["scales"]) <= 1e-6 * smax + 1e-9
    assert Hh.ref_maxabs(got["opacities"], lambda: want()["opacities"]) <= 1.2e-7
    assert Hh.ref_maxabs(got["rotations"], lambda: want()["rotations"]) <= 1e-6
    # the merged model renders at active_sh_degree 0 (gaussians_utils.py:75 builds GaussianModel(4): active degree 0)
    Rm, T, fovx, fovy, W, H, c2w, fx = _cam_args(W=144, H=96)
    cam = scene.camera_from_c2w(c2w, fx, fx, W, H).to(DEV)
    a = dict(means3D=None, opacities=None, view=cam.world_view_transform, proj=cam.full_proj_transform, campos=cam.camera_center, W=W, H=H,
             tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, sh_degree=0, scale_modifier=1.0, bg=torch.zeros(3, device=DEV),
             shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None)
    b = dict(a)
    b.update({k: got[k].contiguous() for k in ("means3D", "opacities", "shs", "scales", "rotations")})
    ours = Hh.run_ours(b, exact=True)
    ref = Hh.run_ref(b)  # the composed parameters: drop-in == reference rasterizer, bit for bit
    assert Hh.ref_same(ours["color"], lambda: ref["color"]) and Hh.ref_same(ours["radii"], lambda: ref["radii"])

    def ref_of_reference_merge():  # the reference rasterizer on the scene composed by the reference's torch ops
        c = dict(a)
        c.update({k: want()[k].contiguous() for k in ("means3D", "opacities", "shs", "scales", "rotations")})
        return Hh.run_ref(c)["color"]
    assert Hh.ref_maxabs(ours["color"], ref_of_reference_merge) <= 2e-4


def test_ply_round_trip_with_reference_gaussian_model(rp, tmp_path):
    """save_ply written by the reference GaussianModel is read by scene.load_ply, and scene.save_ply is read by the reference's
    load_ply (gaussian_model.py:201-266): identical raw parameters both ways; both files are byte-identical."""
    ns = rp.load("ref")
    M = 16
    raw = _scene_raw(3000, M, 31)
    pc = rp.make_model(ns, raw, 3, 3)
    p_ref, p_ours = str(tmp_path / "ref" / "point_cloud.ply"), str(tmp_path / "ours.ply")
    pc.save_ply(p_ref)
    n = lambda t: t.detach().cpu().numpy()  # noqa: E731
    scene.save_ply(p_ours, n(raw["xyz"]), n(raw["f_dc"]), n(raw["f_rest"]), n(raw["opacity"]), n(raw["scaling"]), n(raw["rotation"]))
    assert open(p_ref, "rb").read() == open(p_ours, "rb").read()
    mine = scene.load_ply(p_ref)
    for k, kk in (("xyz", "xyz"), ("f_dc", "f_dc"), ("f_rest", "f_rest"), ("opacity", "opacity"), ("scale", "scaling"), ("rot", "rotation")):
        assert np.array_equal(mine[k], n(raw[kk])), k
    back = ns.gaussian_model.GaussianModel(3)
    back.load_ply(p_ours)
    assert torch.equal(back._xyz, pc._xyz) and torch.equal(back._features_dc, pc._features_dc) and torch.equal(back._features_rest, pc._features_rest)
    assert torch.equal(back._opacity, pc._opacity) and torch.equal(back._scaling, pc._scaling) and torch.equal(back._rotation, pc._rotation)


def test_sugar_style_call_offcentre_projection_and_python_sh(ref_ns):
    """The SuGaR wrapper's call shape (sugar_model.py:2010-2071): M = 25 storage, colours from the reference's Python eval_sh
    (utils/sh_utils.py) passed as colors_precomp, and a projection matrix whose principal point is patched off-centre
    (proj[2,0], proj[2,1] overwritten, sugar_model.py:2029-2030) — drop-in vs compiled reference, bit for bit."""
    from autovfx_b200 import renderer as RD
    g = scene.synthetic_gaussians(20000, seed=77, extent=(1.2, 1.2, 0.6), log_scale_mean=math.log(0.02), log_scale_std=0.5, sh_degree=4)
    cam = scene.lookat_camera((0.5, -3.0, 0.8), (0, 0, 0), 208, 144, 62.0)
    view = cam.world_view_transform.clone()
    proj = scene.projection_matrix(0.01, 100.0, cam.FoVx, cam.FoVy).transpose(0, 1).contiguous()
    proj[2, 0], proj[2, 1] = -0.11, 0.07  # principal point away from the image centre
    full = (view.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    a = Hh.resolve(dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), DEV)
    a["proj"] = full.to(DEV)
    with torch.no_grad():
        d = a["means3D"] - a["campos"]
        d = d / d.norm(dim=1, keepdim=True)
        shs_view = a["shs"].transpose(1, 2).reshape(-1, 3, 25)
        rgb = torch.clamp_min(RD._eval_sh_torch(3, shs_view, d) + 0.5, 0.0).contiguous()
        # the reference's Python eval_sh (utils/sh_utils.py), restated in renderer.py for pipe.convert_SHs_python: equal to float rounding
        assert Hh.ref_maxabs(rgb, lambda: torch.clamp_min(ref_ns()[1].sh_utils.eval_sh(3, shs_view, d) + 0.5, 0.0)) <= 2e-6
    b = dict(a)
    b["shs"], b["colors_precomp"] = None, rgb
    for case in (a, b):  # SH evaluated by the rasterizer at an off-centre projection, and the Python-SH colors_precomp call
        ours, ref = Hh.run_ours(case, exact=True, for_backward=True), Hh.run_ref(case)
        for k in ("color", "depth", "alpha", "radii"):
            assert Hh.ref_same(ours[k], lambda: ref[k]), k
        fast = Hh.run_ours(case)
        Hh.ref_images_close(fast, ref)
        Hh.assert_images_close(fast, ours)  # every pixel, against the exact images that equal the reference's
    # the CUDA SH evaluation agrees with the reference's Python eval_sh to float rounding
    assert Hh.maxabs(Hh.run_ours(a)["color"], Hh.run_ours(b)["color"]) <= 2e-5


def test_config2_one_million_through_the_ply_path(ref_ns, tmp_path):
    """BASELINE config 2 stand-in (SURVEY §8d): P = 1,000,000, seed 1, 4-unit scene, written and re-read through the 3DGS .ply vertex
    layout, activated on the GPU, one 1920x1080 camera, forward — drop-in vs compiled reference, bit for bit (exact image mode),
    and the default mode within tolerance."""
    from autovfx_b200 import edit
    raw = scene.config2_raw()
    path = str(tmp_path / "config2.ply")
    n = lambda t: t.numpy()  # noqa: E731
    scene.save_ply(path, n(raw["xyz"]), n(raw["f_dc"]), n(raw["f_rest"]), n(raw["opacity"]), n(raw["scaling"]), n(raw["rotation"]))
    assert os.path.getsize(path) > 1_000_000 * 62 * 4
    loaded = scene.load_ply(path)
    g = edit.activate({"xyz": torch.from_numpy(loaded["xyz"]), "f_dc": torch.from_numpy(loaded["f_dc"]), "f_rest": torch.from_numpy(loaded["f_rest"]),
                       "opacity": torch.from_numpy(loaded["opacity"]), "scaling": torch.from_numpy(loaded["scale"]),
                       "rotation": torch.from_numpy(loaded["rot"])}, DEV)
    cam = scene.config2_camera()
    a = Hh.resolve(dict(g=g, cam=cam, sh_degree=3, bg=(0.0, 0.0, 0.0), scale_modifier=1.0), DEV)
    ours, ref = Hh.run_ours(a, exact=True, debug=False), Hh.run_ref(a)
    assert Hh.ref_value(lambda: ref["num_rendered"]) == ours["stats"]["num_rendered"] > 1_000_000
    for k in ("color", "depth", "alpha", "radii"):
        assert Hh.ref_same(ours[k], lambda: ref[k]), k
    fast = Hh.run_ours(a, debug=False)
    Hh.ref_images_close(fast, ref)
    Hh.assert_images_close(fast, ours)  # every pixel, against the exact images that equal the reference's
    # the reference's own loader reads the same file to the same parameters (subset check: its per-property Python loops are slow)
    small = str(tmp_path / "small.ply")
    sl = slice(0, 20000)
    scene.save_ply(small, loaded["xyz"][sl], loaded["f_dc"][sl], loaded["f_rest"][sl], loaded["opacity"][sl], loaded["scale"][sl], loaded["rot"][sl])

    @_once
    def m():
        mm = ref_ns()[1].gaussian_model.GaussianModel(3)
        mm.load_ply(small)
        return mm
    with torch.no_grad():
        assert Hh.ref_same(g["means3D"][sl], lambda: m().get_xyz) and Hh.ref_same(g["shs"][sl], lambda: m().get_features)
        assert Hh.ref_same(g["scales"][sl], lambda: m().get_scaling)
