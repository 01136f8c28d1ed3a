"""CPU checks of rasterize_gaussians_multi, the differentiable two-colour-set rasterizer call: like every entry point it has no
CPU path, and it needs its second colour set.  Its numbers are checked on the GPU in
tests/test_gpu_fused_grads.py."""
import pytest
import torch

from autovfx_b200.rasterizer import GaussianRasterizationSettings, rasterize_gaussians_multi


def _settings():
    return GaussianRasterizationSettings(image_height=8, image_width=8, tanfovx=0.5, tanfovy=0.5, bg=torch.zeros(3), scale_modifier=1.0,
                                         viewmatrix=torch.eye(4), projmatrix=torch.eye(4), sh_degree=0, campos=torch.zeros(3),
                                         prefiltered=False, debug=False)


def test_multi_rejects_cpu_tensors():
    m = torch.zeros(4, 3, requires_grad=True)
    with pytest.raises(RuntimeError, match="no CPU path"):
        rasterize_gaussians_multi(m, torch.zeros(4, 3), torch.zeros(4, 16, 3), None, torch.zeros(4, 3), torch.zeros(4, 1), torch.ones(4, 3),
                                  torch.ones(4, 4), None, _settings())
    with pytest.raises(RuntimeError, match=r"means3D must have dimensions \(num_points, 3\)"):
        rasterize_gaussians_multi(torch.zeros(4, 2), m, torch.zeros(4, 16, 3), None, torch.zeros(4, 3), torch.zeros(4, 1), torch.ones(4, 3),
                                  torch.ones(4, 4), None, _settings())


def test_multi_argument_checks():
    m = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="extra_colors"):
        rasterize_gaussians_multi(m, m, torch.zeros(4, 16, 3), None, None, torch.zeros(4, 1), torch.ones(4, 3), torch.ones(4, 4), None,
                                  _settings())
