"""The CUDA Adam step's host side, on the CPU: the exports, gsr_adam_tensor's ctypes mirror against include/gsr_b200.h (compiled
with the system C compiler), the per-tensor scalars against the ones torch's own foreach Adam passes to its list ops, and every
ValueError and RuntimeError of autovfx_b200.optim."""
import ctypes as C
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from autovfx_b200 import _lib, optim  # noqa: E402

FIELDS = ("param", "grad", "exp_avg", "exp_avg_sq", "numel", "lerp_weight", "beta2", "one_minus_beta2", "bias_correction2_sqrt", "eps",
          "step_size")
# the 3DGS trainer's learning rates (arguments/__init__.py, spatial_lr_scale about 5) and SuGaR's, with their eps
LRS = (0.0, 0.00016 * 5.0, 0.0025, 0.0025 / 20.0, 0.05, 0.005, 0.001, 1.6e-6)


def test_library_exports_the_adam_entry_point():
    assert "gsr_adam_step" in _lib.EXPORTS and hasattr(_lib.lib, "gsr_adam_step")
    assert set(optim.__all__) == {"Adam", "use_cuda_adam", "host_scalars"}
    assert issubclass(optim.Adam, torch.optim.Adam)


def test_adam_tensor_struct_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to read the header's layout")
    src = tmp_path / "layout.c"
    body = "".join('    printf("%%s %%zu\\n", "%s", offsetof(gsr_adam_tensor, %s));\n' % (f, f) for f in FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsr_b200.h"\nint main(void) {\n' + body +
                   '    printf("sizeof %zu\\nmax %d\\n", sizeof(gsr_adam_tensor), GSR_ADAM_MAX_TENSORS);\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for f in FIELDS:
        assert int(got[f]) == getattr(_lib.gsr_adam_tensor, f).offset, f
    assert int(got["sizeof"]) == C.sizeof(_lib.gsr_adam_tensor) == 64
    assert int(got["max"]) == _lib.GSR_ADAM_MAX_TENSORS
    assert _lib.lib.gsr_adam_step.argtypes == [C.c_int32, C.POINTER(_lib.gsr_adam_tensor), C.c_void_p]


def _f32_bits(x):
    return int(np.array(x, dtype=np.float32).view(np.int32))


@pytest.mark.parametrize("step", [1, 2, 1000, 15000])
def test_host_scalars_equal_torch_foreach_arguments(monkeypatch, step):
    """Run torch's own foreach Adam (on CPU tensors) from step count `step - 1`, record the scalars it hands to each list op, and
    compare them, rounded to float as the CUDA foreach kernels round them, with host_scalars() through the ctypes descriptor."""
    seen = {}

    def spy(name, pos):
        real = getattr(torch, name)

        def f(*args, **kw):
            seen.setdefault(name, []).append(args[pos] if len(args) > pos else kw)
            return real(*args, **kw)
        monkeypatch.setattr(torch, name, f)
    for name, pos in (("_foreach_lerp_", 2), ("_foreach_mul_", 1), ("_foreach_addcmul_", 3), ("_foreach_div_", 1),
                      ("_foreach_add_", 1), ("_foreach_addcdiv_", 3)):
        spy(name, pos)
    ps = [torch.nn.Parameter(torch.randn(5)) for _ in LRS]
    opt = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(ps, LRS)], lr=0.0, eps=1e-15, foreach=True)
    for p in ps:
        p.grad = torch.randn(5)
        opt.state[p] = {"step": torch.tensor(float(step - 1)), "exp_avg": torch.zeros(5), "exp_avg_sq": torch.zeros(5)}
    opt.step()
    assert [float(opt.state[p]["step"]) for p in ps] == [float(step)] * len(ps)
    for k, (p, lr) in enumerate(zip(ps, LRS)):
        d = _lib.gsr_adam_tensor()
        (d.lerp_weight, d.beta2, d.one_minus_beta2, d.bias_correction2_sqrt, d.eps,
         d.step_size) = optim.host_scalars(0.9, 0.999, lr, 1e-15, float(opt.state[p]["step"]))
        want = {"lerp_weight": seen["_foreach_lerp_"][k], "beta2": seen["_foreach_mul_"][k], "one_minus_beta2": seen["_foreach_addcmul_"][k],
                "bias_correction2_sqrt": seen["_foreach_div_"][k][0], "eps": seen["_foreach_add_"][-1],
                "step_size": seen["_foreach_addcdiv_"][k][0]}
        for f, v in want.items():
            assert _f32_bits(getattr(d, f)) == _f32_bits(v), (step, lr, f, getattr(d, f), v)


def _opt(**kw):
    p = torch.nn.Parameter(torch.zeros(8))
    return torch.optim.Adam([{"params": [p], "name": "xyz"}], lr=0.0, eps=1e-15, **kw), p


@pytest.mark.parametrize("option,kw", [("amsgrad", {"amsgrad": True}), ("weight_decay", {"weight_decay": 1e-4}),
                                       ("maximize", {"maximize": True}), ("capturable", {"capturable": True}),
                                       ("differentiable", {"differentiable": True}), ("fused=True", {"fused": True}),
                                       ("foreach=False", {"foreach": False})])
def test_unsupported_options_raise_at_switch_and_step_time(option, kw):
    opt, p = _opt(**kw)
    with pytest.raises(ValueError, match=option):
        optim.use_cuda_adam(opt)
    opt2, p2 = _opt()
    opt2.__class__ = optim.Adam            # switched while the option was off, then turned on
    opt2.param_groups[0].update(kw)
    p2.grad = torch.zeros(8)
    with pytest.raises(ValueError, match=option):
        opt2.step()


def test_tensor_lr_and_betas_raise():
    opt, _ = _opt()
    opt.param_groups[0]["lr"] = torch.tensor(0.01)
    with pytest.raises(ValueError, match="Tensor lr"):
        optim.use_cuda_adam(opt)
    opt, _ = _opt()
    opt.param_groups[0]["betas"] = (torch.tensor(0.9), torch.tensor(0.999))
    with pytest.raises(ValueError, match="Tensor betas"):
        optim.use_cuda_adam(opt)


def test_other_optimizers_raise():
    p = torch.nn.Parameter(torch.zeros(4))
    for o in (torch.optim.AdamW([p], weight_decay=0.0), torch.optim.SGD([p], lr=0.1)):
        with pytest.raises(ValueError, match="torch.optim.Adam"):
            optim.use_cuda_adam(o)


def test_cpu_tensors_raise_runtime_error():
    opt, p = _opt()
    with pytest.raises(RuntimeError, match="CUDA"):
        optim.use_cuda_adam(opt)
    with pytest.raises(RuntimeError, match="CUDA"):
        optim.Adam([p], lr=0.0, eps=1e-15)
    opt.__class__ = optim.Adam
    p.grad = torch.zeros(8)
    with pytest.raises(RuntimeError, match="CUDA"):
        opt.step()
    assert len(opt.state) == 0  # refused before any state was created


def _switched(p, **state):
    opt = torch.optim.Adam([{"params": [p], "name": "xyz"}], lr=0.0, eps=1e-15)
    opt.__class__ = optim.Adam
    if state:
        opt.state[p] = state
    return opt


def test_bad_tensors_raise_value_error():
    # non-float32 parameter (switch time and step time) and gradient
    p64 = torch.nn.Parameter(torch.zeros(8, dtype=torch.float64))
    with pytest.raises(ValueError, match="float32"):
        optim.use_cuda_adam(torch.optim.Adam([p64]))
    p64.grad = torch.zeros(8, dtype=torch.float64)
    with pytest.raises(ValueError, match="float32"):
        _switched(p64).step()
    p = torch.nn.Parameter(torch.zeros(8))
    p.grad = torch.zeros(8, dtype=torch.float64).float()
    # non-float32 and non-contiguous moments
    for bad, match in ((torch.zeros(8, dtype=torch.float64), "float32"), (torch.zeros(16)[::2], "contiguous")):
        opt = _switched(p, step=torch.tensor(3.0), exp_avg=bad, exp_avg_sq=torch.zeros(8))
        with pytest.raises(ValueError, match=match):
            opt.step()
        assert float(opt.state[p]["step"]) == 3.0
    # a moment of the wrong shape, a step count on a device
    with pytest.raises(ValueError, match="shape"):
        _switched(p, step=torch.tensor(3.0), exp_avg=torch.zeros(9), exp_avg_sq=torch.zeros(8)).step()
    with pytest.raises(ValueError, match="step count"):
        _switched(p, step=torch.tensor(3.0, device="meta"), exp_avg=torch.zeros(8), exp_avg_sq=torch.zeros(8)).step()
    # non-contiguous parameter and gradient
    pt = torch.nn.Parameter(torch.zeros(4, 2).t())
    with pytest.raises(ValueError, match="contiguous"):
        optim.use_cuda_adam(torch.optim.Adam([pt]))
    q = torch.nn.Parameter(torch.zeros(2, 4))
    q.grad = torch.zeros(4, 2).t()
    with pytest.raises(ValueError, match="contiguous"):
        _switched(q).step()
    # sparse gradient
    s = torch.nn.Parameter(torch.zeros(8))
    s.grad = torch.zeros(8).to_sparse()
    with pytest.raises(ValueError, match="sparse"):
        _switched(s).step()


def test_tensors_on_different_devices_raise_value_error():
    a, b = torch.nn.Parameter(torch.zeros(8)), torch.nn.Parameter(torch.zeros(8, device="meta"))
    opt = torch.optim.Adam([{"params": [a]}, {"params": [b]}], lr=0.0)
    with pytest.raises(ValueError, match="other tensors on"):
        optim.use_cuda_adam(opt)
    a.grad, b.grad = torch.zeros(8), torch.zeros(8, device="meta")
    opt.__class__ = optim.Adam
    with pytest.raises(ValueError, match="other tensors on"):
        opt.step()


def test_step_without_gradients_is_a_no_op():
    opt, p = _opt()
    opt.__class__ = optim.Adam
    assert opt.step(closure=lambda: 7.0) == 7.0
    assert len(opt.state) == 0
