"""The trainers' optimizer step in CUDA: ``torch.optim.Adam.step()`` of 3DGS's ``GaussianModel`` ("GS/" =
sugar/gaussian_splatting/scene/gaussian_model.py:164-173, stepped at GS/train.py:183-184 and scene_representation.py:538-540) and of
SuGaR's ``SuGaROptimizer`` (sugar/sugar_scene/sugar_optimizer.py:68-85, stepped at sugar_trainers/coarse_density.py:822), through
``gsr_adam_step``: one launch over every parameter and both moments, bit-identical to torch's default (foreach) Adam.

Opt in with one line after the optimizer exists::

    from autovfx_b200.optim import use_cuda_adam
    gaussians.training_setup(opt)
    use_cuda_adam(gaussians.optimizer)          # GaussianModel
    optimizer = SuGaROptimizer(sugar, opt_params, spatial_lr_scale=spatial_lr_scale)
    use_cuda_adam(optimizer.optimizer)          # SuGaROptimizer

The optimizer object stays the same (its class becomes :class:`Adam`), so every reference to it, its param groups, its state,
``state_dict()``/``load_state_dict()`` and the library's ``densify_and_prune`` keep working unchanged.
"""
from __future__ import annotations

import torch
from torch.optim.optimizer import _get_scalar_dtype, _get_value

from . import _lib

__all__ = ["Adam", "use_cuda_adam", "host_scalars"]


def host_scalars(beta1, beta2, lr, eps, step):
    """The per-tensor scalars of one step, with torch's own Python expressions in double (torch/optim/adam.py:_multi_tensor_adam,
    capturable=False): (lerp weight, beta2, 1 - beta2, bias_correction2_sqrt, eps, step_size) for the step count after the
    increment.  gsr_adam_step receives each rounded to float, as the foreach kernels do."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = (lr / bias_correction1) * -1
    bias_correction2_sqrt = bias_correction2 ** 0.5
    return 1 - beta1, beta2, 1 - beta2, bias_correction2_sqrt, eps, step_size


def _check_group(who, group):
    """ValueError naming the first option of a param group that the one kernel does not reproduce."""
    bad = [name for name, on in (("amsgrad", group.get("amsgrad", False)), ("weight_decay != 0", group.get("weight_decay", 0) != 0),
                                 ("maximize", group.get("maximize", False)), ("capturable", group.get("capturable", False)),
                                 ("differentiable", group.get("differentiable", False)), ("fused=True", bool(group.get("fused"))),
                                 ("foreach=False", group.get("foreach") is False),
                                 ("a Tensor lr", isinstance(group.get("lr"), torch.Tensor)),
                                 ("Tensor betas", any(isinstance(b, torch.Tensor) for b in group.get("betas", ()))))
           if on]
    if bad:
        raise ValueError("%s: param group %r uses %s, which the CUDA Adam step does not reproduce (it is torch's default foreach "
                         "Adam only)" % (who, group.get("name"), bad[0]))


def _check_tensor(who, what, t, dev):
    """ValueError for a tensor the kernel cannot take; the CUDA check comes after every such check (_require_cuda)."""
    if t.dtype != torch.float32:
        raise ValueError("%s: %s must be float32, got %s" % (who, what, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s: %s must be contiguous" % (who, what))
    if t.device != dev:
        raise ValueError("%s: %s is on %s, other tensors on %s" % (who, what, t.device, dev))


def _require_cuda(who, tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("autovfx_b200.%s: every tensor must be a CUDA tensor, got one on %s (there is no CPU path)"
                               % (who, t.device))


def _check_params(who, optimizer):
    dev, seen = None, []
    for group in optimizer.param_groups:
        _check_group(who, group)
        for i, p in enumerate(group["params"]):
            dev = p.device if dev is None else dev
            _check_tensor(who, "parameter %d of param group %r" % (i, group.get("name")), p, dev)
            seen.append(p)
    _require_cuda(who, seen)


class Adam(torch.optim.Adam):
    """``torch.optim.Adam`` whose ``step()`` runs ``gsr_adam_step``: one CUDA launch over every parameter with a gradient and
    both moments, bit-identical to torch's default (foreach) step.  Construction, ``param_groups``, ``state``, ``state_dict()``
    and ``load_state_dict()`` are torch's.

    ``step()`` keeps torch's semantics: a parameter whose ``.grad`` is None is skipped and its ``step`` count does not move; state is
    created lazily as torch creates it (``step`` a CPU scalar tensor, zero moments like the parameter); ``group['lr']`` is read on
    every step; the step counts stay on the CPU and nothing synchronises with the device.

    Raises ValueError, naming it, for what the kernel does not reproduce: amsgrad, weight_decay != 0, maximize, capturable,
    differentiable, fused=True, foreach=False, a Tensor lr or betas; non-float32 or non-contiguous parameters, gradients or
    moments, sparse gradients, tensors on different devices, a ``step`` count that is not a CPU tensor.  CPU tensors raise
    RuntimeError (there is no CPU path)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        _check_params("Adam", self)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        who = "Adam.step"
        work, seen, dev = [], [], None
        # every check before anything changes: a refused step leaves parameters, moments and counts as they were
        for group in self.param_groups:
            _check_group(who, group)
            for i, p in enumerate(group["params"]):
                g = p.grad
                if g is None:
                    continue
                what = "param group %r, parameter %d" % (group.get("name"), i)
                if g.is_sparse:
                    raise ValueError("%s: %s has a sparse gradient" % (who, what))
                dev = p.device if dev is None else dev
                _check_tensor(who, what, p, dev)
                _check_tensor(who, "the gradient of " + what, g, dev)
                seen += [p, g]
                if g.shape != p.shape:
                    raise ValueError("%s: the gradient of %s has shape %s, the parameter %s" % (who, what, tuple(g.shape), tuple(p.shape)))
                state = self.state.get(p)
                if state:
                    for k in ("exp_avg", "exp_avg_sq"):
                        _check_tensor(who, "%s of %s" % (k, what), state[k], dev)
                        seen.append(state[k])
                        if state[k].shape != p.shape:
                            raise ValueError("%s: %s of %s has shape %s, the parameter %s" % (who, k, what, tuple(state[k].shape),
                                                                                             tuple(p.shape)))
                    s = state["step"]
                    if not torch.is_tensor(s) or s.device.type != "cpu" or s.numel() != 1:
                        raise ValueError("%s: the step count of %s must be a CPU scalar tensor (a device count needs capturable)"
                                         % (who, what))
                work.append((group, p, g))
        _require_cuda(who, seen)
        if not work:
            return loss
        for group, p, g in work:
            state = self.state[p]
            if len(state) == 0:  # lazy state, as torch.optim.Adam._init_group creates it
                state["step"] = torch.tensor(0.0, dtype=_get_scalar_dtype())
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        steps = [self.state[p]["step"] for _, p, _ in work]
        torch._foreach_add_(steps, torch.tensor(1.0, device="cpu"), alpha=1.0)
        descs = (_lib.gsr_adam_tensor * len(work))()
        for d, (group, p, g), step in zip(descs, work, steps):
            state = self.state[p]
            beta1, beta2 = group["betas"]
            w, b2, c, bc2, eps, a = host_scalars(beta1, beta2, group["lr"], group["eps"], _get_value(step))
            d.param, d.grad, d.exp_avg, d.exp_avg_sq = p.data_ptr(), g.data_ptr(), state["exp_avg"].data_ptr(), state["exp_avg_sq"].data_ptr()
            d.numel = p.numel()
            d.lerp_weight, d.beta2, d.one_minus_beta2, d.bias_correction2_sqrt, d.eps, d.step_size = w, b2, c, bc2, eps, a
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gsr_adam_step(len(work), descs, _lib.stream_ptr(dev)), "gsr_adam_step")
        return loss


def use_cuda_adam(optimizer):
    """Switch an existing ``torch.optim.Adam`` to :class:`Adam` in place and return it: the same object, param groups and state,
    so ``GaussianModel.optimizer``, ``SuGaROptimizer.optimizer`` and the densifier's reference to it keep working.  Raises
    ValueError for another optimizer class or an option the kernel does not reproduce, RuntimeError for CPU parameters."""
    if type(optimizer) not in (torch.optim.Adam, Adam):
        raise ValueError("use_cuda_adam: expected a torch.optim.Adam, got %s" % type(optimizer).__name__)
    _check_params("use_cuda_adam", optimizer)
    optimizer.__class__ = Adam
    optimizer._patch_step_function()  # step pre/post hooks and the profiler's step record, as torch's constructor sets them up
    return optimizer
