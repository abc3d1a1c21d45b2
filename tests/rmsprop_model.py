"""Rounding-exact model of the RMSprop update of the kernels (csrc/rmsprop_device.cuh ``rmsprop_elem``, used by
``rmsprop_flat_kernel`` and the RMSprop instances of ``sharded_step_kernel``), shared by the CPU test of the model
(tests/test_rmsprop_model.py) and the GPU tests (tests/test_gpu_rmsprop.py).

One update, the scalars computed in fp64 and rounded once to fp32 (c = 1 - alpha):

    g   = fmaf(wd, p, g)                                  only when wd != 0
    sq  = fmaf(c * g, g, sq * alpha)
    centered:  d = g - ga;  ga = fmaf(c, d, ga) if |c| < 0.5 else fmaf(-d, 1 - c, g)
               avg = sqrt(fmaf(-ga, ga, sq)) + eps
    else:      avg = sqrt(sq) + eps
    momentum:  buf = buf * mu + g / avg;  p = fmaf(-lr, buf, p)
    else:      p = fmaf(-lr, g / avg, p)

Every fp32 ``*``, ``-``, ``/`` and ``+`` below is one torch fp32 CPU operation on tensors, which rounds once to nearest;
``sqrt32`` is the correctly rounded fp32 root and ``fma32`` rounds the fused multiply-add once (tests/adamw_model.py,
tests/sgd_options_model.py).  ``fault`` plants one defect a kernel could have; tests/test_rmsprop_model.py shows that the
checks catch each.
"""
import torch

from adamw_model import f32, sqrt32
from sgd_options_model import fma32

FAULTS = ("eps_inside_sqrt", "swapped_alpha", "centered_without_ga_squared", "decoupled_weight_decay",
          "momentum_before_buffer_update", "lr_on_g_not_buf")


def scalars64(lr: float, alpha: float, eps: float, wd: float, momentum: float) -> list:
    """[lr, weight_decay, alpha, 1 - alpha, eps, momentum] in fp64, as ops/optim.py rmsprop_scalars gives them."""
    return [lr, wd, alpha, 1.0 - alpha, eps, momentum]


def rmsprop_update(g, p, sq, ga, buf, lr: float, alpha: float, eps: float, wd: float, momentum: float, centered: bool,
                   fault: str = None):
    """(p, sq, ga, buf) after one update from the fp32 gradient ``g`` (already averaged, and clipped if it is); ``ga`` /
    ``buf`` are passed through unchanged (may be None) when the update is not centered / has no momentum."""
    assert fault in (None,) + FAULTS
    g, p, sq = (x.float().cpu() for x in (g, p, sq))
    ga = ga.float().cpu() if ga is not None else None
    buf = buf.float().cpu() if buf is not None else None
    if fault == "swapped_alpha":
        alpha = 1.0 - alpha
    full = lambda x: torch.full_like(g, f32(x))                   # noqa: E731 - a scalar as a full-size fp32 operand
    lr_, wd_, a_, c_, eps_, mu_ = (full(x) for x in scalars64(lr, alpha, eps, wd, momentum))
    if wd != 0.0:
        if fault == "decoupled_weight_decay":
            p = p * (1.0 - full(lr * wd))
        else:
            g = fma32(wd_, p, g)
    sq = fma32(c_ * g, g, sq * a_)
    inner = sq
    if centered:
        d = g - ga
        ga = fma32(c_, d, ga) if abs(float(c_[0])) < 0.5 else fma32(-d, 1.0 - c_, g)
        if fault != "centered_without_ga_squared":
            inner = fma32(-ga, ga, sq)
    avg = sqrt32(inner + eps_) if fault == "eps_inside_sqrt" else sqrt32(inner) + eps_
    if momentum > 0:
        if fault == "momentum_before_buffer_update":
            p = fma32(-lr_, buf, p)
            buf = buf * mu_ + g / avg
        elif fault == "lr_on_g_not_buf":
            buf = buf * mu_ + g / avg
            p = fma32(-lr_, g / avg, p)
        else:
            buf = buf * mu_ + g / avg
            p = fma32(-lr_, buf, p)
    else:
        p = fma32(-lr_, g / avg, p)
    return p, sq, ga, buf


def rmsprop_fp64(p0, grads: list, lrs: list, alpha: float, eps: float, wd: float, momentum: float, centered: bool):
    """``torch.optim.RMSprop`` in fp64 over the gradient sequence ``grads`` (one lr per update)."""
    w = torch.nn.Parameter(p0.detach().double().cpu().clone())
    opt = torch.optim.RMSprop([w], lr=lrs[0], alpha=alpha, eps=eps, weight_decay=wd, momentum=momentum, centered=centered,
                              foreach=False)
    for g, lr in zip(grads, lrs):
        opt.param_groups[0]["lr"] = lr
        w.grad = g.detach().double().cpu()
        opt.step()
    return w.detach()
