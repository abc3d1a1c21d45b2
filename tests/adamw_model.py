"""Rounding-exact model of the AdamW update of the kernels (csrc/adamw_device.cuh ``adamw_elem``, used by
``adamw_flat_kernel`` and the AdamW instance of ``sharded_step_kernel``), shared by the CPU test of the model
(tests/test_adamw_model.py) and the GPU tests (tests/test_gpu_adamw.py).

Update t (1-based), the scalars computed in fp64 and rounded once to fp32 (``scalars32``):

    p   = p * (1 - lr*wd)
    d   = g - m;   m = fmaf(w1, d, m) if w1 < 0.5 else fmaf(-d, 1 - w1, g)        w1 = 1 - beta1
    v   = fmaf((1 - beta2) * g, g, v * beta2)
    den = sqrt(v) / sqrt(1 - beta2^t) + eps
    p   = fmaf(-(lr / (1 - beta1^t)), m / den, p)

Every fp32 ``*``, ``-``, ``/`` and ``+`` below is one torch fp32 CPU operation on tensors, which rounds once to nearest;
``sqrt32`` takes the root in fp64 and rounds it to fp32, which is the correctly rounded fp32 root (torch's vectorised fp32
CPU ``sqrt`` is not always); ``fma32`` (tests/sgd_options_model.py) rounds the fused multiply-add once.  ``fault`` plants one defect a kernel
could have; tests/test_adamw_model.py shows that the checks catch each.
"""
import math
import struct

import torch

from sgd_options_model import fma32

FAULTS = ("bias_correction_off_by_one", "eps_inside_sqrt", "coupled_weight_decay", "swapped_betas", "missing_sqrt_bc2",
          "decay_after_step")


def f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


def scalars64(lr: float, betas: tuple, eps: float, wd: float, t: int) -> list:
    """[1 - lr*wd, 1 - beta1, beta2, 1 - beta2, lr / bc1, sqrt(bc2), eps] of update t, in fp64."""
    b1, b2 = betas
    return [1.0 - lr * wd, 1.0 - b1, b2, 1.0 - b2, lr / (1.0 - b1 ** t), (1.0 - b2 ** t) ** 0.5, eps]


def _t(x: float) -> torch.Tensor:
    return torch.tensor(f32(x), dtype=torch.float32)


def sqrt32(x: torch.Tensor) -> torch.Tensor:
    """The correctly rounded fp32 square root (__fsqrt_rn): fp64 root, rounded once (53 >= 2 * 24 + 2)."""
    return torch.sqrt(x.double()).float()


def adamw_update(g, p, m, v, lr: float, betas: tuple, eps: float, wd: float, t: int, fault: str = None):
    """(p, m, v) after update ``t`` from the fp32 gradient ``g`` (already averaged, and clipped if it is)."""
    assert fault in (None,) + FAULTS
    g, p, m, v = (x.float().cpu() for x in (g, p, m, v))
    if fault == "swapped_betas":
        betas = betas[::-1]
    tb = t + 1 if fault == "bias_correction_off_by_one" else t
    # the scalars as full-size fp32 operands, each rounded once from fp64 as the binding rounds them
    decay, w1, b2, c2, step, sbc2, e = (torch.full_like(g, f32(x)) for x in scalars64(lr, betas, eps, wd, tb))
    if fault == "coupled_weight_decay":
        g = fma32(_t(wd), p, g)
    elif fault != "decay_after_step":
        p = p * decay
    d = g - m
    m = fma32(w1, d, m) if float(w1[0]) < 0.5 else fma32(-d, 1.0 - w1, g)
    v = fma32(c2 * g, g, v * b2)
    if fault == "eps_inside_sqrt":
        den = sqrt32(v + e) / sbc2
    elif fault == "missing_sqrt_bc2":
        den = sqrt32(v) + e
    else:
        den = sqrt32(v) / sbc2 + e
    p = fma32(-step, m / den, p)
    if fault == "decay_after_step":
        p = p * decay
    return p, m, v


def clip_coef(sqnorms, c: float) -> float:
    """The clip instance's coefficient from grad_sqnorm's fp64 per-bucket sums: the norm sqrt(sum) in fp64 rounded once to
    fp32, then min((1 / (n + 1e-6)) * c, 1) in fp32 (tests/grad_clip_model.py ``coef32``)."""
    from grad_clip_model import coef32

    s = 0.0
    for q in sqnorms:
        s += float(q)
    return float(coef32(f32(math.sqrt(s)), c))


def adamw_fp64(p0, grads: list, lrs: list, betas: tuple, eps: float, wd: float) -> torch.Tensor:
    """``torch.optim.AdamW`` in fp64 over the gradient sequence ``grads`` (one lr per update)."""
    w = torch.nn.Parameter(p0.detach().double().cpu().clone())
    opt = torch.optim.AdamW([w], lr=lrs[0], betas=betas, eps=eps, weight_decay=wd, foreach=False)
    for g, lr in zip(grads, lrs):
        opt.param_groups[0]["lr"] = lr
        w.grad = g.detach().double().cpu()
        opt.step()
    return w.detach()
