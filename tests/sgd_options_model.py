"""Bit-exact model of the optimizer kernels' general update (csrc/sgd_device.cuh sgd_apply_mp, csrc/sgd.cu sgd_flat_kernel):
torch.optim.SGD with dampening 0, weight decay and Nesterov momentum, one fp32 fused multiply-add per operation:

    if wd != 0:  g = fmaf(wd, p, g)
    m = fmaf(mu, m, g)
    d = fmaf(mu, m, g) if nesterov else m
    p = fmaf(-lr, d, p)

``fma32`` computes fmaf exactly for any fp32 operands (not only powers of two): the product of two fp32 values is exact in
fp64, the fp64 sum is rounded to odd (TwoSum gives its exact error), and an fp64 value rounded to odd rounds to the correct
fp32 result (53 >= 24 + 2).  The kernels are built with --use_fast_math, which flushes fp32 subnormals; the inputs here
stay clear of them.  Shared by tests/test_sgd_options.py (which checks fma32 against exact rational arithmetic) and
tests/test_gpu_sgd_options.py.
"""
from fractions import Fraction

import torch


def fma32(a, b, c) -> torch.Tensor:
    """fp32 ``a * b + c`` with one rounding (round to nearest even), elementwise; scalars broadcast."""
    ref = next((t for t in (a, b, c) if isinstance(t, torch.Tensor)), None)
    dev = ref.device if ref is not None else "cpu"
    a, b, c = (torch.as_tensor(t, dtype=torch.float32, device=dev).double() for t in (a, b, c))
    x = a * b                                   # exact: 24 + 24 significant bits
    s = x + c
    bb = s - x                                  # TwoSum: s + e == x + c exactly
    e = (x - (s - bb)) + (c - bb)
    odd = (s.view(torch.int64) & 1) == 1
    fix = (e != 0) & ~odd & torch.isfinite(s)
    s = torch.where(fix, torch.nextafter(s, torch.where(e > 0, torch.full_like(s, float("inf")),
                                                         torch.full_like(s, float("-inf")))), s)
    return s.float()


def sgd_update(g, p, m, mu: float, lr: float, wd: float, nesterov: bool):
    """(params, momentum) after one update from the averaged fp32 gradient ``g``; ``mu``, ``lr``, ``wd`` as the kernels get
    them (rounded to fp32 once)."""
    if wd != 0:
        g = fma32(wd, p, g)
    m = fma32(mu, m, g)
    d = fma32(mu, m, g) if nesterov else m
    return fma32(-lr, d, p), m


def round_f32(q: Fraction) -> float:
    """The exact rational ``q`` rounded once to fp32 (nearest, ties to even), for normal results."""
    if q == 0:
        return 0.0
    sign, q = (-1.0 if q < 0 else 1.0), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while q >= Fraction(2) ** (e + 1):
        e += 1
    while q < Fraction(2) ** e:
        e -= 1
    m = q / Fraction(2) ** (e - 23)             # in [2^23, 2^24)
    n = m.numerator // m.denominator
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return sign * float(n) * 2.0 ** (e - 23)


def torch_sgd_fp64(p0: torch.Tensor, grads: list, lrs: list, mu: float, wd: float, nesterov: bool) -> torch.Tensor:
    """``torch.optim.SGD`` in fp64 over the gradient sequence ``grads`` (one lr per step), from zero momentum."""
    p = p0.detach().double().clone().requires_grad_(False)
    w = torch.nn.Parameter(p)
    opt = torch.optim.SGD([w], lr=lrs[0], momentum=mu, weight_decay=wd, nesterov=nesterov, foreach=False)
    for g, lr in zip(grads, lrs):
        for grp in opt.param_groups:
            grp["lr"] = lr
        w.grad = g.double().to(w.device)
        opt.step()
    return w.detach()
