"""capturable=True without a GPU: the model of the scalar block against the host's fp64 ``adamw_scalars`` and an exact
emulation of its roundings, planted faults in the model, and the constructor's refusals."""
import math
from fractions import Fraction

import pytest
import torch
import torch.nn as nn

import capturable_model as CM
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatLAMB, FlatLARS, FlatSGD, LRSchedule, adamw_scalars

BETAS = [(0.9, 0.999), (0.8, 0.95), (0.95, 0.9999), (0.0, 0.99)]
T_MAX = 10 ** 5


def _rn_pow(b: float, t: int) -> float:
    """Exponentiation by squaring in exact rationals, every product rounded once to the nearest double."""
    r, x = Fraction(1), Fraction(b)
    while t:
        if t & 1:
            r = Fraction(float(r * x))
        x = Fraction(float(x * x))
        t >>= 1
    return float(r)


def _check(betas, lr_of, wd, model=CM.block):
    """Compare the model with adamw_scalars (rounded to fp32) for t = 1..T_MAX; returns (worst ulps, steps that differ)."""
    worst, differ = 0, 0
    for s in range(T_MAX):
        lr = lr_of(s)
        got = model(lr, wd, betas, 1e-8, s)["adamw"]
        want = [CM.f32(x) for x in adamw_scalars(lr, betas, 1e-8, wd, s + 1)]
        d = max(CM.ulps(a, b) for a, b in zip(got, want))
        if got[0] != want[0]:                  # 1 - lr*wd is the host's own operation sequence: exact
            d = max(d, 10 ** 6)
        worst, differ = max(worst, d), differ + (d > 0)
    return worst, differ


SCHED = LRSchedule(warmup_steps=T_MAX // 2, warmup_start=0.01)


@pytest.mark.parametrize("betas", BETAS, ids=str)
def test_model_within_one_ulp_of_adamw_scalars(betas):
    worst, differ = _check(betas, lambda s: SCHED.lr_at(1.0, s), 0.1)
    print(f"betas {betas}: {differ} of {T_MAX} steps differ from adamw_scalars by at most {worst} ulp")
    assert worst <= 1


@pytest.mark.parametrize("betas", BETAS[:2], ids=str)
def test_model_squaring_is_the_rounded_sequence(betas):
    """flat_pow is the device's rounding sequence exactly, and differs from Python's ``**`` for some t (so the model
    really is the squaring order, not pow)."""
    ts = list(range(1, 200)) + list(range(200, T_MAX, 997)) + [2 ** 40 + 3]
    pow_differs = 0
    for b in betas:
        for t in ts:
            assert CM.flat_pow(b, t) == _rn_pow(b, t), (b, t)
            pow_differs += CM.flat_pow(b, t) != b ** t
    assert pow_differs > 0


def test_planted_faults_are_caught():
    lr_of = lambda s: SCHED.lr_at(1.0, s)      # noqa: E731
    # update t taken as the counter itself (off by one)
    off = lambda lr, wd, betas, eps, s: CM.block(lr, wd, betas, eps, s - 1 if s else 0)   # noqa: E731
    assert _check((0.9, 0.999), lr_of, 0.1, off)[0] > 1
    # weight decay rounded to fp32 before 1 - lr*wd
    f32wd = lambda lr, wd, betas, eps, s: CM.block(lr, CM.f32(wd), betas, eps, s)          # noqa: E731
    assert _check((0.9, 0.999), lr_of, 0.1, f32wd)[1] > 0
    # pow instead of the squaring order: with beta2 = 1 - 1e-8 a block computed with pow differs from the model in some fp32
    # field at some counters (tests/test_gpu_capturable.py holds the device to the model at exactly those), and the model's
    # squaring is the exact emulation of the device's roundings there
    betas = (0.9, 0.99999999)
    LR32 = CM.f32(1e-3)
    differ = [s for s in range(2000)
              if CM.block(LR32, 0.0, betas, 1e-8, s, pow_fn=pow)["adamw"] != CM.block(LR32, 0.0, betas, 1e-8, s)["adamw"]]
    print(f"pow instead of squaring: {len(differ)} of 2000 blocks differ")
    assert differ
    assert all(CM.flat_pow(b, s + 1) == _rn_pow(b, s + 1) for b in betas for s in differ)


def test_capturable_refusals_without_a_gpu():
    net = nn.Sequential(nn.Linear(4, 4))
    with pytest.raises(ValueError, match="capturable"):
        FlatSGD(net, capturable=True)
    with pytest.raises(ValueError, match="capturable"):
        FlatAdamW(nn.Sequential(nn.Linear(4, 4)), capturable=True)
    for cls in (FlatLAMB, FlatLARS):
        with pytest.raises(TypeError):
            cls(nn.Sequential(nn.Linear(4, 4)), capturable=True)


def test_default_is_not_capturable():
    opt = FlatSGD(nn.Sequential(nn.Linear(4, 4)))
    assert opt.capturable is False and opt.steps == 0
    opt.step()
    assert opt.steps == 1
