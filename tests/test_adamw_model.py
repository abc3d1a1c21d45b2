"""The AdamW model of tests/adamw_model.py against fp64 ``torch.optim.AdamW``, and the planted faults the checks must catch.

Bound: after 30 updates the model's largest parameter error against fp64 is at most 4x the error of
``torch.optim.AdamW(foreach=False)`` in fp32 on the same inputs, plus one fp32 ulp of the largest parameter.  Every planted
fault lands far outside that bound and changes the model's bits."""
import pytest
import torch

import adamw_model as A

STEPS = 30
CFG = [dict(lr=0.01, betas=(0.8, 0.95), eps=1e-3, wd=0.1), dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, wd=1e-2),
       dict(lr=0.02, betas=(0.3, 0.9), eps=1e-6, wd=0.0)]      # the last: beta1 < 0.5, the lerp's other branch


def _inputs(seed, n=4096):
    g = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * 0.1 for _ in range(STEPS)]
    for gr in grads:
        gr[:256] = 0                          # zero-gradient elements: den == eps until they see a gradient
    return p0, grads


def _model(p0, grads, c, fault=None):
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t, g in enumerate(grads, 1):
        p, m, v = A.adamw_update(g, p, m, v, c["lr"], c["betas"], c["eps"], c["wd"], t, fault)
    return p


def _torch32(p0, grads, c):
    w = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([w], lr=c["lr"], betas=c["betas"], eps=c["eps"], weight_decay=c["wd"], foreach=False)
    for g in grads:
        w.grad = g.clone()
        opt.step()
    return w.detach()


def _bound(p0, grads, c):
    ref = A.adamw_fp64(p0, grads, [c["lr"]] * len(grads), c["betas"], c["eps"], c["wd"])
    e_torch = float((_torch32(p0, grads, c).double() - ref).abs().max())
    big = ref.abs().max().float()
    ulp = float(torch.nextafter(big, torch.tensor(float("inf"))) - big)
    return ref, 4 * e_torch + ulp


@pytest.mark.parametrize("k", range(len(CFG)))
def test_model_is_within_the_bound_of_fp64(k):
    p0, grads = _inputs(k)
    ref, bound = _bound(p0, grads, CFG[k])
    err = float((_model(p0, grads, CFG[k]).double() - ref).abs().max())
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("fault", A.FAULTS)
def test_planted_faults_are_caught(fault):
    c = CFG[0]
    p0, grads = _inputs(7)
    ref, bound = _bound(p0, grads, c)
    clean, bad = _model(p0, grads, c), _model(p0, grads, c, fault)
    assert not torch.equal(clean, bad), f"{fault}: the bit-for-bit check would not see it"
    err = float((bad.double() - ref).abs().max())
    assert err > 10 * bound, f"{fault}: error {err} within 10x the bound {bound}"


def test_zero_gradient_elements_move_by_the_decay_only():
    """g = m = v = 0: den == eps exactly, m / den == 0, so p becomes p * (1 - lr*wd) and nothing else."""
    p = torch.randn(64)
    z = torch.zeros(64)
    c = CFG[1]
    q, m, v = A.adamw_update(z, p, z, z, c["lr"], c["betas"], c["eps"], c["wd"], 1)
    assert torch.equal(q, p * torch.tensor(A.f32(1 - c["lr"] * c["wd"]))) and not m.any() and not v.any()
