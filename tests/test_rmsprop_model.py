"""The RMSprop model of tests/rmsprop_model.py against fp64 ``torch.optim.RMSprop``, and the planted faults the checks must
catch.

Bound: after 30 updates the model's largest parameter error against fp64 is at most 4x the error of
``torch.optim.RMSprop(foreach=False)`` in fp32 on the same inputs, plus one fp32 ulp of the largest parameter.  It is checked
for every momentum x centered combination, with and without weight decay.  Every planted fault lands far outside that bound
and changes the model's bits."""
import itertools

import pytest
import torch

import rmsprop_model as R

STEPS = 30
# (momentum, centered) x weight decay; alpha 0.9 / eps 0.0316 is torchvision's recipe, alpha 0.3 the lerp's other branch
OPTIONS = list(itertools.product((0.0, 0.9), (False, True), (0.0, 0.05)))
HP = [dict(lr=0.01, alpha=0.99, eps=1e-8), dict(lr=0.003, alpha=0.9, eps=0.0316), dict(lr=0.002, alpha=0.3, eps=1e-6)]


def _inputs(seed, n=4096):
    g = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * 0.1 + 0.02 for _ in range(STEPS)]
    for gr in grads:
        gr[:256] = 0                          # zero-gradient elements: avg == eps, g / avg == 0 (without decay)
    return p0, grads


def _model(p0, grads, c, fault=None):
    p, sq = p0.clone(), torch.zeros_like(p0)
    ga = torch.zeros_like(p0) if c["centered"] else None
    buf = torch.zeros_like(p0) if c["momentum"] > 0 else None
    for g in grads:
        p, sq, ga, buf = R.rmsprop_update(g, p, sq, ga, buf, c["lr"], c["alpha"], c["eps"], c["wd"], c["momentum"],
                                          c["centered"], fault)
    return p


def _torch32(p0, grads, c):
    w = torch.nn.Parameter(p0.clone())
    opt = torch.optim.RMSprop([w], lr=c["lr"], alpha=c["alpha"], eps=c["eps"], weight_decay=c["wd"], momentum=c["momentum"],
                              centered=c["centered"], foreach=False)
    for g in grads:
        w.grad = g.clone()
        opt.step()
    return w.detach()


def _bound(p0, grads, c):
    ref = R.rmsprop_fp64(p0, grads, [c["lr"]] * len(grads), c["alpha"], c["eps"], c["wd"], c["momentum"], c["centered"])
    e_torch = float((_torch32(p0, grads, c).double() - ref).abs().max())
    big = ref.abs().max().float()
    ulp = float(torch.nextafter(big, torch.tensor(float("inf"))) - big)
    return ref, 4 * e_torch + ulp


@pytest.mark.parametrize("h", range(len(HP)))
@pytest.mark.parametrize("momentum,centered,wd", OPTIONS)
def test_model_is_within_the_bound_of_fp64(momentum, centered, wd, h):
    c = dict(HP[h], momentum=momentum, centered=centered, wd=wd)
    p0, grads = _inputs(h)
    ref, bound = _bound(p0, grads, c)
    err = float((_model(p0, grads, c).double() - ref).abs().max())
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("fault", R.FAULTS)
def test_planted_faults_are_caught(fault):
    c = dict(HP[0], momentum=0.9, centered=True, wd=0.05)
    p0, grads = _inputs(7)
    ref, bound = _bound(p0, grads, c)
    clean, bad = _model(p0, grads, c), _model(p0, grads, c, fault)
    assert not torch.equal(clean, bad), f"{fault}: the bit-for-bit check would not see it"
    err = float((bad.double() - ref).abs().max())
    assert err > 10 * bound, f"{fault}: error {err} within 10x the bound {bound}"


def test_zero_gradient_elements_do_not_move_without_decay():
    """g = sq = 0: avg == eps exactly and g / avg == 0, so p, sq and the momentum buffer stay as they are."""
    p = torch.randn(64)
    z = torch.zeros(64)
    q, sq, ga, buf = R.rmsprop_update(z, p, z, z, z, 0.01, 0.99, 1e-8, 0.0, 0.9, True)
    assert torch.equal(q, p) and not sq.any() and not ga.any() and not buf.any()
