"""The grouped model (tests/param_groups_model.py) is the ungrouped model run on each tensor's segment with its group's
scalars, bit for bit, and every planted fault changes the result."""
import pytest
import torch

import param_groups_model as G
from adamw_model import adamw_update
from sgd_options_model import sgd_update

BETAS, EPS, MU = (0.9, 0.999), 1e-8, 0.9
# tensors of 6, 1, 9, 4 and 13 elements laid out at multiples of 4, in groups 0, 1, 1, 2, 0 (group 1: no decay)
SIZES, GIDS = [6, 1, 9, 4, 13], [0, 1, 1, 2, 0]
LRS, WDS = [0.01, 0.003, 0.05], [0.1, 0.0, 0.02]


def _layout():
    offs, n = [], 0
    for s in SIZES:
        offs.append(n)
        n += (s + 3) // 4 * 4
    gmap = torch.tensor([GIDS[max(i for i, o in enumerate(offs) if o <= 4 * v)] for v in range(n // 4)], dtype=torch.uint8)
    return offs, n, gmap


def _state(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for _ in range(3)] + [torch.rand(n, generator=g)]


def _segments(offs, n):
    return [(o, offs[i + 1] if i + 1 < len(offs) else n, GIDS[i]) for i, o in enumerate(offs)]


@pytest.mark.parametrize("nesterov", [False, True])
def test_grouped_sgd_is_the_ungrouped_model_per_segment(nesterov):
    offs, n, gmap = _layout()
    g, p, m, _ = _state(n)
    gp, gm = G.grouped_sgd(g, p, m, gmap, LRS, WDS, MU, nesterov)
    for lo, hi, gi in _segments(offs, n):
        rp, rm = sgd_update(g[lo:hi], p[lo:hi], m[lo:hi], G.f32(MU), G.f32(LRS[gi]), G.f32(WDS[gi]), nesterov)
        assert torch.equal(gp[lo:hi], rp) and torch.equal(gm[lo:hi], rm), (lo, hi)


def test_grouped_adamw_is_the_ungrouped_model_per_segment():
    offs, n, gmap = _layout()
    g, p, m, v = _state(n)
    for t in (1, 2, 7):
        gp, gm, gv = G.grouped_adamw(g, p, m, v, gmap, LRS, WDS, BETAS, EPS, t)
        for lo, hi, gi in _segments(offs, n):
            rp, rm, rv = adamw_update(g[lo:hi], p[lo:hi], m[lo:hi], v[lo:hi], LRS[gi], BETAS, EPS, WDS[gi], t)
            assert torch.equal(gp[lo:hi], rp) and torch.equal(gm[lo:hi], rm) and torch.equal(gv[lo:hi], rv), (t, lo)


@pytest.mark.parametrize("fault", G.FAULTS)
def test_every_planted_fault_is_caught(fault):
    offs, n, gmap = _layout()
    g, p, m, v = _state(n, seed=1)
    caught = []
    if fault != "lr_after_bc1_rounding":              # SGD has no bias correction
        ok = G.grouped_sgd(g, p, m, gmap, LRS, WDS, MU, False)
        bad = G.grouped_sgd(g, p, m, gmap, LRS, WDS, MU, False, fault=fault)
        caught.append(not torch.equal(ok[0], bad[0]))
    lrs, steps = LRS, range(1, 9)
    if fault == "lr_after_bc1_rounding":              # an lr and update whose lr / bc1 rounds otherwise from the rounded 1 / bc1
        lr, t = next((lr, t) for lr in (0.0001 * k for k in range(1, 500)) for t in range(1, 9)
                     if G.f32(G.group_step_sizes([lr], BETAS, t)[0]) != G.group_step_sizes([lr], BETAS, t, fault)[0])
        lrs, steps = [lr, lr, lr], [t]
        p = torch.zeros_like(p)                       # p = -step * (m / den): one ulp of step shows in every element
    hits = 0
    for t in steps:
        ok = G.grouped_adamw(g, p, m, v, gmap, lrs, WDS, BETAS, EPS, t)
        bad = G.grouped_adamw(g, p, m, v, gmap, lrs, WDS, BETAS, EPS, t, fault=fault)
        hits += not torch.equal(ok[0], bad[0])
    caught.append(hits > 0)
    assert all(caught), (fault, caught)
