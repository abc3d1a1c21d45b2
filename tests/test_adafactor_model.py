"""The rounding-exact model of FlatAdafactor's kernels (tests/adafactor_model.py) on the CPU: its chunk table never crosses a
tensor and covers every element once, it stays within the stated bound of an fp64 Adafactor on every shape class (with decay
on and off, and with d > 1 so that the update clipping is active), and every planted fault misses that bound by a wide
margin.

The bound, per tensor: max |model - fp64| <= 4 * max |torch fp32 - fp64| + 2 ulp(max |fp64|), torch fp32 being
``torch.optim.Adafactor(foreach=False)`` on the CPU."""
import math

import pytest
import torch

import adafactor_model as M

SPECS = [((), None), ((7,), None), ((5, 3), None), ((2, 3, 4), None), ((6, 4, 3, 3), "cl"), ((100, 130), None),
         ((1, 9000), None), ((9000, 1), None)]
HP = dict(beta2_decay=-0.8, eps1=torch.finfo(torch.float32).eps, eps2=1e-3)


def _layout():
    tensors, o = [], 0
    for shp, fmt in SPECS:
        t = torch.empty(shp)
        st = t.to(memory_format=torch.channels_last).stride() if fmt else t.stride()
        tensors.append((o, shp, st, 0))
        o += (math.prod(shp) + 3) // 4 * 4
    return tensors, o


def _ratios(fault=None, wd=0.1, d=1.5, steps=3, seed=0):
    """Per tensor: the model's error against fp64 over the bound (> 1 fails), after ``steps`` scheduled updates."""
    torch.manual_seed(seed)
    tensors, n = _layout()
    hp = dict(HP, d=d)
    p0 = torch.randn(n)
    state = torch.zeros(M.state_offsets([t[1] for t in tensors])[1])
    views = lambda f: [f[o:o + math.prod(s)].as_strided(s, st) for o, s, st, _ in tensors]  # noqa: E731
    p, gs, lrs = p0.clone(), [], []
    for t in range(1, steps + 1):
        g = torch.randn(n) * (3.0 ** t)                 # growing gradients: ||u|| / sqrt(numel) > d, the clipping acts
        o2, o3, o4 = tensors[2][0], tensors[3][0], tensors[4][0]
        g[o2:o2 + 15] *= 1e-5                           # v below eps1: the eps1^2 clamp matters
        g[o3:o3 + 12] *= 10                             # slices of different scale: the per-slice mean matters
        g[o4:o4 + 144] *= 10
        lr = 1e-2 * (0.5 + 0.25 * t)                    # a schedule: rho_t from the scheduled lr
        gs.append(g)
        lrs.append(lr)
        p, state, _, _ = M.adafactor_step(p, g, state, tensors, [(lr, wd, 1e-2)], hp, t, fault)
    ref = M.adafactor_fp64(views(p0), [views(g) for g in gs], hp, [[lr] * len(tensors) for lr in lrs],
                           [[wd] * len(tensors)] * steps)
    ws = [torch.nn.Parameter(v.clone()) for v in views(p0)]
    opt = torch.optim.Adafactor([{"params": [w]} for w in ws], lr=1e-2, beta2_decay=hp["beta2_decay"], eps=(None, hp["eps2"]),
                                d=d, weight_decay=wd, foreach=False)
    for g, lr in zip(gs, lrs):
        for grp, w, gv in zip(opt.param_groups, ws, views(g)):
            grp["lr"] = lr
            w.grad = gv.clone()
        opt.step()
    out = []
    for v, r, w in zip(views(p), ref, ws):
        em = float((v.double() - r).abs().max())
        et = float((w.detach().double() - r).abs().max())
        out.append(em / (4 * et + 2 * float(r.abs().max()) * 2.0 ** -23) if not math.isnan(em) else math.inf)
    return out


def test_table_covers_every_element_once_and_never_crosses_a_tensor():
    shapes = [(), (7,), (5, 3), (300, 300), (3, 70, 200), (1, 20000), (20000, 1), (64, 32, 3, 3), (0, 5)]
    for shape, (chunks, whole, TR, TC) in zip(shapes, M.table(shapes)):
        n = math.prod(shape)
        f = M.factors(shape) or (1, 1, n)
        seen = torch.zeros(f, dtype=torch.int32) if n else None
        for b0, nb, r0, nr, c0, nc in chunks:
            assert 0 < nb * nr * nc <= M.CHUNK and b0 + nb <= f[0] and r0 + nr <= f[1] and c0 + nc <= f[2]
            assert nb == 1 or (nr, nc) == f[1:], "several slices only when whole"
            seen[b0:b0 + nb, r0:r0 + nr, c0:c0 + nc] += 1
        assert n == 0 or bool((seen == 1).all()), shape


@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("d", [1.0, 1.5])
def test_model_within_the_bound_of_fp64(wd, d):
    r = _ratios(wd=wd, d=d)
    assert max(r) <= 1.0, r


@pytest.mark.parametrize("fault", M.FAULTS)
def test_every_planted_fault_misses_the_bound_widely(fault):
    r = _ratios(fault=fault)
    assert max(r) > 10.0, (fault, r)
