"""The LAMB / LARS cases of tests/test_layerwise_model.py, which the kernel and sharded-model tests reuse: the shapes,
hyperparameters and inputs, and the bound against fp64.

Bound: after 50 updates the model's largest parameter error against fp64 is at most 4x the error of the fp32 torch-op path
(what FlatLAMB / FlatLARS run on CPU tensors) on the same inputs, plus one fp32 ulp of the largest parameter."""
import torch

import layerwise_model as L

STEPS = 50
CHUNK = 64                      # small chunks: many chunk boundaries and several chunks per tensor at small sizes
# tensors of different scales; the 1-D ones are excluded (the default rule); sizes not multiples of 4 leave alignment gaps
SHAPES = [(13, 11), (11,), (300,), (7, 9), (1,), (130,)]
ADAPT = [len(s) > 1 for s in SHAPES]
LAMB_HP = [dict(lr=1e-2, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01),
           dict(lr=2e-2, betas=(0.3, 0.9), eps=1e-3, weight_decay=0.1)]        # beta1 < 0.5: the lerp's other branch
LARS_HP = [dict(lr=0.1, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-3, eps=1e-8, nesterov=False),
           dict(lr=0.5, momentum=0.8, weight_decay=5e-2, trust_coefficient=2e-2, eps=1e-2, nesterov=True)]


def layout(shapes=SHAPES):
    offsets, numels, n = [], [], 0
    for s in shapes:
        k = int(torch.Size(s).numel())
        offsets.append(n)
        numels.append(k)
        n += (k + 3) // 4 * 4
    return offsets, numels, n


def inputs(seed, steps=STEPS, shapes=SHAPES):
    offsets, numels, n = layout(shapes)
    gen = torch.Generator().manual_seed(seed)
    p0, grads = torch.zeros(n), [torch.zeros(n) for _ in range(steps)]
    for i, (o, k) in enumerate(zip(offsets, numels)):
        scale = 4.0 ** (i % 3 - 1)
        p0[o:o + k] = torch.randn(k, generator=gen) * scale
        for g in grads:
            g[o:o + k] = torch.randn(k, generator=gen) * 0.1 / scale
    return offsets, numels, p0, grads


def run_torch_ops(kind, hp, seed):
    offsets, numels, p0, grads = inputs(seed)
    ps = [p0[o:o + k].clone() for o, k in zip(offsets, numels)]
    ms, vs = [torch.zeros_like(p) for p in ps], [torch.zeros_like(p) for p in ps]
    for t, g in enumerate(grads, 1):
        gs = [g[o:o + k] for o, k in zip(offsets, numels)]
        for i in range(len(ps)):
            if kind == "lamb":
                L.torch_lamb_tensor(ps[i], gs[i], ms[i], vs[i], ADAPT[i], hp, t)
            else:
                r = L.torch_lars_ratio(ps[i], gs[i], ADAPT[i], hp)
                d = L.torch_lars_direction(ps[i], gs[i], ADAPT[i], hp, r)
                L.torch_sgd(ps[i], d, ms[i], hp)
    out = p0.clone()
    for (o, k), p in zip(zip(offsets, numels), ps):
        out[o:o + k] = p
    return out


def bound(kind, hp, seed):
    offsets, numels, p0, grads = inputs(seed)
    ref = (L.lamb_fp64 if kind == "lamb" else L.lars_fp64)(p0, grads, offsets, numels, ADAPT, hp)
    e_torch = float((run_torch_ops(kind, hp, seed).double() - ref).abs().max())
    big = ref.abs().max().float()
    ulp = float(torch.nextafter(big, torch.tensor(float("inf"))) - big)
    return ref, 4 * e_torch + ulp


CASES = [("lamb", k) for k in range(len(LAMB_HP))] + [("lars", k) for k in range(len(LARS_HP))]


def _hp(kind, k):
    return (LAMB_HP if kind == "lamb" else LARS_HP)[k]
