"""The LAMB / LARS kernel model of tests/layerwise_model.py against the fp64 references, and the planted faults the checks
must catch.

Bound: after 50 updates the model's largest parameter error against fp64 is at most 4x the error of the fp32 torch-op path
(what FlatLAMB / FlatLARS run on CPU tensors) on the same inputs, plus one fp32 ulp of the largest parameter.  Every planted
fault changes the model's bits and lands outside that bound."""
import pytest
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


def run_model(kind, hp, seed, fault=None, chunk=CHUNK):
    offsets, numels, p, grads = inputs(seed)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for t, g in enumerate(grads, 1):
        if kind == "lamb":
            p, m, v, _ = L.lamb_step(p, g, m, v, offsets, numels, ADAPT, hp, t, fault=fault, chunk=chunk)
        else:
            p, m, _ = L.lars_step(p, g, m, offsets, numels, ADAPT, hp, fault=fault, chunk=chunk)
    return p


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


@pytest.mark.parametrize("kind,k", CASES)
def test_model_is_within_the_bound_of_fp64(kind, k):
    ref, b = bound(kind, _hp(kind, k), 10 + k)
    err = float((run_model(kind, _hp(kind, k), 10 + k).double() - ref).abs().max())
    assert err <= b, (err, b)


@pytest.mark.parametrize("kind,fault", [("lamb", f) for f in L.FAULTS_LAMB] + [("lars", f) for f in L.FAULTS_LARS])
def test_planted_faults_are_caught(kind, fault):
    hp = _hp(kind, 1)
    ref, b = bound(kind, hp, 7)
    clean, bad = run_model(kind, hp, 7), run_model(kind, hp, 7, fault)
    assert not torch.equal(clean, bad), f"{fault}: the bit-for-bit check would not see it"
    err = float((bad.double() - ref).abs().max())
    assert err > b, f"{fault}: error {err} within the bound {b}"


def test_chunk_table_never_crosses_a_tensor():
    offsets, numels, _ = layout([(L.CHUNK + 1,), (3,), (2 * L.CHUNK,), (L.CHUNK - 1,)])
    table = L.chunk_table(offsets, numels)
    assert all(ln <= L.CHUNK for _, ln, _ in table)
    for start, ln, t in table:
        assert offsets[t] <= start and start + ln <= offsets[t] + numels[t]
    assert [t for *_, t in table] == [0, 0, 1, 2, 2, 3]


def test_zero_tensor_and_zero_gradient_have_ratio_one():
    offsets, numels = [0, 8], [8, 8]
    p = torch.cat([torch.zeros(8), torch.randn(8)])
    g = torch.cat([torch.randn(8), torch.zeros(8)])
    z = torch.zeros(16)
    hp = dict(LARS_HP[0])
    _, _, r = L.lars_step(p, g, z, offsets, numels, [True, True], hp)
    assert r == [1.0, 1.0]
    _, _, _, r = L.lamb_step(p, torch.zeros(16), z, z, offsets, numels, [True, True], dict(LAMB_HP[0], weight_decay=0.0), 1)
    assert r == [1.0, 1.0]                    # without decay, a zero gradient gives u == 0


def test_chunk_partials_follow_the_thread_order():
    """One chunk of 3 vectors + a tail: thread t holds its vector's fmaf chain, thread 0..2 a tail element as well."""
    x = torch.randn(4 * 300 + 3)
    s = L.chunk_sqsum(x)
    assert abs(s - float((x.double() ** 2).sum())) <= 1e-5 * s
