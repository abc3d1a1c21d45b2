"""The LAMB / LARS kernel model of tests/layerwise_model.py against the fp64 references, and the planted faults the checks
must catch.

Bound: after 50 updates the model's largest parameter error against fp64 is at most 4x the error of the fp32 torch-op path
(what FlatLAMB / FlatLARS run on CPU tensors) on the same inputs, plus one fp32 ulp of the largest parameter.  Every planted
fault changes the model's bits and lands outside that bound."""
import pytest
import torch

import layerwise_model as L
from layerwise_cases import ADAPT, CASES, CHUNK, LAMB_HP, LARS_HP, _hp, bound, inputs, layout


def run_model(kind, hp, seed, fault=None, chunk=CHUNK):
    offsets, numels, p, grads = inputs(seed)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for t, g in enumerate(grads, 1):
        if kind == "lamb":
            p, m, v, _ = L.lamb_step(p, g, m, v, offsets, numels, ADAPT, hp, t, fault=fault, chunk=chunk)
        else:
            p, m, _ = L.lars_step(p, g, m, offsets, numels, ADAPT, hp, fault=fault, chunk=chunk)
    return p


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
