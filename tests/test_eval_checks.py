"""CPU tier: the references and checks of tests/eval_checks.py -- the fp64 reference against ``Net.eval()``, a plain fp32
model of the evaluation kernel passing every check, the size table covering the kernel's schedule, and planted faults in
that model that the checks must report (bounded checks by at least 10x)."""
import math

import numpy as np
import pytest
import torch

import batched_checks
import eval_checks as E
import step_oracle as O
from dist_tuto.pth_b200.data import MNIST_MEAN, MNIST_STD
from dist_tuto.pth_b200.models.convnet import Net
from dist_tuto.pth_b200.ops.convnet_fused import pack_params, unpack_params

S = 8
G = 4            # a small device: S * G = 32 samples per wave keeps the fp32 model cheap
MEAN, STD = 0.4, 0.2
TIE_A, TIE_B = 3, 6


def emulate(params, x, y, mean, std, fault=None):
    """The kernel's ``(out_logp, result)`` in plain fp32: the forward of ``Net.eval()`` on the normalised image, log-probs
    as ``logit - (max + log(sum exp(logit - max)))``, ties to the lowest index, each CTA's nll summed sample by sample in
    fp32 over its groups c, c + grid, ..., the slots added in fp64 in CTA order.  ``fault`` plants one bug."""
    mean_k, std_k = (MNIST_MEAN, MNIST_STD) if fault == "mnist_norm" else (mean, std)
    xin = E.model_input(x, mean_k, std_k)
    if fault == "renormalise" and x.dtype != torch.uint8:
        xin = (xin - np.float32(mean)) * (np.float32(1) / np.float32(std))
    p = O._params(params, torch.float32)
    if fault == "conv2_bias":
        p["conv2.bias"][7] = 0.0
    N = xin.shape[0]
    m = O.dropout_masks(5, 0, N, 1, 0.5) if fault == "dropout" else torch.ones(N, 70)
    z = O.masked_forward(p, xin, m[:, :20], m[:, 20:])
    mx = z.max(dim=1, keepdim=True).values
    logp = z - mx if fault == "no_lse" else z - (mx + torch.log(torch.exp(z - mx).sum(dim=1, keepdim=True)))
    sch = E.schedule(N, G, S)
    grid, groups = sch["grid"], (N + S - 1) // S
    if fault == "stale_row":                    # the last sample's row from the same slot of its CTA's previous group
        logp[N - 1] = logp[N - 1 - S * grid]
    pred = 9 - z.flip(1).argmax(dim=1) if fault == "ties_high" else z.argmax(dim=1)
    nll = -logp.gather(1, y[:, None])[:, 0]
    loss = [np.float32(0)] * grid
    corr = [0] * grid
    for g in range(groups):
        c = g % grid
        for i in range(g * S, min(N, g * S + S)):
            if fault == "skip_last" and i == N - 1 and N % S:
                continue
            loss[c] = np.float32(loss[c] + np.float32(nll[i]))
            corr[c] += int(pred[i] == y[i])
    total = 0.0
    for c in range(grid):
        total += float(loss[c])
    n = groups * S if fault == "whole_groups" else N
    return logp, [total, float(sum(corr)), float(n)]


def _net(seed=0):
    torch.manual_seed(seed)
    return Net()


def _inputs(N, u8, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (N, 28, 28), generator=g, dtype=torch.uint8) if u8 else torch.randn(N, 1, 28, 28, generator=g)
    return x, torch.randint(0, 10, (N,), generator=g)


def _refs(params, x, y, mean=MEAN, std=STD):
    return E.reference(params, x, y, mean, std), E.reference(params, x, y, mean, std, torch.float32)


# ------------------------------------------------------------------------------------------------------- reference
@pytest.mark.parametrize("u8", [True, False])
def test_reference_is_net_eval_in_fp64(u8):
    net = _net(3)
    x, y = _inputs(37, u8)
    ref = E.reference(pack_params(net), x, y, MEAN, STD)
    with torch.no_grad():
        out = net.double().eval()(E.model_input(x, MEAN, STD).double())
    assert torch.allclose(ref["logp"], out, rtol=1e-13, atol=1e-13)
    assert torch.allclose(ref["loss"], -out.gather(1, y[:, None])[:, 0], rtol=1e-13, atol=1e-13)
    assert torch.equal(ref["argmax"], out.argmax(1))
    top2 = out.topk(2, dim=1).values                  # log_softmax shifts a row's logits alike: the same margin
    assert torch.allclose(ref["margin"], top2[:, 0] - top2[:, 1], rtol=1e-9, atol=1e-13)
    # log-sum-exp and largest |logit| of the logits the log-probs come from
    z = ref["logp"] + ref["lse"][:, None]
    assert torch.allclose(torch.logsumexp(z, 1), ref["lse"], rtol=1e-13, atol=1e-13)
    assert torch.allclose(z.abs().amax(1), ref["zmax"], rtol=1e-12, atol=1e-13)


def test_uint8_normalisation_uses_the_mean_and_std_passed_as_the_kernel_does():
    xu = torch.tensor([0, 1, 128, 255], dtype=torch.uint8).repeat(196).reshape(1, 28, 28)
    f32 = np.float32
    want = (xu.float() * (f32(1) / f32(255)) - f32(0.5)) * (f32(1) / f32(0.25))
    assert torch.equal(E.normalize_u8(xu, 0.5, 0.25), want.reshape(1, 1, 28, 28))
    # with MNIST's constants it is the batched engine's normalisation, bit for bit
    assert torch.equal(E.normalize_u8(xu, MNIST_MEAN, MNIST_STD), batched_checks.normalize_u8(xu).reshape(1, 1, 28, 28))
    assert torch.equal(E.model_input(xu.float().reshape(1, 1, 28, 28), 0.5, 0.25), xu.float().reshape(1, 1, 28, 28))


def test_invalid_labels_give_an_infinite_reference_loss():
    x, _ = _inputs(4, True)
    y = torch.tensor([-1, 10, 2 ** 40, 3])
    ref = E.reference(pack_params(_net()), x, y, MEAN, STD)
    assert ref["loss"][:3].tolist() == [math.inf] * 3 and math.isfinite(float(ref["loss"][3]))


# ------------------------------------------------------------------------------------------------------- size table
@pytest.mark.parametrize("g", [132, 114])
def test_size_table_reaches_every_schedule_edge(g):
    table = E.eval_sizes(g, S)
    assert E.gaps(g, S, table) == []
    assert len(set(table)) == len(table)
    SG = S * g
    assert {0, 1, 7, 8, 9, SG - 1, SG, SG + 1} <= set(table)
    assert any(SG < n < 2 * SG for n in table) and any(E.schedule(n, g, S)["groups"].min() >= 3 for n in table if n)
    assert {n % S for n in table} == set(range(S))


def test_gaps_notices_a_missing_edge():
    table = E.eval_sizes(132, S)
    assert E.gaps(132, S, [n for n in table if n != 1056]) == ["N = 1056 never runs"]
    assert any("3rd or later" in s and "= 5" in s for s in E.gaps(132, S, [n for n in table if n < 2 * 1056 or n % S != 5]))
    assert "no case where every CTA runs three or more groups" in E.gaps(132, S, [n for n in table if n < 3 * 1056])


def test_schedule_follows_the_persistent_grid():
    s = E.schedule(2 * 32 + 8 + 3, 4, 8)           # 10 groups on 4 CTAs: 3, 3, 2, 2 groups; the last (3 samples) on CTA 1
    assert s["grid"] == 4 and s["groups"].tolist() == [3, 3, 2, 2] and s["samples"].tolist() == [24, 19, 16, 16]
    assert s["last_cta_groups"] == 3 and s["residue"] == 3
    assert E.schedule(5, 4, 8)["grid"] == 1 and E.schedule(0, 4, 8)["grid"] == 0


# ------------------------------------------------------------------------------------------------- fp32 passes
@pytest.mark.parametrize("u8", [True, False])
def test_plain_fp32_model_passes_every_check_on_the_size_table(u8):
    net = _net(7)
    params = pack_params(net)
    table = E.eval_sizes(G, S)
    x, y = _inputs(max(table), u8, seed=2)
    r64, r32 = _refs(params, x, y)
    worst = {}
    for n in table:
        lp, res = emulate(params, x[:n], y[:n], MEAN, STD)
        rep = E.check_eval(res, lp, y[:n], E.sliced(r64, 0, n), E.sliced(r32, 0, n), G, S, where=f"N={n}: ")
        assert not rep.failures, rep.message()
        for k, v in rep.ratios.items():
            worst[k] = max(worst.get(k, 0.0), v)
    assert worst["logp"] < 1.0 and worst["loss"] < 1.0 and worst["sum"] <= 1.0


def test_plain_fp32_model_passes_on_exact_ties_and_a_saturated_softmax():
    params = pack_params(_net(8))
    x, _ = _inputs(75, True, seed=3)
    y = torch.where(torch.arange(75) % 3 == 0, TIE_B, TIE_A)
    tied = E.tie_fc2(params, TIE_A, TIE_B)
    r64, r32 = _refs(tied, x, y)
    assert bool((r64["margin"] == 0).all()) and bool((r64["argmax"] == TIE_A).all())
    lp, res = emulate(tied, x, y, MEAN, STD)
    assert res[1] == int((y == TIE_A).sum())
    rep = E.check_eval(res, lp, y, r64, r32, G, S)
    assert not rep.failures, rep.message()
    hot = params.clone()
    unpack_params(hot)["fc2.weight"].mul_(1e3)
    unpack_params(hot)["fc2.bias"].mul_(1e3)
    y = _inputs(75, True, seed=3)[1]
    r64, r32 = _refs(hot, x, y)
    assert float(r64["zmax"].max()) > 100
    lp, res = emulate(hot, x, y, MEAN, STD)
    rep = E.check_eval(res, lp, y, r64, r32, G, S)
    assert not rep.failures, rep.message()


# ------------------------------------------------------------------------------------------------- planted faults
# (fault, input is uint8, tied fc2, the check that must catch it)
FAULTS = [
    ("no_lse", True, False, "logp"),              # log-probs as logit - max
    ("conv2_bias", True, False, "logp"),          # one conv2 channel's bias dropped
    ("mnist_norm", True, False, "logp"),          # MNIST mean / std instead of the ones passed
    ("ties_high", True, True, "correct"),         # ties to the highest index
    ("skip_last", True, False, "sum"),            # the last sample of a partial group left out of the loss sum
    ("stale_row", True, False, "logp"),           # a row from the same slot of the CTA's previous group
    ("dropout", True, False, "logp"),             # dropout applied in eval mode
    ("renormalise", False, False, "logp"),        # fp32 input normalised a second time
    ("whole_groups", True, False, "n"),           # result[2] counting whole groups
]


@pytest.mark.parametrize("fault,u8,tied,check", FAULTS, ids=[f[0] for f in FAULTS])
def test_planted_fault_is_caught(fault, u8, tied, check):
    N = 2 * S * G + S + 3                         # the last group (3 samples) is its CTA's 3rd
    params = pack_params(_net(11))
    x, y = _inputs(N, u8, seed=4)
    if tied:
        params = E.tie_fc2(params, TIE_A, TIE_B)
        y = torch.where(torch.arange(N) % 3 == 0, TIE_B, TIE_A)
    r64, r32 = _refs(params, x, y)
    lp, res = emulate(params, x, y, MEAN, STD)
    clean = E.check_eval(res, lp, y, r64, r32, G, S)
    assert not clean.failures, clean.message()
    lp, res = emulate(params, x, y, MEAN, STD, fault=fault)
    rep = E.check_eval(res, lp, y, r64, r32, G, S)
    assert rep.failures, f"{fault} not caught"
    assert rep.ratios[check] >= 10.0, f"{fault}: {check} only {rep.ratios[check]:.3g}x its bound\n{rep.message()}"
    print(f"{fault}: caught by {check} at {rep.ratios[check]:.3g}x the bound")
