"""Batched tensor-core engine (csrc/convnet_batched.cu) vs its plain-PyTorch fp32 model (ops/batched_reference.py).

The model rounds to bf16 exactly where the kernels do, so every intermediate and every gradient is compared with a bound
that an indexing / layout / descriptor bug cannot pass (round-1's TC test accepted rel < 0.2).  A per-tensor error report
is written to <tmpdir>/batched_diag/ before anything is asserted."""
import json
import os
import tempfile

import pytest
import torch

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops import batched_reference as R
from dist_tuto.pth_b200.ops.convnet_batched import STAGES, BatchedBuffers, BatchedTrainer, batched_forward, batched_loss_and_grads
from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads, pack_params, unpack_params

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda:0"


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _dump(name, payload):
    d = os.path.join(tempfile.gettempdir(), "batched_diag")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "w") as f:
        json.dump(payload, f, indent=1)


def _case(B, seed, training):
    torch.manual_seed(seed)
    net = b2.Net()
    params = pack_params(net, DEV)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(B, 1, 28, 28, generator=g).to(DEV)
    y = torch.randint(0, 10, (B,), generator=g).to(DEV)
    step = torch.full((1,), 3, dtype=torch.int64, device=DEV)
    m2 = dm = None
    if training:      # the dropout masks of this (seed, sample, step): exported by the per-sample engine (same Philox stream)
        _, _, masks = convnet_loss_and_grads(params, x, y, training=True, seed=77, step=step, return_masks=True)
        m2, dm = masks[:, :20].contiguous(), masks[:, 20:70].contiguous()
    return params, x, y, step, m2, dm


@pytest.mark.parametrize("B,training", [(2, False), (64, True), (333, True)])
def test_every_stage_matches_the_rounding_exact_model(B, training):
    params, x, y, step, m2, dm = _case(B, 11 + B, training)
    ref0 = R.forward_backward(params, x, y, m2, dm, emulate_bf16=True)
    loss, grads, bufs = batched_loss_and_grads(params, x, y, training=training, seed=77, step=step)
    torch.cuda.synchronize()
    rep = {"B": B, "training": training}
    p1 = bufs.P1.view(B, 12, 12, 16)[..., :10].permute(0, 3, 1, 2).float()
    rep["p1_vs_torch_conv"] = _rel(p1, ref0["p1"])                 # different fp32 summation order: a few bf16 ulps
    rep["p1_ones_channel_intact"] = bool((bufs.P1.view(B, 12, 12, 16)[..., 10] == 1).all() and (bufs.P1.view(B, 12, 12, 16)[..., 11:] == 0).all())
    code = bufs.A1.view(B, 10, 12, 12)
    a1 = (code & 3).long()
    ry, rx = (ref0["a1"] // 24) % 2, (ref0["a1"] % 24) % 2
    rep["a1_agree"] = float(((a1 == ry * 2 + rx) | (ref0["p1"] == 0)).float().mean())
    rep["a1_dead_flag"] = float((((code & 4) != 0) == (p1 == 0)).float().mean())
    # everything downstream is compared on the engine's own (bit-identical) conv1 output
    ref = R.forward_backward(params, x, y, m2, dm, emulate_bf16=True, p1_override=p1, a1_override=a1)
    rep["p2"] = _rel(bufs.P2.view(B, 320), ref["p2"])
    rep["hrelu"] = _rel(bufs.Hrelu.view(B, 64)[:, :50], ref["hrelu"])
    rep["loss"] = abs(float(loss) - float(ref["loss"])) / abs(float(ref["loss"]))
    rep["dh"] = _rel(bufs.DH.view(B, 64)[:, :50], ref["dh"])
    rep["dc"] = _rel(bufs.DC.view(B, 32, 8, 8)[:, :20], ref["dc"])
    rep["dc_pad_zero"] = bool((bufs.DC.view(B, 32, 64)[:, 20:] == 0).all())
    rep["g1"] = _rel(bufs.G1.view(B, 10, 12, 12), ref["g1"])
    mine, want = unpack_params(grads), unpack_params(ref["grads"])
    for n in want:
        rep["grad/" + n] = _rel(mine[n], want[n])
    _dump(f"batched_diag_B{B}.json", rep)
    loose = ("a1_agree", "a1_dead_flag", "p1_vs_torch_conv")
    bad = {k: v for k, v in rep.items() if isinstance(v, float) and k not in loose and v > 5e-3}
    assert not bad, rep
    assert rep["a1_agree"] > 0.999 and rep["a1_dead_flag"] == 1.0 and rep["p1_vs_torch_conv"] < 5e-3, rep
    assert rep["p1_ones_channel_intact"] and rep["dc_pad_zero"], rep


def test_forward_only_matches_net_eval():
    params, x, y, _, _, _ = _case(100, 5, False)
    net = b2.Net().to(DEV).eval()
    net.load_state_dict({k: v.clone() for k, v in unpack_params(params).items()})
    with torch.no_grad():
        want = net(x)
    got = batched_forward(params, x)
    torch.cuda.synchronize()
    assert float((got - want).abs().max()) < 5e-2
    assert float((got.argmax(1) == want.argmax(1)).float().mean()) > 0.97


def test_uint8_input_is_normalised_in_kernel():
    B = 48
    torch.manual_seed(9)
    params = pack_params(b2.Net(), DEV)
    xu = torch.randint(0, 256, (B, 1, 28, 28), dtype=torch.uint8, device=DEV)
    y = torch.randint(0, 10, (B,), device=DEV)
    xf = ((xu.float() / 255.0) - 0.1307) / 0.3081
    l0, g0, _ = batched_loss_and_grads(params, xf, y)
    l1, g1, _ = batched_loss_and_grads(params, xu, y)
    torch.cuda.synchronize()
    assert abs(float(l0) - float(l1)) < 1e-4 * abs(float(l0))
    assert _rel(g1, g0) < 1e-3


def test_trainer_tracks_torch_sgd_on_the_model():
    """20 steps of the batched trainer (CUDA graph, fused SGD kernel) vs torch.optim.SGD on the fp32 Net, eval mode."""
    B = 256
    torch.manual_seed(21)
    net = b2.Net().to(DEV).eval()
    tr = BatchedTrainer(B, lr=0.05, momentum=0.5, seed=1, device=DEV, init_from=net)
    tr.eval()
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.5)
    g = torch.Generator().manual_seed(4)
    xs = torch.randn(8, B, 1, 28, 28, generator=g)
    ys = torch.randint(0, 10, (8, B), generator=g)
    ref_losses = []
    for it in range(20):
        x, y = xs[it % 8], ys[it % 8]
        tr.step(x.pin_memory(), y.pin_memory())
        opt.zero_grad()
        loss = torch.nn.functional.nll_loss(net(x.to(DEV)), y.to(DEV))
        loss.backward()
        opt.step()
        ref_losses.append(float(loss))
    total = tr.pop_loss_sum()
    assert abs(total - sum(ref_losses)) < 2e-2 * sum(ref_losses), (total, sum(ref_losses))
    mine = unpack_params(tr.params)
    for n, p in net.named_parameters():
        assert _rel(mine[n], p.detach()) < 2e-2, (n, _rel(mine[n], p.detach()))
    sd = tr.state_dict()
    assert sd["steps"] == 20 and set(sd["momentum"]) == {n for n, _ in net.named_parameters()}
