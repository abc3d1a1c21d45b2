"""Batched tensor-core engine (csrc/convnet_batched.cu) vs its plain-PyTorch fp32 model (ops/batched_reference.py).

The model rounds to bf16 exactly where the kernels do, so every intermediate and every gradient is compared with a bound
that an indexing / layout / descriptor bug cannot pass (round-1's TC test accepted rel < 0.2).  Intermediates are compared
sample by sample (tests/batched_checks.py), at batch sizes up to where every persistent loop and mbarrier ring of the
engine wraps.  A per-stage error report is written to <tmpdir>/batched_diag/ before anything is asserted."""
import json
import os
import tempfile

import pytest
import torch

import batched_checks as BC
import step_oracle as SO
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops import _ext
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


def _case(B, seed, training, u8=False, sample_base=0, step_value=3):
    """Parameters, engine input (uint8 or fp32), the model's fp32 input, targets, the step counter and the dropout scales."""
    torch.manual_seed(seed)
    net = b2.Net()
    params = pack_params(net, DEV)
    g = torch.Generator().manual_seed(seed + 1)
    if u8:
        xin = torch.randint(0, 256, (B, 1, 28, 28), dtype=torch.uint8, generator=g).to(DEV)
        x = BC.normalize_u8(xin)
    else:
        xin = x = torch.randn(B, 1, 28, 28, generator=g).to(DEV)
    y = torch.randint(0, 10, (B,), generator=g).to(DEV)
    step = torch.full((1,), step_value, dtype=torch.int64, device=DEV)
    m2 = dm = None
    if training:      # the dropout masks of this (seed, sample, step): exported by the per-sample engine (same Philox stream)
        _, _, masks = convnet_loss_and_grads(params, x, y, training=True, seed=77, step=step, sample_base=sample_base,
                                             return_masks=True)
        assert torch.equal(masks.cpu(), SO.dropout_masks(77, sample_base, B, step_value, 0.5)), "masks != host Philox"
        m2, dm = masks[:, :20].contiguous(), masks[:, 20:70].contiguous()
    return params, xin, x, y, step, m2, dm


def _size(B):
    """A batch size, or the name of one in tests/batched_checks.batch_sizes (derived from this GPU's SM count)."""
    if isinstance(B, int):
        return B
    return BC.batch_sizes(torch.cuda.get_device_properties(0).multi_processor_count)[B]


# size name -> (uint8 input, sample_base, step counter, gradient bucket pre-filled with the negated model result)
VARIANTS = {"1": (False, 0, 3, False), "3": (True, 0, 3, False), "4S+1": (False, 1000, 7, True), "8S+3": (True, 0, 3, True),
            "2048": (False, 0, 3, False), "4096": (True, 3 * 4096, 12345, False), "32S+1": (False, 0, 3, True),
            "8191": (True, 8191, 5, True)}


def _no_tf32():
    """The model's convolutions in full fp32 (cuDNN would otherwise run F.conv2d in TF32); matmuls are fp32 by default."""
    assert not torch.backends.cuda.matmul.allow_tf32
    return torch.backends.cudnn.flags(enabled=True, allow_tf32=False)


@pytest.mark.parametrize("B,training", [(2, False), (64, True), (333, True)] + [(n, n != "1") for n in BC.SIZE_NAMES])
def test_every_stage_matches_the_rounding_exact_model(B, training):
    """Every stage, sample by sample, at the batch sizes where the engine's persistent loops and mbarrier rings wrap."""
    name, B = str(B), _size(B)
    u8, sample_base, step_value, prefill = VARIANTS.get(name, (False, 0, 3, False))
    params, xin, x, y, step, m2, dm = _case(B, 11 + B, training, u8, sample_base, step_value)
    with _no_tf32():
        ref0 = R.forward_backward(params, x, y, m2, dm, emulate_bf16=True)
    bucket = BC.prefill_bucket(ref0["named"], DEV) if prefill else None
    before = bucket.clone() if prefill else None
    loss, grads, bufs = batched_loss_and_grads(params, xin, y, training=training, seed=77, step=step,
                                               sample_base=sample_base, grads=bucket)
    torch.cuda.synchronize()
    rep = {"B": B, "size": name, "training": training, "uint8": u8, "sample_base": sample_base, "step": step_value,
           "prefilled_bucket": prefill}
    p1 = bufs.P1.view(B, 12, 12, 16)[..., :10].permute(0, 3, 1, 2).float()
    rep["p1_vs_torch_conv"] = _rel(p1, ref0["p1"])                 # different fp32 summation order: a few bf16 ulps
    code = bufs.A1.view(B, 10, 12, 12)
    a1 = (code & 3).long()
    ry, rx = (ref0["a1"] // 24) % 2, (ref0["a1"] % 24) % 2
    rep["a1_agree"] = float(((a1 == ry * 2 + rx) | (ref0["p1"] == 0)).float().mean())
    rep["a1_dead_flag"] = float((((code & 4) != 0) == (p1 == 0)).float().mean())
    bad = []
    if prefill:       # the kernels only accumulate: their sum is bucket - prefill; padding keeps its sentinel
        grads = grads.double() - before.double()
        pads = BC.pad_slots().to(DEV)
        rep["pad_slots_written"] = int((bucket[pads] != BC.SENTINEL).sum())
        if rep["pad_slots_written"]:
            bad.append("padding slots of the gradient bucket were written")
    # everything downstream is compared on the engine's own conv1 output, pool codes, P2 and fc1 output
    with _no_tf32():
        bad += BC.compare_pipeline(rep, bufs, params, x, y, m2, dm, grads=grads, loss=loss)[0]
    _dump(f"batched_diag_B{B}.json", rep)
    assert not bad, (bad, rep)
    assert rep["a1_agree"] > 0.999 and rep["a1_dead_flag"] == 1.0 and rep["p1_vs_torch_conv"] < 5e-3, rep


@pytest.mark.parametrize("size", BC.SIZE_NAMES)
def test_forward_only_matches_the_model_at_every_size(size):
    """batched_forward (no backward, log-probabilities out) on the engine's own P1 / codes / P2 / fc1 output."""
    B = _size(size)
    params, xin, x, y, _, _, _ = _case(B, 31 + B, False, VARIANTS[size][0])
    bufs = BatchedBuffers(B, DEV)
    got = batched_forward(params, xin, bufs)
    torch.cuda.synchronize()
    rep = {"B": B, "size": size, "uint8": VARIANTS[size][0]}
    with _no_tf32():
        bad, ref = BC.compare_pipeline(rep, bufs, params, x, y, None, None, backward=False)
    bad += BC.check_rows(rep, "logp", got, ref["logp"], BC.STAGE_BOUNDS["logp"], BC.BATCH_BOUND)
    _dump(f"batched_forward_B{B}.json", rep)
    assert not bad, (bad, rep)


def test_empty_batch_raises_and_launches_nothing():
    params = pack_params(b2.Net(), DEV)
    C = _ext.C()
    bufs = BatchedBuffers(0, DEV)
    grads = torch.full((params.numel(),), BC.SENTINEL, device=DEV)
    acc = torch.zeros(2, device=DEV)
    x, y = torch.empty(0, 1, 28, 28, device=DEV), torch.empty(0, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="empty batch"):
        C.bt_step(params, grads, x, y, bufs.as_list(), acc, None, None, 0, 0, True, 1.0, 0.5, 255)
    with pytest.raises(RuntimeError, match="empty batch"):
        batched_forward(params, x)
    torch.cuda.synchronize()
    assert bool((grads == BC.SENTINEL).all()) and bool((acc == 0).all())


def test_forward_only_matches_net_eval():
    params, _, x, y, _, _, _ = _case(100, 5, False)
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
