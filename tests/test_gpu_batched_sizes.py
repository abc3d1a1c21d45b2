"""Batched tensor-core engine (csrc/convnet_batched.cu) at the batch sizes it trains at, one kernel and one step at a time.

* Each gradient kernel runs alone (``stage_mask``) on operands the test writes in the engine's buffer layouts, at every
  size of ``batched_checks.batch_sizes``, against an exact fp64 result; the gradient bucket is pre-filled with the negated
  result and a sentinel in every slot the kernel must not touch.
* ``BatchedTrainer`` at 2048 and 4096 raw-uint8 samples (bench.py's large-batch configuration): after every CUDA-graph
  step and one odd eager tail batch, the step's gradient is recovered from the momentum buffer and compared with the model
  evaluated at the previous parameters, stage by stage and sample by sample.
Per-kernel and per-step error reports go to <tmpdir>/batched_diag/."""
import json
import os
import tempfile

import pytest
import torch

import batched_checks as BC
import step_oracle as SO
from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.ops.convnet_batched import BatchedBuffers, BatchedTrainer
from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda:0"


def _dump(name, payload):
    d = os.path.join(tempfile.gettempdir(), "batched_diag")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "w") as f:
        json.dump(payload, f, indent=1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run_alone(kernel, B, op, grads, bufs):
    """One launch of ``kernel`` through bt_step's stage mask, on the operands ``op`` written into ``bufs``."""
    for k, v in op["bufs"].items():
        getattr(bufs, k).view(-1)[:v.numel()].copy_(v.reshape(-1))
    C = _ext.C()
    C.bt_pack_weights(op["params"], bufs.as_list())
    y = torch.zeros(B, dtype=torch.int64, device=DEV)
    C.bt_step(op["params"], grads, op["x"].contiguous(), y, bufs.as_list(), None, None, None, 0, 0, False, 1.0 / B, 0.5,
              BC.STAGE_BIT[kernel])
    torch.cuda.synchronize()


@pytest.mark.parametrize("size", BC.SIZE_NAMES)
@pytest.mark.parametrize("kernel,x_u8", [("conv2_wgrad", False), ("conv1_wgrad", False), ("conv1_wgrad", True),
                                         ("fc_wgrad", False)])
def test_reduction_kernel_matches_fp64(kernel, x_u8, size):
    B = BC.batch_sizes(_sms())[size]
    op = BC.synthetic(kernel, B, seed=1000 + B, device=DEV, x_u8=x_u8)
    grads = BC.prefill_bucket(op["want"], DEV)
    _run_alone(kernel, B, op, grads, BatchedBuffers(B, DEV))
    rep = {"kernel": kernel, "x_u8": x_u8, "B": B, "size": size,
           "loops": BC.loop_depths(B, _sms(), BC.kernel_geometry())}
    bad = BC.check_bucket(rep, kernel, grads, op["want"], BC.REDUCTION_BOUND)
    _dump(f"reduction_{kernel}{'_u8' if x_u8 else ''}_B{B}.json", rep)
    assert not bad, (bad, rep)


@pytest.mark.parametrize("size", BC.SIZE_NAMES)
def test_conv2_dgrad_matches_fp64_per_sample(size):
    B = BC.batch_sizes(_sms())[size]
    op = BC.synthetic("conv2_dgrad", B, seed=2000 + B, device=DEV)
    bufs = BatchedBuffers(B + 2, DEV)               # two samples past the batch: the odd last tile must not write there
    bufs.G1.fill_(BC.SENTINEL)
    grads = torch.full((BC.NPAR_ALLOC,), BC.SENTINEL, device=DEV)
    _run_alone("conv2_dgrad", B, op, grads, bufs)
    rep = {"kernel": "conv2_dgrad", "B": B, "size": size, "loops": BC.loop_depths(B, _sms(), BC.kernel_geometry())}
    bad = BC.check_rows(rep, "g1", bufs.G1[:B * 1440].view(B, 1440), op["want"]["G1"], BC.DGRAD_BOUND)
    rep["g1_past_batch_written"] = int((bufs.G1[B * 1440:] != BC.SENTINEL).sum())
    rep["bucket_written"] = int((grads != BC.SENTINEL).sum())
    _dump(f"reduction_conv2_dgrad_B{B}.json", rep)
    assert not bad and rep["g1_past_batch_written"] == 0 and rep["bucket_written"] == 0, (bad, rep)


def _packed(params):
    """The bf16 operand copies bt_pack_weights must have made of ``params`` (layouts in csrc/convnet_batched.cu)."""
    p = {n: params[BC.param_slots(n)] for n in ("conv2.weight", "fc1.weight", "fc1.bias")}
    w2 = p["conv2.weight"].view(20, 10, 25)
    w2k = torch.zeros(32, 28, 16, device=DEV)
    w2k[:20, :25, :10] = w2.permute(0, 2, 1)
    w2r = torch.zeros(25, 16, 64, device=DEV)
    w2r[:, :10, :20] = w2.permute(2, 1, 0)
    w3k = torch.zeros(64, 320, device=DEV)
    w3k[:50] = p["fc1.weight"].view(50, 320)
    b3p = torch.zeros(64, device=DEV)
    b3p[:50] = p["fc1.bias"]
    bf = torch.bfloat16
    return {"W2K": w2k.view(-1).to(bf), "W2R": w2r.view(-1).to(bf), "W3K": w3k.view(-1).to(bf),
            "W3T": w3k.t().contiguous().view(-1).to(bf), "B3P": b3p}


@pytest.mark.parametrize("B", [2048, 4096])
def test_trainer_steps_match_the_model_one_at_a_time(B):
    """Graph-replayed steps and an odd eager tail batch of the bench configuration, each checked on its own: the gradient
    g_k = m_k - mu * m_{k-1} against the model at p_{k-1} with the masks of the step counter the kernels read,
    p_k = p_{k-1} - lr * m_k, and the bf16 weight copies the next step will read."""
    lr, mu, tail = 0.05, 0.5, 1001
    tr = BatchedTrainer(B, lr=lr, momentum=mu, seed=4321, device=DEV, p_drop=0.5, raw_uint8=True)
    g = torch.Generator().manual_seed(B)
    batches = [(torch.randint(0, 256, (n, 1, 28, 28), dtype=torch.uint8, generator=g),
                torch.randint(0, 10, (n,), generator=g)) for n in [B] * 5 + [tail]]
    reports, bad = [], []
    for k, (xu, y) in enumerate(batches):
        tr.stream.synchronize()
        p0, m0 = tr.params.clone(), tr.momentum.clone()
        step0, loss0 = int(tr.step_counter.item()), float(tr.loss_acc[0].item())
        tr.step(xu.pin_memory(), y.pin_memory())
        tr.stream.synchronize()
        n = y.numel()
        rep = {"B": B, "step": k, "batch": n, "path": "eager" if k == 0 or n != B else "graph", "step_counter": step0}
        # the step's gradient from the momentum buffer: m_k = mu * m_{k-1} + g_k
        grad = tr.momentum.double() - mu * m0.double()
        # p_k = p_{k-1} - lr * m_k: one fused multiply-add, so within one fp32 ulp (<= 0.5 observed)
        want_p = p0.double() - float(torch.tensor(lr, dtype=torch.float32)) * tr.momentum.double()
        ulp = torch.finfo(torch.float32).eps * want_p.abs().clamp_min(torch.finfo(torch.float32).tiny)
        rep["sgd_max_ulps"] = float(((tr.params.double() - want_p).abs() / ulp).max())
        if rep["sgd_max_ulps"] > 1.0:
            bad.append(f"step {k}: p_k - (p_(k-1) - lr m_k) is {rep['sgd_max_ulps']:.1f} ulps")
        if int(tr.step_counter.item()) != step0 + 1:
            bad.append(f"step {k}: step counter {int(tr.step_counter.item())} after {step0}")
        for name, want in _packed(tr.params).items():
            if not torch.equal(getattr(tr.bufs, name)[:want.numel()], want):
                bad.append(f"step {k}: {name} is not the bf16 copy of the updated parameters")
        xd, yd = BC.normalize_u8(xu.to(DEV)), y.to(DEV)
        step_t = torch.full((1,), step0, dtype=torch.int64, device=DEV)
        _, _, masks = convnet_loss_and_grads(p0, xd, yd, training=True, seed=tr.seed, step=step_t, sample_base=0,
                                             p_drop=0.5, return_masks=True)
        if not torch.equal(masks.cpu(), SO.dropout_masks(tr.seed, 0, n, step0, 0.5)):
            bad.append(f"step {k}: the per-sample engine's masks differ from the host Philox reference")
        loss =float(tr.loss_acc[0].item()) - loss0
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            bad += [f"step {k}: {b}" for b in BC.compare_pipeline(rep, tr.bufs, p0, xd, yd, masks[:, :20].contiguous(),
                                                                  masks[:, 20:70].contiguous(), grads=grad, loss=loss)[0]]
        reports.append(rep)
    _dump(f"trainer_B{B}.json", reports)
    assert not bad, (bad, reports)
