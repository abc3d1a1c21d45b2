"""GPU-single tier: the one-GPU step without atomics -- per-CTA slots and per-sample fc1 factors from the step kernel
(csrc/convnet.cu), summed in a fixed order by the optimizer kernel reduce_sgd (csrc/sgd.cu, csrc/convnet_reduce.cuh)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.fixture(scope="module")
def dev():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda", 0)


def _batch(dev, B, seed=1):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, 1, 28, 28, generator=g).to(dev)
    y = torch.randint(0, 10, (B,), generator=g).to(dev)
    return x, y


def test_default_trainer_bsz128_is_bit_reproducible(dev):
    """Two runs of 12 dropout steps at batch 128 with the default trainer (no `deterministic` flag) are bit-equal."""
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    batches = [_batch(dev, 128, seed=300 + i) for i in range(12)]
    res = []
    for _ in range(2):
        tr = FusedTrainer(128, lr=0.05, momentum=0.5, seed=17, device=dev, p_drop=0.5)
        assert tr.cluster == 1 and tr.grad_slots is not None
        for x, y in batches:
            tr.step(x.cpu().pin_memory(), y.cpu().pin_memory())
        tr.sync_lag(0)
        torch.cuda.synchronize()
        res.append((tr.params.clone(), tr.momentum.clone(), tr.loss_acc.clone()))
    assert float(res[0][1].abs().max()) > 0
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)


def test_ctas_carrying_several_samples_match_torch_sgd(dev):
    """Batch 200 on 64 step CTAs (so CTAs carry 3-4 samples and the factor GEMM takes two passes of 128 samples), three
    momentum-SGD steps through reduce_sgd == Net autograd + torch SGD."""
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_fused import FAC_STRIDE, NPAR_ALLOC, FusedTrainer, unpack_params
    torch.manual_seed(13)
    ref = Net(p_drop=0.0).to(dev)
    tr = FusedTrainer(200, lr=0.05, momentum=0.5, seed=13, device=dev, p_drop=0.0, init_from=ref)
    C = tr.C
    B, n = 200, 64
    slots = torch.full((n * NPAR_ALLOC,), float("nan"), device=dev)      # the fc1.weight range of a slot is never read
    factors = torch.zeros(B * FAC_STRIDE, device=dev)
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    losses = []
    for i in range(3):
        x, y = _batch(dev, B, seed=400 + i)
        C.convnet_step(tr.params, tr.grads, x, y, tr.loss_acc, None, None, tr.step_counter, 13, 0, True, 1.0 / B, 0.0, n,
                       tr.grad_stride, 1, tr.aux, None, slots, factors)
        C.reduce_sgd(slots, n, factors, B, tr.params, tr.momentum, tr.step_counter, tr.done_counter, 0.05, 0.5, tr.aux, tr.loss_acc)
        opt.zero_grad()
        loss = F.nll_loss(ref(x), y)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    torch.cuda.synchronize()
    assert int(tr.step_counter.item()) == 3
    assert abs(float(tr.loss_acc[0]) - sum(losses)) < 1e-3 * max(1.0, abs(sum(losses)))
    views = unpack_params(tr.params)
    for name, p in ref.named_parameters():
        assert torch.allclose(views[name], p.detach(), atol=2e-4, rtol=1e-3), name
    assert float(tr.grads.abs().max()) == 0.0            # no bucket on this path


def test_native_executor_bucket_steps_between_slot_steps(dev):
    """Batch 544 (> 4 CTAs per SM): the C++ executor runs the full batches on the bucket path while the short tail batch of
    every epoch takes the slots path eagerly.  The bucket step after a slots step must find its bucket zeroed; two epochs
    through run_native == the same batches stepped from Python (slots path throughout)."""
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    ds = D.SyntheticMNIST(n=2 * 544 + 100, seed=4)
    part = D.Partition(ds, list(range(len(ds))))
    res = []
    for native in (True, False):
        loader = D.NativeBatchLoader(part, 544, seed=9, raw_uint8=True, pin_memory=True, num_buffers=8)
        tr = FusedTrainer(544, lr=0.05, seed=3, device=dev, p_drop=0.5, raw_uint8=True)
        assert tr._native_slots() == (None, None)
        for _ in range(2):
            if native:
                done, finished = tr.run_native(loader)
                assert done == 3 and finished
            else:
                n = 0
                for x, y in loader:
                    tr.step(x, y)
                    n += 1
                assert n == 3
        torch.cuda.synchronize()
        res.append((tr.params.clone(), tr.pop_loss_sum(), int(tr.step_counter.item())))
    assert res[0][2] == res[1][2] == 6
    assert abs(res[0][1] - res[1][1]) < 1e-3 * abs(res[1][1])
    assert torch.allclose(res[0][0], res[1][0], atol=1e-5, rtol=1e-4)
