"""GPU-single tier: the one-CTA-per-sample step kernel (csrc/convnet.cu) at the batch where it is the flagship path (128
samples, no clusters), trained through the optimizer kernel, and with CTAs that carry several samples each."""
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


def test_fused_trainer_bsz128_matches_torch_sgd(dev):
    """Six momentum-SGD steps at batch 128 (one CTA per sample, conv2.weight staged from the optimizer's aux copy) == torch."""
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer, unpack_params
    torch.manual_seed(11)
    ref = Net(p_drop=0.0).to(dev)
    tr = FusedTrainer(128, lr=0.05, momentum=0.5, seed=11, device=dev, p_drop=0.0, init_from=ref)
    assert tr.cluster == 1
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    losses = []
    for i in range(6):
        x, y = _batch(dev, 128, seed=100 + i)
        tr.step(x.cpu().pin_memory(), y.cpu().pin_memory())
        opt.zero_grad()
        loss = F.nll_loss(ref(x), y)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    got = tr.pop_loss_sum()
    assert abs(got - sum(losses)) < 1e-3 * max(1.0, abs(sum(losses)))
    views = unpack_params(tr.params)
    for name, p in ref.named_parameters():
        assert torch.allclose(views[name], p.detach(), atol=2e-4, rtol=1e-3), name
    x, _ = _batch(dev, 8, seed=999)
    assert torch.allclose(tr.eval()(x), tr.to_module().to(dev).eval()(x), atol=2e-4)


def test_native_executor_bsz128_matches_python_loop(dev):
    """C++ StepExecutor == stepping the same loader from Python, at batch 128 (one CTA per sample)."""
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    ds = D.SyntheticMNIST(n=1000, seed=2)                 # 1000 = 7 x 128 + 104 -> the short tail batch too
    part = D.Partition(ds, list(range(1000)))
    res = []
    for native in (True, False):
        loader = D.NativeBatchLoader(part, 128, seed=9, raw_uint8=True, pin_memory=True, num_buffers=8)
        tr = FusedTrainer(128, lr=0.05, seed=3, device=dev, p_drop=0.5, raw_uint8=True)
        if native:
            done, finished = tr.run_native(loader)
            assert done == 8 and finished
        else:
            n = 0
            for x, y in loader:
                tr.step(x, y)
                n += 1
            assert n == 8
        torch.cuda.synchronize()
        res.append((tr.params.clone(), tr.pop_loss_sum(), int(tr.step_counter.item())))
    assert res[0][2] == res[1][2] == 8
    assert abs(res[0][1] - res[1][1]) < 1e-3 * abs(res[1][1])
    assert torch.allclose(res[0][0], res[1][0], atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("det", [False, True])
def test_ctas_carrying_several_samples_give_the_same_gradients(dev, det):
    """The fc1.weight gradient leaves the kernel per sample (no per-CTA accumulator): 64 samples on 13 CTAs must give the
    gradient of 64 samples on 64 CTAs, both with red.add into the bucket and with per-CTA deterministic slots."""
    from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC, FusedTrainer
    tr = FusedTrainer(64, seed=5, device=dev, p_drop=0.5)
    C = tr.C
    x, y = _batch(dev, 64, seed=21)
    step = torch.zeros(1, dtype=torch.int64, device=dev)

    def grads(max_ctas):
        g = torch.zeros(NPAR_ALLOC, dtype=torch.float32, device=dev)
        acc = torch.zeros(2, dtype=torch.float32, device=dev)
        slots = torch.zeros(tr.sms * NPAR_ALLOC, dtype=torch.float32, device=dev) if det else None
        C.convnet_step(tr.params, g, x, y, acc, None, None, step, 7, 0, True, 1.0 / 64, 0.5, max_ctas, 0, 1, tr.aux, None, slots)
        if det:
            C.det_reduce(slots, max_ctas if max_ctas > 0 else 64, g, step, 0, acc)
        torch.cuda.synchronize()
        return g, acc

    (g_all, acc_all), (g_few, acc_few) = grads(0), grads(13)
    assert float(g_all.abs().max()) > 0
    assert torch.allclose(g_few, g_all, atol=1e-6, rtol=1e-4), (g_few - g_all).abs().max()
    assert torch.allclose(acc_few, acc_all, atol=1e-5, rtol=1e-5)
