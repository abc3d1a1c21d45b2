"""FlatSGD (ops/optim.py) against torch.optim.SGD -- the optimizer of the reference loop (train_dist.py:110)."""
import copy

import pytest
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as dist
from dist_tuto.pth_b200.models.resnet import ResNet18


def _steps(model, opt, xs, ys, avg=False):
    losses = []
    for x, y in zip(xs, ys):
        opt.zero_grad()
        loss = F.cross_entropy(model(x), y)
        loss.backward()
        if avg:
            dist.average_gradients(model)
        opt.step()
        losses.append(float(loss.detach()))
    return losses


def _pair(dev, wd, channels_last=False):
    torch.manual_seed(0)
    ref = dist.Net().to(dev).eval()            # eval: dropout off, so both replicas see the same function
    if channels_last:
        ref = ref.to(memory_format=torch.channels_last)
    ours = copy.deepcopy(ref)
    xs = [torch.randn(16, 1, 28, 28, device=dev) for _ in range(4)]
    ys = [torch.randint(0, 10, (16,), device=dev) for _ in range(4)]
    o_ref = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5, weight_decay=wd)
    o_ours = dist.FlatSGD(ours, lr=0.05, momentum=0.5, weight_decay=wd)
    return ref, ours, o_ref, o_ours, xs, ys


@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("channels_last", [False, True])
def test_flat_sgd_matches_torch_sgd_cpu(wd, channels_last):
    ref, ours, o_ref, o_ours, xs, ys = _pair(torch.device("cpu"), wd, channels_last)
    l_ref, l_ours = _steps(ref, o_ref, xs, ys), _steps(ours, o_ours, xs, ys)
    assert l_ref == pytest.approx(l_ours, rel=1e-5)
    for (n, a), b in zip(ref.named_parameters(), ours.parameters()):
        assert torch.allclose(a, b, atol=1e-6), n
    # parameters are views of ONE flat buffer, gradients were re-zeroed by step()
    assert len(o_ours.param_flats) == 1 and o_ours.param_flats[0].numel() >= 21840
    assert float(o_ours.buckets[0].flat.abs().max()) == 0.0
    base = o_ours.param_flats[0].data_ptr()
    assert all(base <= p.data_ptr() < base + 4 * o_ours.param_flats[0].numel() for p in ours.parameters())


def test_flat_sgd_state_dict_roundtrip():
    _, ours, _, opt, xs, ys = _pair(torch.device("cpu"), 0.0)
    _steps(ours, opt, xs[:2], ys[:2])
    sd = opt.state_dict()
    snap = copy.deepcopy(ours.state_dict())
    _steps(ours, opt, xs[2:], ys[2:])
    after = copy.deepcopy(ours.state_dict())
    ours.load_state_dict(snap)
    opt.load_state_dict(sd)
    _steps(ours, opt, xs[2:], ys[2:])
    for k, v in ours.state_dict().items():
        assert torch.equal(v, after[k]), k


def test_flat_sgd_rejects_low_precision_master_weights():
    m = dist.Net().to(torch.bfloat16)
    with pytest.raises(TypeError):
        dist.FlatSGD(m)


@pytest.mark.gpu
@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_flat_sgd_kernel_matches_torch_sgd_gpu(wd):
    dev = torch.device("cuda:0")
    # only the optimizers may differ: both replicas get bit-identical gradients (no TF32, and deterministic cuDNN backward
    # algorithms -- the default ones sum with atomics, and that run-to-run noise compounds over the steps)
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic,
            torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        ref, ours, o_ref, o_ours, xs, ys = _pair(dev, wd)
        l_ref, l_ours = _steps(ref, o_ref, xs, ys), _steps(ours, o_ours, xs, ys)
        assert l_ref == pytest.approx(l_ours, rel=1e-4)
        for (n, a), b in zip(ref.named_parameters(), ours.parameters()):
            assert torch.allclose(a, b, atol=1e-5), n
        assert float(o_ours.buckets[0].flat.abs().max()) == 0.0
    finally:
        (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic,
         torch.backends.cudnn.benchmark) = prev


@pytest.mark.gpu
def test_flat_sgd_with_ddp_buckets_resnet_channels_last_gpu():
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ref = ResNet18(num_classes=10).to(dev).to(memory_format=torch.channels_last)
    ours = copy.deepcopy(ref)
    ddp = dist.DistributedDataParallel(ours, bucket_cap_bytes=4 << 20, broadcast=False)
    o_ref = torch.optim.SGD(ref.parameters(), lr=0.01, momentum=0.5)
    o_ours = dist.FlatSGD(ddp, lr=0.01, momentum=0.5)
    assert len(o_ours.buckets) > 1
    xs = [torch.randn(8, 3, 64, 64, device=dev).to(memory_format=torch.channels_last) for _ in range(3)]
    ys = [torch.randint(0, 10, (8,), device=dev) for _ in range(3)]
    for x, y in zip(xs, ys):
        for model, opt, avg in ((ref, o_ref, False), (ddp, o_ours, True)):
            opt.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(x), y)
            loss.backward()
            if avg:
                dist.average_gradients(ours)
            opt.step()
    for (n, a), b in zip(ref.named_parameters(), ours.parameters()):
        assert torch.allclose(a, b, atol=2e-3, rtol=2e-2), n


def test_flat_sgd_with_a_padded_bucket_buffer():
    """Buckets that live in symmetric memory are padded (64-element granularity): the optimizer must only touch the
    laid-out prefix.  Emulated on CPU by swapping in a longer flat buffer."""
    ref, ours, o_ref, o_ours, xs, ys = _pair(torch.device("cpu"), 0.0)
    gb = o_ours.buckets[0]
    padded = torch.zeros(gb.numel + 40)
    gb.flat = padded
    gb.views = [padded[o:o + p.numel()].view(p.shape) for o, p in zip(gb.offsets, gb.params)]
    for p in gb.params:
        p.grad = None
    gb.attach()
    gb.zero_()
    padded[gb.numel:] = 123.0                      # garbage in the padding must be neither read nor cleared
    l_ref, l_ours = _steps(ref, o_ref, xs, ys), _steps(ours, o_ours, xs, ys)
    assert l_ref == pytest.approx(l_ours, rel=1e-5)
    for a, b in zip(ref.parameters(), ours.parameters()):
        assert torch.allclose(a, b, atol=1e-6)
    assert bool((padded[gb.numel:] == 123.0).all()) and float(padded[:gb.numel].abs().max()) == 0.0
