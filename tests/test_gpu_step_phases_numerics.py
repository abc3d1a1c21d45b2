"""GPU-single tier: one step of the one-CTA-per-sample kernel (csrc/convnet.cu) in the configuration the benchmark runs --
batch 128, conv2.weight staged from the optimizer's aux copy, uint8 input normalised in the kernel, per-CTA slots and
per-sample fc1 factors -- against an fp64 oracle that applies the dropout scales the kernel reports (mask_out).

p = 0.5 drops about half of the conv2 channels, so the conv2 data-gradient warps skip channels; p = 0 keeps every channel,
which gives every such warp its full share of work."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

B = 128


@pytest.fixture(scope="module")
def dev():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda", 0)


def _masked_forward(net, x, m2, mh):
    h = F.relu(F.max_pool2d(net.conv1(x), 2))
    h = net.conv2(h) * m2[:, :, None, None]
    h = F.relu(F.max_pool2d(h, 2)).reshape(-1, 320)
    h = F.relu(net.fc1(h)) * mh
    return F.log_softmax(net.fc2(h), dim=1)


def _step(tr, xu, y, p_drop, input_ready):
    """One backward step on the slot + factor path; returns (flat local gradient, loss, dropout scales)."""
    from dist_tuto.pth_b200.ops.convnet_fused import FAC_STRIDE, NPAR_ALLOC
    dev = xu.device
    slots = torch.zeros(B * NPAR_ALLOC, device=dev)
    factors = torch.zeros(B * FAC_STRIDE, device=dev)
    masks = torch.zeros(B * 70, device=dev)
    step = torch.tensor([5], dtype=torch.int64, device=dev)
    tr.C.convnet_step(tr.params, tr.grads, xu, y, tr.loss_acc, None, masks, step, 29, 0, True, 1.0 / B, p_drop, 0,
                      tr.grad_stride, 1, tr.aux, None, slots, factors, input_ready=input_ready)
    torch.cuda.synchronize()
    s = slots.view(B, NPAR_ALLOC).double()
    g = s[:, :21848].sum(0)
    fac = factors.view(B, FAC_STRIDE).double()
    g[5284:21284] = torch.einsum("bj,bi->ji", fac[:, :50], fac[:, 64:384]).reshape(-1)   # sum_b dh_b (x) p2_b
    return g, float(s[:, 21848].sum()), masks.view(B, 70)


@pytest.mark.parametrize("p_drop", [0.5, 0.0])
def test_bsz128_step_gradients_match_fp64_masked_oracle(dev, p_drop):
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer, unpack_params
    torch.manual_seed(31)
    net = Net(p_drop=p_drop).to(dev)
    tr = FusedTrainer(B, seed=29, device=dev, p_drop=p_drop, raw_uint8=True, init_from=net)
    g = torch.Generator(device="cpu").manual_seed(32)
    xu = torch.randint(0, 256, (B, 1, 28, 28), dtype=torch.uint8, generator=g).to(dev)
    y = torch.randint(0, 10, (B,), generator=g).to(dev)

    grads, loss, masks = _step(tr, xu, y, p_drop, input_ready=True)
    if p_drop > 0:
        assert 0.3 < float((masks[:, :20] > 0).float().mean()) < 0.7
    else:
        assert bool((masks == 1.0).all())

    net64 = net.double()
    x64 = (xu.double() / 255.0 - 0.1307) / 0.3081
    ref_loss = F.nll_loss(_masked_forward(net64, x64, masks[:, :20].double(), masks[:, 20:].double()), y)
    ref_loss.backward()
    assert abs(loss - float(ref_loss)) < 1e-4 * max(1.0, abs(float(ref_loss)))
    views = unpack_params(grads)
    errs = {}
    for name, p in net64.named_parameters():
        scale = p.grad.abs().max().clamp_min(1e-9)
        errs[name] = float((views[name] - p.grad).abs().max() / scale)
    assert max(errs.values()) < 1e-3, errs

    # loading the batch after griddepcontrol.wait instead of before it computes the same bits
    grads_late, loss_late, masks_late = _step(tr, xu, y, p_drop, input_ready=False)
    assert torch.equal(grads_late, grads) and loss_late == loss and torch.equal(masks_late, masks)
