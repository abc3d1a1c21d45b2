"""The fp32 model of the batched tensor-core engine (ops/batched_reference.py) against autograd of the reference Net.

GPU tests compare the sm_90a kernels with that model at a tight tolerance; this CPU test makes sure the model itself
(hand-written backward, im2col/col2im index conventions, dropout scaling) is the network of train_dist.py:53-71."""
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops import batched_reference as R
from dist_tuto.pth_b200.ops.convnet_fused import pack_params, unpack_params


def _oracle(net, x, y, m2, dm):
    """train_dist.py Net.forward with explicit dropout masks, autograd gradients."""
    h = F.relu(F.max_pool2d(net.conv1(x), 2))
    h = F.relu(F.max_pool2d(net.conv2(h) * m2.view(-1, 20, 1, 1), 2))
    h = F.relu(net.fc1(h.view(-1, 320))) * dm
    logp = F.log_softmax(net.fc2(h), dim=1)
    loss = F.nll_loss(logp, y)
    net.zero_grad()
    loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in net.named_parameters()}


def _setup(B, seed, training):
    torch.manual_seed(seed)
    net = b2.Net()
    x = torch.randn(B, 1, 28, 28)
    y = torch.randint(0, 10, (B,))
    if training:
        m2 = (torch.rand(B, 20) >= 0.5).float() * 2.0
        dm = (torch.rand(B, 50) >= 0.5).float() * 2.0
    else:
        m2, dm = torch.ones(B, 20), torch.ones(B, 50)
    return net, x, y, m2, dm


def test_unrounded_model_is_the_reference_network():
    for training in (False, True):
        net, x, y, m2, dm = _setup(16, 3, training)
        loss, grads = _oracle(net, x, y, m2, dm)
        out = R.forward_backward(pack_params(net), x, y, m2, dm, emulate_bf16=False)
        assert torch.allclose(out["loss"], loss, atol=1e-6)
        mine = unpack_params(out["grads"])
        for n, g in grads.items():
            assert torch.allclose(mine[n], g, atol=2e-6, rtol=1e-4), (n, training, float((mine[n] - g).abs().max()))


def test_overrides_with_the_models_own_values_change_nothing():
    """Feeding the model's own conv1 output and codes, conv2 codes, P2 and fc1 output back through the overrides (as the
    GPU tests do with the engine's) must reproduce every output bit for bit."""
    for training in (False, True):
        net, x, y, m2, dm = _setup(16, 7, training)
        params = pack_params(net)
        out = R.forward_backward(params, x, y, m2, dm)
        again = R.forward_backward(params, x, y, m2, dm, p1_override=out["p1"],
                                   a1_override=R.pool_codes(out["a1"], out["m1"], 24),
                                   a2_override=R.pool_codes(out["a2"], out["mp2"], 8), p2_override=out["p2"],
                                   hrelu_override=out["hrelu"])
        assert bool(((R.pool_codes(out["a2"], out["mp2"], 8) & 4) != 0).any())      # the dead bit is exercised
        for k, v in out.items():
            if k != "named":
                assert torch.equal(again[k], v), (k, training)


def test_bf16_emulation_stays_within_bf16_accuracy():
    net, x, y, m2, dm = _setup(64, 5, True)
    loss, grads = _oracle(net, x, y, m2, dm)
    out = R.forward_backward(pack_params(net), x, y, m2, dm, emulate_bf16=True)
    assert abs(float(out["loss"]) - float(loss)) < 2e-2 * abs(float(loss))
    mine = unpack_params(out["grads"])
    for n, g in grads.items():
        rel = float((mine[n] - g).norm() / g.norm().clamp_min(1e-12))
        assert rel < 0.1, (n, rel)            # bf16 operands + a few pool-argmax flips; indexing bugs give O(1)
