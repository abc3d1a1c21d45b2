"""GPU tier: the forward-only evaluation kernel (csrc/convnet_eval.cu) against an fp64 oracle, its determinism, and
evaluation through the trainers and train() without disturbing training."""
import pytest
import torch

import dist_tuto.pth_b200 as b2
import eval_workers as W
from dist_tuto.pth_b200.data import SyntheticMNIST

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

TEST_SEED = 777


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _oracle(net, x, y, mean, std):
    """Net.eval() in float64 on CPU: log-probs, nll sum, #correct, and the mask of samples whose top-2 logit margin is
    below 1e-4 (their argmax may go either way in fp32)."""
    net = net.double().eval()
    xd = ((x.double() / 255.0 - mean) / std).unsqueeze(1) if x.dtype == torch.uint8 else x.double()
    with torch.no_grad():
        logp = net(xd)
    top2 = logp.topk(2, dim=1).values              # log_softmax shifts all logits of a sample alike: same margin
    near = (top2[:, 0] - top2[:, 1]) < 1e-4
    right = logp.argmax(1) == y
    return logp, float(-logp.gather(1, y[:, None]).sum()), right, near


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("n", [1, 5, 131, 1000, 10007])
def test_eval_kernel_matches_fp64_oracle(dev, n, u8):
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    from dist_tuto.pth_b200.ops.convnet_fused import pack_params
    g = torch.Generator().manual_seed(n * 2 + u8)
    torch.manual_seed(n)
    net = Net()
    # a non-MNIST normalisation on one case shows the kernel uses the mean / std it is given
    mean, std = (0.5, 0.25) if (u8 and n == 131) else (0.1307, 0.3081)
    x = torch.randint(0, 256, (n, 28, 28), generator=g, dtype=torch.uint8) if u8 else torch.randn(n, 1, 28, 28, generator=g)
    y = torch.randint(0, 10, (n,), generator=g)
    logp = torch.empty(n, 10, device=dev)
    res = convnet_evaluate(pack_params(net, dev), x.to(dev), y.to(dev), mean, std, out_logp=logp).tolist()
    ref_logp, ref_nll, right, near = _oracle(net, x, y, mean, std)
    assert float((logp.cpu().double() - ref_logp).abs().max()) < 2e-4
    assert abs(res[0] - ref_nll) <= 1e-5 * abs(ref_nll), (res[0], ref_nll)
    assert res[2] == n
    sure = int((right & ~near).sum())
    assert sure <= res[1] <= sure + int(near.sum()), (res[1], sure, int(near.sum()))


def test_eval_kernel_is_bit_reproducible_and_empty_input_gives_zeros(dev):
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    from dist_tuto.pth_b200.ops.convnet_fused import pack_params
    torch.manual_seed(3)
    params = pack_params(Net(), dev)
    ds = SyntheticMNIST(n=60000, seed=TEST_SEED)
    x, y = ds.images.to(dev), ds.labels.to(dev)
    outs = []
    for _ in range(2):
        lp = torch.empty(60000, 10, device=dev)
        outs.append((convnet_evaluate(params, x, y, ds.mean, ds.std, out_logp=lp).cpu(), lp.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][0][2].item() == 60000
    empty = convnet_evaluate(params, x[:0], y[:0])
    assert empty.tolist() == [0.0, 0.0, 0.0]


def _train_batches(k, seed, raw=False):
    ds = SyntheticMNIST(n=128 * k, seed=seed)
    out = []
    for i in range(k):
        idx = torch.arange(i * 128, (i + 1) * 128)
        x, y = (ds.images[idx].unsqueeze(1).contiguous(), ds.labels[idx]) if raw else ds.gather(idx)
        out.append((x.pin_memory(), y.pin_memory()))
    return out


def _state(tr):
    torch.cuda.synchronize()
    return (tr.params.clone(), tr.momentum.clone(), tr.loss_acc.clone(), int(tr.step_counter.item()))


def _same(a, b):
    return all(torch.equal(u, v) for u, v in zip(a[:3], b[:3])) and a[3] == b[3]


def test_fused_trainer_evaluate_leaves_graph_training_untouched(dev):
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    test = SyntheticMNIST(n=3001, seed=TEST_SEED)
    batches = _train_batches(8, seed=11)
    states, result = [], None
    for with_eval in (False, True):
        tr = FusedTrainer(128, lr=0.05, seed=4, device=dev)
        for x, y in batches[:4]:
            tr.step(x, y)
        if with_eval:
            result = tr.evaluate(test)
            torch.cuda.synchronize()
            ref = convnet_evaluate(tr.params, test.images.to(dev), test.labels.to(dev), test.mean, test.std).tolist()
            assert result == {"loss": ref[0] / 3001, "accuracy": int(ref[1]) / 3001, "correct": int(ref[1]), "n": 3001}
            assert tr.training
        for x, y in batches[4:]:
            tr.step(x, y)
        states.append(_state(tr))
    assert states[0][3] == 8 and _same(states[0], states[1])


def test_fused_trainer_evaluate_leaves_native_training_untouched(dev):
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    ds, test = SyntheticMNIST(n=128 * 10, seed=12), SyntheticMNIST(n=2000, seed=TEST_SEED)
    states = []
    for with_eval in (False, True):
        loader = D.NativeBatchLoader(D.Partition(ds, list(range(len(ds)))), 128, seed=9, raw_uint8=True, pin_memory=True,
                                     num_buffers=8)
        tr = FusedTrainer(128, lr=0.05, seed=4, device=dev, raw_uint8=True)
        done, _ = tr.run_native(loader, max_steps=4)
        assert done == 4
        mid = _state(tr)
        if with_eval:
            r = tr.evaluate(test)
            ref = convnet_evaluate(tr.params, test.images.to(dev), test.labels.to(dev), test.mean, test.std).tolist()
            assert r["correct"] == int(ref[1]) and r["loss"] == ref[0] / 2000
        done, _ = tr.run_native(loader, max_steps=None, new_epoch=False)     # the rest of the same epoch
        assert done == 6
        states.append((mid, _state(tr)))
    assert _same(states[0][0], states[1][0]) and _same(states[0][1], states[1][1])


def test_batched_trainer_evaluate_equals_functional(dev):
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    ds, test = SyntheticMNIST(n=2048 * 3, seed=13), SyntheticMNIST(n=4099, seed=TEST_SEED)
    tr = BatchedTrainer(2048, lr=0.05, seed=4, device=dev)
    for i in range(3):
        x, y = ds.gather(torch.arange(i * 2048, (i + 1) * 2048))
        tr.step(x.pin_memory(), y.pin_memory())
    r = tr.evaluate(test)
    torch.cuda.synchronize()
    ref = convnet_evaluate(tr.params, test.images.to(dev), test.labels.to(dev), test.mean, test.std).tolist()
    assert r == {"loss": ref[0] / 4099, "accuracy": int(ref[1]) / 4099, "correct": int(ref[1]), "n": 4099}
    assert r == b2.evaluate(tr, test)


def test_evaluate_net_on_cuda_goes_through_the_kernel(dev):
    from dist_tuto.pth_b200.models.convnet import Net
    torch.manual_seed(6)
    net = Net()
    test = SyntheticMNIST(n=1500, seed=TEST_SEED)
    cpu = b2.evaluate(net, test)
    gpu = b2.evaluate(net.to(dev), test)
    assert gpu["n"] == cpu["n"] == 1500
    assert abs(gpu["loss"] - cpu["loss"]) <= 1e-5 * abs(cpu["loss"]) and abs(gpu["correct"] - cpu["correct"]) <= 2


def test_train_fused_world1_with_evaluation(dev):
    ds, test = SyntheticMNIST(n=60032), SyntheticMNIST(n=10000, seed=TEST_SEED)    # 60032 = 469 full batches of 128
    outs = []
    for eval_ds in (None, test):
        out = {}

        def fn(rank, size):
            out.update(b2.train(rank, size, b2.TrainConfig(epochs=1, dataset=ds, engine="fused", eval_dataset=eval_ds,
                                                           log=lambda *a: None)))

        b2.init_processes(0, 1, fn, backend="b200", master_port=b2.find_free_port())
        outs.append(out)
    off, on = outs
    assert off["eval"] == [] and on["steps"] == off["steps"] == 469
    assert on["loss"] == off["loss"]
    assert len(on["eval"]) == 1 and on["eval"][0]["epoch"] == 0 and on["eval"][0]["n"] == 10000
    assert on["eval"][0]["accuracy"] >= 0.95, on["eval"]
    assert on["eval_seconds"] > 0.0


@pytest.mark.multigpu
def test_fused_evaluate_world2_equals_one_process():
    b2.launch(W.w_fused_evaluate_world, size=2, backend="b200", join_timeout_s=600)
