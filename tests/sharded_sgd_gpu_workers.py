"""Workers of tests/test_gpu_sharded_sgd_multi.py (one process per GPU, ``backend="b200"``): ``DistributedDataParallel`` +
``FlatSGD(sharded=True)`` through the public API on a small conv model."""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2

STEPS = 10
OPTS = dict(lr=0.05, momentum=0.9, weight_decay=1e-3, nesterov=True)


class ConvNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1, self.conv2 = nn.Conv2d(3, 16, 3, padding=1), nn.Conv2d(16, 32, 3, padding=1)
        self.fc1, self.fc2 = nn.Linear(32 * 4 * 4, 67), nn.Linear(67, 10)

    def forward(self, x):
        x = F.max_pool2d(F.relu(self.conv1(x)), 2)
        x = F.max_pool2d(F.relu(self.conv2(x)), 2)
        return self.fc2(F.relu(self.fc1(x.flatten(1))))


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _train(rank, sharded, overlap, grad_dtype, steps=STEPS, resume=None):
    torch.manual_seed(11)
    net = ConvNet().to(_dev())
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=32 << 10, overlap=overlap, grad_dtype=grad_dtype)
    opt = b2.FlatSGD(ddp, sharded=sharded, **OPTS)
    first = 0
    if resume is not None:
        net.load_state_dict(resume["model"])
        opt.load_named_momentum(net, resume["momentum"])
        opt.steps = first = resume["steps"]
    for it in range(first, first + steps):
        g = torch.Generator().manual_seed(100 * it + rank)
        x, y = torch.randn(8, 3, 16, 16, generator=g).to(_dev()), torch.randint(0, 10, (8,), generator=g).to(_dev())
        opt.zero_grad()
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        opt.step()
    torch.cuda.synchronize()
    ddp.remove_hooks()
    return net, opt


def _flat(net):
    return torch.cat([p.detach().reshape(-1) for p in net.parameters()])


def _replicas_identical(net):
    flat = _flat(net)
    other = flat.clone()
    b2.broadcast(other, src=0)
    assert torch.equal(flat, other)


def w_sharded_ddp(rank, size):
    os.environ["B200DIST_AR_VARIANT"] = "twoshot"                   # the unsharded arm: the same slices, the same rank order
    for overlap in (True, False):
        net_u, opt_u = _train(rank, False, overlap, None)
        net_s, opt_s = _train(rank, True, overlap, None)
        assert opt_s._shard_mode == "kernel" and len(opt_s.buckets) > 2
        assert torch.equal(_flat(net_u), _flat(net_s)), f"overlap {overlap}: fp32 parameters differ from sharded=False"
        _replicas_identical(net_s)
        for k, gb in enumerate(opt_s.buckets):
            assert opt_s.momentum_flats[k].numel() * size < gb.flat.numel() + 4 * size + 64 and not gb.flat.any()
        nu, ns = opt_u.named_momentum(net_u), opt_s.named_momentum(net_s)
        assert nu.keys() == ns.keys() and all(torch.equal(nu[k], ns[k]) for k in nu)
    # bf16 gradient buckets: fp32 accumulation, the update from the unrounded mean; close to the bf16 all-reduce path
    for overlap in (True, False):
        net_b, opt_b = _train(rank, True, overlap, torch.bfloat16)
        assert opt_b._shard_mode == "kernel"
        _replicas_identical(net_b)
        net_r, _ = _train(rank, False, overlap, torch.bfloat16)
        assert torch.allclose(_flat(net_b), _flat(net_r), atol=2e-2, rtol=2e-2)
    # checkpoint round trip: 5 + 5 steps through the per-name momentum, sharded -> unsharded -> sharded
    net_a, opt_a = _train(rank, True, True, None, steps=5)
    blob = {"model": {k: v.clone() for k, v in net_a.state_dict().items()}, "momentum": opt_a.named_momentum(net_a),
            "steps": opt_a.steps}
    net_c, opt_c = _train(rank, False, True, None, steps=2, resume=blob)
    blob2 = {"model": {k: v.clone() for k, v in net_c.state_dict().items()}, "momentum": opt_c.named_momentum(net_c),
             "steps": opt_c.steps}
    net_d, opt_d = _train(rank, True, True, None, steps=3, resume=blob2)
    assert opt_d.steps == STEPS and torch.equal(_flat(net_d), _flat(net_s))
    os.environ.pop("B200DIST_AR_VARIANT", None)
    b2.barrier()


def w_world1(rank, size):
    """One GPU: sharded=True is the unsharded path (sgd_flat in step())."""
    net_u, opt_u = _train(rank, False, True, None, steps=3)
    net_s, opt_s = _train(rank, True, True, None, steps=3)
    assert opt_s._shard_mode is None and torch.equal(_flat(net_u), _flat(net_s))
    assert opt_s.momentum_flats[0].numel() == opt_s.buckets[0].numel
