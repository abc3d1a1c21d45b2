"""Workers of tests/test_gpu_rmsprop.py and tests/test_gpu_rmsprop_multi.py (one process per GPU, ``backend="b200"``):
``DistributedDataParallel`` + ``FlatRMSprop`` through the public API."""
import os

import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from sharded_sgd_gpu_workers import ConvNet, _flat, _replicas_identical

STEPS = 10
# torchvision's recipe (alpha 0.9, eps 0.0316, momentum 0.9), plus the centered variant
OPTS = [dict(lr=1e-3, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4),
        dict(lr=1e-3, alpha=0.99, eps=1e-6, centered=True, weight_decay=0.0)]


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _train(rank, sharded, overlap, grad_dtype, opts, steps=STEPS, resume=None):
    torch.manual_seed(11)
    net = ConvNet().to(_dev())
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=32 << 10, overlap=overlap, grad_dtype=grad_dtype)
    opt = b2.FlatRMSprop(ddp, sharded=sharded, **opts)
    first = 0
    if resume is not None:
        net.load_state_dict(resume["model"])
        opt.load_named_state(net, resume["state"])
        first = opt.steps
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


def w_sharded_ddp(rank, size):
    """Real ranks: sharded FlatRMSprop (the RMSprop instances of the sharded kernel across NVLink) against sharded=False on
    the two-shot all-reduce, bit for bit with fp32 buckets, close with bf16 buckets; identical replicas; a checkpoint round
    trip through named_state across sharded and unsharded runs."""
    os.environ["B200DIST_AR_VARIANT"] = "twoshot"                   # the unsharded arm: the same slices, the same rank order
    for opts in OPTS:
        for overlap in (True, False):
            net_u, opt_u = _train(rank, False, overlap, None, opts)
            net_s, opt_s = _train(rank, True, overlap, None, opts)
            assert opt_s._shard_mode == "kernel" and len(opt_s.buckets) > 2
            assert torch.equal(_flat(net_u), _flat(net_s)), f"{opts} overlap {overlap}: parameters differ from sharded=False"
            _replicas_identical(net_s)
            su, ss = opt_u.named_state(net_u), opt_s.named_state(net_s)
            assert su.keys() == ss.keys() and all(torch.equal(su[k][q], ss[k][q]) for k in su for q in su[k])
        net_b, opt_b = _train(rank, True, True, torch.bfloat16, opts)
        _replicas_identical(net_b)
        net_r, _ = _train(rank, False, True, torch.bfloat16, opts)
        assert torch.allclose(_flat(net_b), _flat(net_r), atol=2e-2, rtol=2e-2)
    opts = OPTS[0]
    net_a, opt_a = _train(rank, True, True, None, opts, steps=5)
    blob = {"model": {k: v.clone() for k, v in net_a.state_dict().items()}, "state": opt_a.named_state(net_a)}
    net_c, opt_c = _train(rank, False, True, None, opts, steps=2, resume=blob)
    blob2 = {"model": {k: v.clone() for k, v in net_c.state_dict().items()}, "state": opt_c.named_state(net_c)}
    net_d, opt_d = _train(rank, True, True, None, opts, steps=3, resume=blob2)
    net_s, _ = _train(rank, True, True, None, opts)
    assert opt_d.steps == STEPS and torch.equal(_flat(net_d), _flat(net_s))
    os.environ.pop("B200DIST_AR_VARIANT", None)
    b2.barrier()


def w_world1(rank, size):
    """One GPU: sharded=True is the unsharded path (rmsprop_flat in step())."""
    for opts in OPTS:
        net_u, opt_u = _train(rank, False, True, None, opts, steps=3)
        net_s, opt_s = _train(rank, True, True, None, opts, steps=3)
        assert opt_s._shard_mode is None and torch.equal(_flat(net_u), _flat(net_s))
        assert opt_s.square_avg_flats[0].numel() == opt_s.buckets[0].numel


def w_resnet(rank, size):
    """A ResNet-18 with SyncBatchNorm under bf16 autocast, torchvision's RMSprop settings: FlatRMSprop's losses stay within
    5% of torch.optim.RMSprop's over six steps, and step() never synchronises the host."""
    from dist_tuto.pth_b200.models.resnet import ResNet18
    dev = _dev()
    hp = dict(lr=1e-3, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-5)
    losses = {}
    for flat in (False, True):
        torch.manual_seed(0)
        net = b2.SyncBatchNorm.convert_sync_batchnorm(ResNet18()).to(dev).to(memory_format=torch.channels_last)
        ddp = b2.DistributedDataParallel(net)
        opt = b2.FlatRMSprop(ddp, **hp) if flat else torch.optim.RMSprop(net.parameters(), **hp)
        g = torch.Generator(device=dev).manual_seed(3)
        out = []
        for it in range(6):
            x = torch.randn(32, 3, 32, 32, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
            t = torch.randint(0, 10, (32,), generator=g, device=dev)
            opt.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(ddp(x), t)
            loss.backward()
            b2.average_gradients(ddp)
            if flat and it > 0:
                torch.cuda.set_sync_debug_mode("error")
                try:
                    opt.step()
                finally:
                    torch.cuda.set_sync_debug_mode(0)
            else:
                opt.step()
            out.append(float(loss))
        ddp.remove_hooks()
        losses[flat] = out
    print(f"ResNet-18 losses, torch.optim.RMSprop {losses[False]}, FlatRMSprop {losses[True]}")
    for a, b_ in zip(losses[False], losses[True]):
        assert abs(a - b_) <= 0.05 * abs(a), losses
    assert losses[True][-1] < losses[True][0], losses
