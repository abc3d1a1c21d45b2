"""Workers of tests/test_gpu_param_groups.py and tests/test_gpu_param_groups_multi.py (one process per GPU,
``backend="b200"``): ``FlatSGD`` / ``FlatAdamW`` with ``param_groups`` through the public API."""
import os

import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from sharded_sgd_gpu_workers import ConvNet, _flat, _replicas_identical


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _no_decay(net):
    nd = [p for p in net.parameters() if p.ndim <= 1]
    return [{"params": nd, "weight_decay": 0.0}, {"params": [list(net.parameters())[-2]], "lr": 3e-3}]


def w_resnet_groups(rank, size):
    """A ResNet-18 with SyncBatchNorm under bf16 autocast and no-decay groups: FlatAdamW's / FlatSGD's losses stay close to
    torch.optim.AdamW's / SGD's with the same groups, step() never synchronises the host, and with zero gradients the
    ndim <= 1 tensors receive no decay while the others do."""
    from dist_tuto.pth_b200.models.resnet import ResNet18
    dev = _dev()
    for kind in ("adamw", "sgd"):
        hp = dict(lr=1e-3, weight_decay=0.05) if kind == "adamw" else dict(lr=0.02, momentum=0.9, weight_decay=5e-3)
        losses = {}
        for flat in (False, True):
            torch.manual_seed(0)
            net = b2.SyncBatchNorm.convert_sync_batchnorm(ResNet18()).to(dev).to(memory_format=torch.channels_last)
            ddp = b2.DistributedDataParallel(net)
            groups = _no_decay(net)
            if flat:
                opt = (b2.FlatAdamW if kind == "adamw" else b2.FlatSGD)(ddp, param_groups=groups, **hp)
                assert all(m is not None for m in opt._maps)
            else:
                rest = [p for p in net.parameters() if not any(p is q for g in groups for q in g["params"])]
                opt = (torch.optim.AdamW if kind == "adamw" else torch.optim.SGD)(groups + [{"params": rest}], **hp)
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
        for a, b_ in zip(losses[False], losses[True]):
            assert abs(a - b_) <= 0.05 * abs(a), (kind, losses)
        assert losses[True][-1] < losses[True][0], (kind, losses)
        # a first update from zero gradients (zero state) is the decay alone: only the decayed tensors move
        torch.manual_seed(0)
        net = ResNet18().to(dev)
        ddp = b2.DistributedDataParallel(net)
        opt = (b2.FlatAdamW if kind == "adamw" else b2.FlatSGD)(ddp, param_groups=_no_decay(net), **hp)
        before = {n: p.detach().clone() for n, p in net.named_parameters()}
        opt.zero_grad()
        b2.average_gradients(ddp)
        opt.step()
        for n, p in net.named_parameters():
            assert torch.equal(p, before[n]) == (p.ndim <= 1 or not before[n].any()), (kind, n)
        ddp.remove_hooks()


def _train(rank, Flat, hp, sharded, steps=6):
    torch.manual_seed(11)
    net = ConvNet().to(_dev())
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=32 << 10, overlap=True)
    opt = Flat(ddp, sharded=sharded, param_groups=_no_decay(net), **hp)
    for it in range(steps):
        g = torch.Generator().manual_seed(100 * it + rank)
        x, y = torch.randn(8, 3, 16, 16, generator=g).to(_dev()), torch.randint(0, 10, (8,), generator=g).to(_dev())
        opt.zero_grad()
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        opt.step()
    torch.cuda.synchronize()
    ddp.remove_hooks()
    return net, opt


def w_sharded_groups_ddp(rank, size):
    """Real ranks: grouped sharded FlatSGD / FlatAdamW (fp32 buckets) equal grouped unsharded bit for bit on the two-shot
    all-reduce, and the replicas are identical."""
    os.environ["B200DIST_AR_VARIANT"] = "twoshot"
    for Flat, hp in ((b2.FlatSGD, dict(lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True)),
                     (b2.FlatAdamW, dict(lr=2e-3, weight_decay=0.05))):
        net_u, _ = _train(rank, Flat, hp, False)
        net_s, opt_s = _train(rank, Flat, hp, True)
        assert opt_s._shard_mode == "kernel" and len(opt_s.buckets) > 2
        assert torch.equal(_flat(net_u), _flat(net_s)), Flat.__name__
        _replicas_identical(net_s)
    os.environ.pop("B200DIST_AR_VARIANT", None)
    b2.barrier()
