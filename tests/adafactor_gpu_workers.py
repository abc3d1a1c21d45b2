"""Workers of tests/test_gpu_adafactor.py and tests/test_gpu_adafactor_multi.py (one process per GPU, ``backend="b200"``):
``DistributedDataParallel`` + ``FlatAdafactor`` through the public API."""
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from sharded_sgd_gpu_workers import ConvNet, _flat, _replicas_identical

HP = dict(lr=1e-2, beta2_decay=-0.8, eps=(None, 1e-3), d=1.0, weight_decay=1e-3)


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _batch(it, rank):
    g = torch.Generator().manual_seed(100 * it + rank)
    return torch.randn(8, 3, 16, 16, generator=g).to(_dev()), torch.randint(0, 10, (8,), generator=g).to(_dev())


def w_ddp(rank, size):
    """Real ranks: the replicas stay bit-identical, and the result equals a FlatAdafactor over one non-symmetric bucket of a
    copy of the model fed the averaged gradients (every sum of the update is per tensor, so the bucket layout does not
    matter)."""
    from dist_tuto.pth_b200.parallel.ddp import GradBucket
    torch.manual_seed(11)
    net = ConvNet().to(_dev()).to(memory_format=torch.channels_last)
    torch.manual_seed(11)
    ref = ConvNet().to(_dev()).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=32 << 10)
    opt = b2.FlatAdafactor(ddp, **HP)
    names = {id(p): n for n, p in net.named_parameters()}
    grads = []
    for it in range(6):
        x, y = _batch(it, rank)
        opt.zero_grad()
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        grads.append({names[id(p)]: gv.clone() for gb in ddp.buckets for p, gv in zip(gb.params, gb.views)})
        opt.step()
    torch.cuda.synchronize()
    _replicas_identical(net)
    gb = GradBucket(list(ref.parameters()), symmetric=False)
    object.__setattr__(ref, "_grad_bucket", gb)
    ropt = b2.FlatAdafactor(ref, **HP)
    rnames = {id(p): n for n, p in ref.named_parameters()}
    for gs in grads:
        for p, gv in zip(gb.params, gb.views):
            gv.copy_(gs[rnames[id(p)]])
        ropt.step()
    torch.cuda.synchronize()
    assert torch.equal(_flat(ref), _flat(net)), "one bucket fed the averaged gradients differs"
    ddp.remove_hooks()
    b2.barrier()


def w_resnet(rank, size):
    """A ResNet-18 with SyncBatchNorm under bf16 autocast, channels_last: FlatAdafactor's losses stay within 5% of
    torch.optim.Adafactor's over six steps, and step() never synchronises the host."""
    from dist_tuto.pth_b200.models.resnet import ResNet18
    dev = _dev()
    hp = dict(lr=1e-2, weight_decay=1e-4)
    losses = {}
    for flat in (False, True):
        torch.manual_seed(0)
        net = b2.SyncBatchNorm.convert_sync_batchnorm(ResNet18()).to(dev).to(memory_format=torch.channels_last)
        ddp = b2.DistributedDataParallel(net)
        opt = b2.FlatAdafactor(ddp, **hp) if flat else torch.optim.Adafactor(net.parameters(), foreach=False, **hp)
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
    print(f"ResNet-18 losses, torch.optim.Adafactor {losses[False]}, FlatAdafactor {losses[True]}")
    for a, b_ in zip(losses[False], losses[True]):
        assert abs(a - b_) <= 0.05 * abs(a), losses
    assert losses[True][-1] < losses[True][0], losses


def w_no_sync(rank, size):
    """FlatAdafactor with clipping, parameter groups and an lr schedule on a channels_last ConvNet: step() never
    synchronises the host, the gradients are re-zeroed, and the update equals torch.optim.Adafactor on CUDA to 1e-5."""
    torch.manual_seed(11)
    net = ConvNet().to(_dev()).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=32 << 10)
    groups = [{"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0, "lr": 2e-2}]
    opt = b2.FlatAdafactor(ddp, max_grad_norm=1.0, param_groups=groups,
                           lr_schedule=b2.LRSchedule(warmup_steps=2, decay="cosine", total_steps=8), **HP)
    for it in range(4):
        x, y = _batch(it, rank)
        opt.zero_grad()
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert all(not gb.flat.any() for gb in ddp.buckets)
    assert opt.steps == 4 and opt.grad_norm() > 0
    ddp.remove_hooks()
