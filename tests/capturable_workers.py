"""End-to-end runs of capturable FlatSGD / FlatAdamW under DistributedDataParallel: N eager steps, or warm-up steps on a
side stream, one captured step and replays, from the same seeded state.  Used in-process at world 1 and by real ranks."""
import torch
import torch.nn as nn
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2

WARMUP = 3


def net():
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), b2.SyncBatchNorm(8), nn.ReLU(), nn.Conv2d(8, 16, 3, padding=1),
                         b2.SyncBatchNorm(16), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(16, 10))


def optimizers():
    """(name, constructor of the optimizer for a model) of the cases the end-to-end tests cover."""
    def groups(m):
        return [{"params": [p for p in m.parameters() if p.ndim <= 1], "weight_decay": 0.0, "lr": 0.02}]
    return [
        ("sgd nesterov groups clip cosine",
         lambda ddp, m, **kw: b2.FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True, max_grad_norm=0.5,
                                         param_groups=groups(m), lr_schedule=b2.LRSchedule(decay="cosine", total_steps=12,
                                                                                           min_factor=0.1), **kw)),
        ("adamw groups clip warmup",
         lambda ddp, m, **kw: b2.FlatAdamW(ddp, lr=3e-3, weight_decay=0.05, max_grad_norm=1.0, param_groups=groups(m),
                                           lr_schedule=b2.LRSchedule(warmup_steps=8, warmup_start=0.1), **kw)),
    ]


def run(make_opt, n, graph, dev, rank=0, capturable=True, sharded=False, bucket_cap_bytes=8 << 20):
    """``n`` steps; with ``graph`` the steps from WARMUP on are replays of one captured step.  Returns the model, the
    optimizer and each step's ``grad_norm()``-carrying optimizer state."""
    torch.manual_seed(7)
    m = net().to(dev).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(m, bucket_cap_bytes=bucket_cap_bytes)
    kw = dict(capturable=True) if capturable else {}
    opt = make_opt(ddp, m, sharded=sharded, **kw)
    gen = torch.Generator().manual_seed(100 + rank)
    xs = [torch.randn(16, 3, 12, 12, generator=gen).to(dev).contiguous(memory_format=torch.channels_last) for _ in range(n)]
    ys = [torch.randint(0, 10, (16,), generator=gen).to(dev) for _ in range(n)]
    x, y = xs[0].clone(), ys[0].clone()

    def step():
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        opt.step()

    if not graph:
        for i in range(n):
            x.copy_(xs[i]); y.copy_(ys[i])
            step()
    else:
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):                       # warm-up on a side stream, as torch requires before a capture
            for i in range(WARMUP):
                x.copy_(xs[i]); y.copy_(ys[i])
                step()
        torch.cuda.current_stream(dev).wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for i in range(WARMUP, n):
            x.copy_(xs[i]); y.copy_(ys[i])
            g.replay()
    torch.cuda.synchronize(dev)
    ddp.remove_hooks()
    return m, opt


def state(m, opt):
    """(parameters and buffers, the optimizer's state flats, the last pre-clip norm, the checkpointed step count).  The
    first are replicated on every rank; sharded, the flats are this rank's slices."""
    flats = [f for name in ("momentum_flats", "exp_avg_flats", "exp_avg_sq_flats") for f in getattr(opt, name, [])]
    return ([t.detach().clone(memory_format=torch.contiguous_format) for t in m.state_dict().values()],
            [f.clone() for f in flats], opt.grad_norm(), opt.state_dict()["steps"])


def _bits_equal(ta, tb):
    bits = lambda t: t.reshape(-1).view(torch.uint8)      # noqa: E731 - bit for bit, -0 and NaN included
    return len(ta) == len(tb) and all(x.dtype == y.dtype and torch.equal(bits(x), bits(y)) for x, y in zip(ta, tb))


def same(a, b):
    """Two state() results are bit for bit equal."""
    return _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]


def w_graph_equals_eager(rank, size):
    """Real ranks: sharded capturable FlatSGD / FlatAdamW, graph replays against eager steps, bit for bit and identical
    across ranks."""
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    for name, make in optimizers():
        for sharded in (False, True):
            mk = _no_clip(name) if sharded else make       # a sharded optimizer cannot clip
            a = state(*run(mk, 12, False, dev, rank, sharded=sharded, bucket_cap_bytes=32 << 10))
            b = state(*run(mk, 12, True, dev, rank, sharded=sharded, bucket_cap_bytes=32 << 10))
            assert same(a, b), (name, sharded, rank)
            # the replicated state (parameters and buffers; the optimizer's flats too when it is not sharded) is the same
            # on every rank; sharded, each rank holds its own slice of the optimizer state
            replicated = b[0] + ([] if sharded else b[1])
            flat = torch.cat([t.reshape(-1).view(torch.uint8) for t in replicated])
            got = [torch.empty_like(flat) for _ in range(size)]
            torch.distributed.all_gather(got, flat)
            assert all(torch.equal(got[0], g) for g in got), (name, sharded)


def _no_clip(name):
    if name.startswith("sgd"):
        return lambda ddp, m, **kw: b2.FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True,
                                               lr_schedule=b2.LRSchedule(decay="cosine", total_steps=12, min_factor=0.1), **kw)
    return lambda ddp, m, **kw: b2.FlatAdamW(ddp, lr=3e-3, weight_decay=0.05,
                                             lr_schedule=b2.LRSchedule(warmup_steps=8, warmup_start=0.1), **kw)
