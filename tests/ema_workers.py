"""Workers of tests/test_ema_cpu.py (gloo CPU ranks): ``FlatEMA`` over every flat optimizer and mode against
``torch.optim.swa_utils.AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=True)``, driven as
torchvision's ``--model-ema`` drives it: ``update_parameters`` every ``every`` steps, and ``n_averaged.fill_(0)`` after an
update during warmup.

The reference averages a plain module (no DDP) that is loaded, after every step, with the DDP model's live parameters and
buffers, so it follows the same training bit for bit and any difference is the EMA's own.  The model has a BatchNorm, so its
running statistics (fp32 buffers, different on every rank) are averaged too."""
import os

import torch
import torch.nn as nn
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatEMA, FlatLAMB, FlatLARS, FlatSGD
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel

STEPS = 12
# (every, warmup_steps, decay): both sides of w = 1 - decay = 0.5
SETTINGS = [(1, 0, 0.9), (1, 4, 0.3), (3, 0, 0.3), (3, 4, 0.9)]
FLAT = {"sgd": FlatSGD, "adamw": FlatAdamW, "lamb": FlatLAMB, "lars": FlatLARS}
# (name, optimizer, kwargs, micro-batches per step)
CASES = [("sgd groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, groups=True), 1),
         ("sgd clip", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.05), 1),
         ("sgd sharded groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, sharded=True, groups=True), 1),
         ("adamw groups", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, groups=True), 1),
         ("adamw clip", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05), 1),
         ("adamw sharded", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, sharded=True), 1),
         ("lamb", "lamb", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1), 1),
         ("lars", "lars", dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4), 1),
         ("sgd sharded no_sync k=2", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, sharded=True), 2)]


class Net(nn.Module):
    def __init__(self, seed=5):
        super().__init__()
        torch.manual_seed(seed)
        self.fc1, self.bn = nn.Linear(13, 24), nn.BatchNorm1d(24)
        self.fc2, self.fc3 = nn.Linear(24, 7), nn.Linear(7, 5)

    def forward(self, x):
        return self.fc3(torch.tanh(self.fc2(torch.relu(self.bn(self.fc1(x))))))


def build(kind, hp, **ema_kw):
    """(net, ddp, optimizer, FlatEMA or None)."""
    hp = dict(hp)
    net = Net()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
    if hp.pop("groups", False):
        hp["param_groups"] = [{"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0}]
    opt = FLAT[kind](ddp, **hp)
    return net, ddp, opt, (FlatEMA(opt, **ema_kw) if ema_kw else None)


def batch(rank, it, j):
    g = torch.Generator().manual_seed(7919 * it + 101 * j + rank)
    return torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)


def train_step(ddp, opt, rank, it, k=1):
    for j in range(k):
        x, y = batch(rank, it, j)
        if j < k - 1:
            with ddp.no_sync():
                (((ddp(x) - y) ** 2).mean() / k).backward()
        else:
            (((ddp(x) - y) ** 2).mean() / k).backward()
    b2.average_gradients(ddp)
    opt.step()


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().cpu().contiguous().view(torch.int32)


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def averaged(avg: AveragedModel) -> dict:
    """The reference's EMA: parameters and fp32 buffers by name."""
    out = {n: p for n, p in avg.module.named_parameters()}
    out.update({n: b for n, b in avg.module.named_buffers() if b.dtype == torch.float32})
    return out


def check_against(named: dict, avg: AveragedModel, what: str) -> None:
    ref = averaged(avg)
    assert sorted(named) == sorted(ref), (what, sorted(named), sorted(ref))
    for n, t in ref.items():
        assert same_bits(named[n], t), f"{what}: {n} differs by {float((named[n] - t.detach().cpu()).abs().max())}"


def raises(exc, fn, match=""):
    try:
        fn()
    except exc as e:
        assert match in str(e), (match, str(e))
        return
    raise AssertionError(f"{fn} did not raise {exc.__name__}")


def enter_twice(ema):
    with ema.average_parameters():
        pass


def check_average_parameters(net, ddp, opt, ema, avg, what, probe=None):
    """Inside the block the model holds the EMA (integer buffers stay live); update(), step() and nesting raise; an eval
    forward of ``probe`` runs; afterwards the live values and the EMA are back bit for bit."""
    live = {n: t.detach().clone() for n, t in net.state_dict().items()}
    flats = [e.clone() for e in ema.ema_flats + ema.ema_buffers]
    ref = averaged(avg)
    saved = ema.state_dict()
    with ema.average_parameters():
        sd = net.state_dict()
        for n, t in ref.items():
            assert same_bits(sd[n], t), f"{what}: average_parameters() shows {n} other than the EMA"
        check_against(ema.named_ema(ddp), avg, f"{what}: named_ema() inside average_parameters()")
        inside = ema.state_dict()
        assert all(same_bits(a, b) for a, b in zip(inside["ema"], saved["ema"])), what
        assert all(same_bits(inside["buffers"][n], saved["buffers"][n]) for n in saved["buffers"]), what
        assert all(torch.equal(t, live[n]) for n, t in sd.items() if not t.is_floating_point())
        raises(RuntimeError, ema.update, "inside average_parameters")
        raises(RuntimeError, opt.step, "inside FlatEMA.average_parameters")
        raises(RuntimeError, lambda: enter_twice(ema), "inside average_parameters")
        if probe is not None:
            with torch.no_grad():
                net.eval()
                ddp(probe)
                net.train()
    for n, t in net.state_dict().items():
        assert torch.equal(bits(t) if t.is_floating_point() else t, bits(live[n]) if t.is_floating_point() else live[n]), \
            f"{what}: {n} not restored"
    for a, b in zip(ema.ema_flats + ema.ema_buffers, flats):
        assert same_bits(a, b), f"{what}: the EMA changed across average_parameters()"


def w_against_reference(rank, size):
    for name, kind, hp, k in CASES:
        for every, warmup, decay in SETTINGS:
            what = f"{name}, every={every}, warmup_steps={warmup}, decay={decay}, rank {rank} of {size}"
            net, ddp, opt, ema = build(kind, hp, decay=decay, every=every, warmup_steps=warmup)
            ref = Net()
            ref.load_state_dict(net.state_dict())
            avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=True)
            check_against(ema.named_ema(ddp), avg, what + ", construction")
            for it in range(STEPS):
                train_step(ddp, opt, rank, it, k)
                ema.update()
                t = it + 1
                ref.load_state_dict(net.state_dict())
                if t % every == 0:
                    avg.update_parameters(ref)
                    if t <= warmup:
                        avg.n_averaged.fill_(0)
                check_against(ema.named_ema(ddp), avg, f"{what}, step {t}")
                if t == 7:
                    check_average_parameters(net, ddp, opt, ema, avg, what, batch(0, 999, 0)[0])
            if hp.get("sharded") and size > 1:     # 1/W of the EMA per rank
                assert sum(e.numel() for e in ema.ema_flats) < sum(p.numel() for p in opt.param_flats), what
            ddp.remove_hooks()


def w_checkpoints(rank, size):
    """state_dict round trips, sharded and not; a whole EMA into a sharded one; the refusals of load_state_dict."""
    hp = dict(lr=0.05, momentum=0.9)
    for sharded in (False, True):
        net, ddp, opt, ema = build("sgd", dict(hp, sharded=sharded), decay=0.8, every=2, warmup_steps=1)
        for it in range(5):
            train_step(ddp, opt, rank, it)
            ema.update()
        sd = ema.state_dict()
        assert sd["decay"] == 0.8 and sd["every"] == 2 and sd["warmup_steps"] == 1 and bool(sd.get("sharded")) == sharded
        named = ema.named_ema(ddp)
        net2, ddp2, opt2, ema2 = build("sgd", dict(hp, sharded=sharded), decay=0.8, every=2, warmup_steps=1)
        ema2.load_state_dict(sd)
        for a, b in zip(ema.ema_flats + ema.ema_buffers, ema2.ema_flats + ema2.ema_buffers):
            assert same_bits(a, b)
        # other settings: refused before anything is loaded
        _, ddp3, opt3, ema3 = build("sgd", dict(hp, sharded=sharded), decay=0.7, every=2, warmup_steps=1)
        before = [e.clone() for e in ema3.ema_flats + ema3.ema_buffers]
        raises(ValueError, lambda: ema3.load_state_dict(sd), "written with")
        for a, b in zip(ema3.ema_flats + ema3.ema_buffers, before):
            assert same_bits(a, b)
        # a shard loads on its own rank of its own world size only
        if sharded:
            _, ddp4, _, ema4 = build("sgd", dict(hp, sharded=False), decay=0.8, every=2, warmup_steps=1)
            raises(ValueError, lambda: ema4.load_state_dict(sd), "shard")
            other = dict(sd, rank=(rank + 1) % size)
            raises(ValueError, lambda: ema2.load_state_dict(other), "shard")
            ddp4.remove_hooks()
        else:                                   # a whole EMA loads into a sharded one as each rank's slice
            _, ddp5, _, ema5 = build("sgd", dict(hp, sharded=True), decay=0.8, every=2, warmup_steps=1)
            ema5.load_state_dict(sd)
            got = ema5.named_ema(ddp5)
            assert sorted(got) == sorted(named) and all(same_bits(got[n], named[n]) for n in named)
            ddp5.remove_hooks()
        # named_ema / load_named_ema round trip
        _, ddp6, _, ema6 = build("sgd", dict(hp, sharded=sharded), decay=0.8, every=2, warmup_steps=1)
        assert ema6.load_named_ema(ddp6, named) == len(named)
        got = ema6.named_ema(ddp6)
        assert all(same_bits(got[n], named[n]) for n in named)
        for d in (ddp, ddp2, ddp3, ddp6):
            d.remove_hooks()


def w_sharded_exchange_refused(rank, size):
    """Sharded: a gradient exchange inside average_parameters() raises before it updates anything."""
    net, ddp, opt, ema = build("sgd", dict(lr=0.05, momentum=0.9, sharded=True), decay=0.8)
    for it in range(2):
        train_step(ddp, opt, rank, it)
        ema.update()
    params = [p.clone() for p in opt.param_flats]
    state = [m.clone() for m in opt.momentum_flats] + [e.clone() for e in ema.ema_flats + ema.ema_buffers]
    with ema.average_parameters():
        inside = [p.clone() for p in opt.param_flats]
        x, y = batch(rank, 5, 0)
        net.eval()                       # in train mode the forward itself would move the BatchNorm statistics
        with ddp.no_sync():
            ((ddp(x) - y) ** 2).mean().backward()
        net.train()
        raises(RuntimeError, lambda: b2.average_gradients(ddp), "inside FlatEMA.average_parameters")
        assert all(same_bits(a, b) for a, b in zip(opt.param_flats, inside))
    assert all(same_bits(a, b) for a, b in zip(opt.param_flats, params))
    assert all(same_bits(a, b) for a, b in zip(opt.momentum_flats + ema.ema_flats + ema.ema_buffers, state))
    assert opt.steps == 2
    ddp.remove_hooks()


def w_save_named(rank, size):
    """Sharded at this world size: train, then write named_ema (rank 0) to $B2_EMA_CKPT."""
    net, ddp, opt, ema = build("adamw", dict(lr=0.01, sharded=True), decay=0.8)
    for it in range(4):
        train_step(ddp, opt, rank, it)
        ema.update()
    named = ema.named_ema(ddp)
    if rank == 0:
        torch.save({n: t for n, t in named.items() if not n.startswith("bn.running")}, os.environ["B2_EMA_CKPT"])
    b2.barrier()
    ddp.remove_hooks()


def w_load_named(rank, size):
    """Sharded at another world size: load_named_ema of the saved parameters gives them back from named_ema."""
    net, ddp, opt, ema = build("adamw", dict(lr=0.01, sharded=True), decay=0.8)
    saved = torch.load(os.environ["B2_EMA_CKPT"])
    assert ema.load_named_ema(ddp, saved) == len(saved)
    got = ema.named_ema(ddp)
    for n, t in saved.items():
        assert same_bits(got[n], t), n
    ddp.remove_hooks()


# ---------------------------------------------------------------------------------------------------- GPU (tests/test_gpu_ema*.py)
GPU_STEPS = 20


def resnet_sync_bn(dev):
    from dist_tuto.pth_b200.models.resnet import ResNet18

    torch.manual_seed(0)
    return b2.SyncBatchNorm.convert_sync_batchnorm(ResNet18()).to(dev).to(memory_format=torch.channels_last)


def gpu_optimizers():
    """(name, constructor) of every flat optimizer on its CUDA kernel path."""
    def groups(m):
        return [{"params": [p for p in m.parameters() if p.ndim <= 1], "weight_decay": 0.0}]
    return [("sgd groups", lambda ddp, m: FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, param_groups=groups(m))),
            ("sgd clip", lambda ddp, m: FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.5)),
            ("adamw groups", lambda ddp, m: FlatAdamW(ddp, lr=3e-3, weight_decay=0.05, param_groups=groups(m))),
            ("lamb", lambda ddp, m: FlatLAMB(ddp, lr=2e-3)),
            ("lars", lambda ddp, m: FlatLARS(ddp, lr=0.3, trust_coefficient=1e-2))]


def resnet_step(ddp, opt, dev, it, rank=0):
    import torch.nn.functional as F

    g = torch.Generator(device=dev).manual_seed(10007 * it + rank)
    x = torch.randn(16, 3, 32, 32, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), generator=g, device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.cross_entropy(ddp(x), y)
    loss.backward()
    b2.average_gradients(ddp)
    opt.step()


def w_gpu_training(rank, size):
    """ResNet-18 (SyncBatchNorm, bf16 autocast) on every optimizer's kernel path: the EMA equals AveragedModel on CUDA bit
    for bit after every step, with every = 2, warmup_steps = 3; average_parameters() shows it and restores the live model."""
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    for name, make in gpu_optimizers():
        for decay in (0.999, 0.3):
            m = resnet_sync_bn(dev)
            avg = AveragedModel(m, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=True)
            ddp = DistributedDataParallel(m, bucket_cap_bytes=4 << 20)
            opt = make(ddp, m)
            ema = FlatEMA(opt, decay=decay, every=2, warmup_steps=3)
            assert len(ema.ema_buffers) == 40          # running mean and variance of ResNet-18's 20 norms
            for it in range(GPU_STEPS):
                resnet_step(ddp, opt, dev, it, rank)
                ema.update()
                t = it + 1
                if t % 2 == 0:
                    avg.update_parameters(m)
                    if t <= 3:
                        avg.n_averaged.fill_(0)
                check_against(ema.named_ema(ddp), avg, f"{name}, decay {decay}, step {t}")
            check_average_parameters(m, ddp, opt, ema, avg, name)
            ddp.remove_hooks()


def graphed_ema(make, n, graph, dev, every=3, warmup_steps=4, warmup=3):
    """Capturable optimizer + FlatEMA: ``warmup`` eager steps on a side stream, then ``n`` eager steps or replays of one
    captured step + update().  Returns the model state, the EMA and the optimizer's step count."""
    import torch.nn.functional as F

    import capturable_workers as CW
    torch.manual_seed(7)
    m = CW.net().to(dev).to(memory_format=torch.channels_last)
    ddp = DistributedDataParallel(m)
    opt = make(ddp, m, capturable=True)
    ema = FlatEMA(opt, decay=0.9, every=every, warmup_steps=warmup_steps)
    gen = torch.Generator().manual_seed(100)
    xs = [torch.randn(8, 3, 12, 12, generator=gen).to(dev).contiguous(memory_format=torch.channels_last)
          for _ in range(warmup + n)]
    ys = [torch.randint(0, 10, (8,), generator=gen).to(dev) for _ in range(warmup + n)]
    x, y = xs[0].clone(), ys[0].clone()

    def step():
        F.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        opt.step()
        ema.update()

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for i in range(warmup):
            x.copy_(xs[i]); y.copy_(ys[i])
            step()
    torch.cuda.current_stream(dev).wait_stream(s)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for i in range(warmup, warmup + n):
            x.copy_(xs[i]); y.copy_(ys[i])
            g.replay()
    else:
        for i in range(warmup, warmup + n):
            x.copy_(xs[i]); y.copy_(ys[i])
            step()
    torch.cuda.synchronize(dev)
    ddp.remove_hooks()
    return [t.detach().clone() for t in m.state_dict().values()], [e.clone() for e in ema.ema_flats + ema.ema_buffers], opt.steps


def w_gpu_multi(rank, size):
    """Real ranks: a sharded kernel-mode FlatSGD's EMA (1/W per rank) equals the unsharded run's, and so does the model
    inside average_parameters(); afterwards the live parameters are back."""
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    runs = []
    for sharded in (False, True):
        m = resnet_sync_bn(dev)
        ddp = DistributedDataParallel(m, bucket_cap_bytes=4 << 20)
        opt = FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, sharded=sharded)
        assert (opt._shard_mode == "kernel") == sharded
        ema = FlatEMA(opt, decay=0.9, every=2, warmup_steps=1)
        for it in range(6):
            resnet_step(ddp, opt, dev, it, rank)
            ema.update()
        runs.append((m, ddp, opt, ema))
    (mu, du, ou, eu), (ms, ds, os_, es) = runs
    want, got = eu.named_ema(du), es.named_ema(ds)
    assert sorted(want) == sorted(got) and all(same_bits(want[n], got[n]) for n in want), rank
    assert sum(e.numel() for e in es.ema_flats) * size <= sum(e.numel() for e in eu.ema_flats) + 64 * size * len(es.ema_flats)
    live = {n: t.detach().clone() for n, t in ms.state_dict().items()}
    with es.average_parameters():
        sd = ms.state_dict()
        assert all(same_bits(sd[n], want[n]) for n in want), rank
    assert all(torch.equal(t, live[n]) for n, t in ms.state_dict().items()), rank
    du.remove_hooks()
    ds.remove_hooks()
