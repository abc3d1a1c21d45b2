"""Workers of tests/test_adafactor_cpu.py (spawned processes, gloo @127.0.0.1): ``FlatAdafactor`` on CPU ranks against a
reference without DDP -- the same module and micro-batches, autograd's accumulation into ``p.grad``, an all-reduce average in
flat buffers laid out like the DDP buckets (so that gloo adds the same values in the same order), then
``torch.optim.Adafactor(foreach=False)``, driven by its own ``torch.amp.GradScaler("cpu")`` in the scaled cases."""
import os

import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdafactor, FlatEMA, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel, GradBucket
from dist_tuto.pth_b200.utils.checkpoint import load_checkpoint, save_checkpoint

STEPS = 5
SCHED = LRSchedule(warmup_steps=2, decay="cosine", total_steps=7, min_factor=0.1)
POISON = {1: float("inf"), 3: float("nan")}        # step -> factor of rank 0's loss in the scaled cases

# (name, FlatAdafactor kwargs, micro-batches per step, GradScaler)
CASES = [
    ("plain", dict(lr=1e-2), 1, False),
    ("decay d groups", dict(lr=1e-2, weight_decay=0.05, d=1.5, eps=(1e-30, 1e-3), groups=True), 2, False),
    ("clip groups", dict(lr=2e-2, beta2_decay=-0.5, weight_decay=0.01, max_grad_norm=0.05, groups=True), 1, False),
    ("scaled clip", dict(lr=1e-2, weight_decay=0.01, max_grad_norm=0.05), 2, True),
]


class Net(nn.Module):
    """Every shape class Adafactor distinguishes: 0-D, 1-D, 2-D (R == 1 and C == 1 included), 3-D and a channels_last conv
    weight factored over its kernel dimensions."""

    def __init__(self, seed=3):
        super().__init__()
        torch.manual_seed(seed)
        self.conv = nn.Conv2d(3, 4, 3).to(memory_format=torch.channels_last)
        self.lin = nn.Linear(16, 5)
        self.row = nn.Parameter(torch.randn(1, 5) * 0.1)          # R == 1
        self.col = nn.Parameter(torch.randn(5, 1) * 0.1)          # C == 1
        self.cube = nn.Parameter(torch.randn(2, 5, 5) * 0.1)      # 3-D
        self.scale = nn.Parameter(torch.tensor(1.0))              # 0-D

    def forward(self, x):
        h = self.conv(x).flatten(1)
        y = self.lin(h) * self.scale + self.row
        y = y + (self.cube.sum(0) @ self.col).t()
        return y


def _groups(net):
    return [{"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0},
            {"params": [net.lin.weight], "lr": 3e-2}]


def _loss(model, rank, it, j, k, poison=1.0):
    g = torch.Generator().manual_seed(10007 * it + 101 * j + rank)
    x, y = torch.randn(4, 3, 4, 4, generator=g), torch.randn(4, 5, generator=g)
    return (model(x) - y).pow(2).mean() / k * poison


def make(hp):
    """(net, ddp, FlatAdafactor, reference net, torch.optim.Adafactor, base lr per reference group, reference buckets,
    parameter names in bucket order)."""
    hp = dict(hp)
    groups = hp.pop("groups", False)
    net = Net()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=300)
    opt = FlatAdafactor(ddp, lr_schedule=SCHED, param_groups=_groups(net) if groups else None, **hp)
    ref = Net()
    t_hp = {k: v for k, v in hp.items() if k != "max_grad_norm"}
    named = {id(q) for g in _groups(ref) for q in g["params"]}
    ref_groups = (_groups(ref) + [{"params": [p for p in ref.parameters() if id(p) not in named]}]) if groups \
        else [{"params": list(ref.parameters())}]
    topt = torch.optim.Adafactor(ref_groups, foreach=False, **t_hp)
    base = [g["lr"] for g in topt.param_groups]
    names = {id(p): n for n, p in net.named_parameters()}
    rp = dict(ref.named_parameters())
    order = [names[id(p)] for gb in ddp.buckets for p in gb.params]
    rbs = [GradBucket([rp[names[id(p)]] for p in gb.params], symmetric=False) for gb in ddp.buckets]
    return net, ddp, opt, ref, topt, base, rbs, order


def _backward(model, rank, it, k, scaler=None, poison=1.0):
    for j in range(k):
        loss = _loss(model, rank, it, j, k, poison)
        loss = scaler.scale(loss) if scaler is not None else loss
        if j < k - 1 and hasattr(model, "no_sync"):
            with model.no_sync():
                loss.backward()
        else:
            loss.backward()


def _scaler():
    return torch.amp.GradScaler("cpu", init_scale=1000.0, growth_interval=2)


def compare(net, opt, ref, topt, what):
    rp = dict(ref.named_parameters())
    for n, p in net.named_parameters():
        assert torch.equal(p, rp[n]), (what, n)
    mine = opt.named_state(net)
    for n, p in ref.named_parameters():
        st = topt.state[p]
        assert set(mine[n]) == set(st), (what, n, set(mine[n]), set(st))
        for key in st:
            assert torch.equal(mine[n][key], st[key]), (what, n, key)


def w_against_torch(rank, size, case):
    """One case of CASES: parameters and state bit for bit torch.optim.Adafactor(foreach=False), the scalers equal, skipped
    steps skipped on every rank with the buckets zeroed, and the replicas identical."""
    name, hp, k, scaled = next(c for c in CASES if c[0] == case)
    net, ddp, opt, ref, topt, base, rbs, order = make(hp)
    scaler, rscaler = (_scaler(), _scaler()) if scaled else (None, None)
    applied = 0
    for it in range(STEPS):
        poison = POISON.get(it, 1.0) if scaled and rank == 0 else 1.0
        opt.zero_grad()
        _backward(ddp, rank, it, k, scaler, poison)
        b2.average_gradients(ddp)
        if scaled:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        for gb in rbs:
            gb.zero_()
        _backward(ref, rank, it, k, rscaler, poison)
        for gb in rbs:
            gb.all_reduce_average_()
        if rscaler is not None:
            rscaler.unscale_(topt)
        if "max_grad_norm" in hp:
            rp = dict(ref.named_parameters())
            tn = torch.nn.utils.clip_grad_norm_([rp[n] for n in order], hp["max_grad_norm"], foreach=False)
        for g, b in zip(topt.param_groups, base):
            g["lr"] = SCHED.lr_at(b, applied)
        skipped = False
        if rscaler is not None:
            rscaler.step(topt)
            skipped = sum(float(v) for v in rscaler._found_inf_per_device(topt).values()) > 0
            rscaler.update()
            assert scaler.get_scale() == rscaler.get_scale()
            assert skipped == (it in POISON), (it, skipped)
            if skipped:
                assert all(not gb.flat.any() for gb in opt.buckets), "a skipped step leaves the buckets zeroed"
        else:
            topt.step()
        applied += not skipped
        assert opt.steps == applied
        if "max_grad_norm" in hp and not skipped:
            assert opt.grad_norm() == float(tn), (name, it)
        compare(net, opt, ref, topt, (name, it))
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)
    ddp.remove_hooks()
    b2.barrier()


def w_all_cases(rank, size):
    for case in CASES:
        w_against_torch(rank, size, case[0])


def w_ema(rank, size):
    """FlatEMA over FlatAdafactor equals torch._foreach_copy_ / _foreach_lerp_ over the reference's parameters."""
    net, ddp, opt, ref, topt, base, rbs, order = make(dict(lr=1e-2, weight_decay=0.01))
    ema = FlatEMA(opt, decay=0.8)
    rema = None
    for it in range(4):
        opt.zero_grad()
        _backward(ddp, rank, it, 1)
        b2.average_gradients(ddp)
        opt.step()
        ema.update()
        for gb in rbs:
            gb.zero_()
        _backward(ref, rank, it, 1)
        for gb in rbs:
            gb.all_reduce_average_()
        for g, b in zip(topt.param_groups, base):
            g["lr"] = SCHED.lr_at(b, it)
        topt.step()
        params = [p.detach() for p in ref.parameters()]
        if rema is None:
            rema = [p.clone() for p in params]
        else:
            torch._foreach_lerp_(rema, params, 1 - 0.8)
    got = ema.named_ema(net)
    for (n, _), e in zip(ref.named_parameters(), rema):
        assert torch.equal(got[n], e), n
    ddp.remove_hooks()
    b2.barrier()


def _train(ddp, opt, rank, first, n):
    for it in range(first, first + n):
        opt.zero_grad()
        _backward(ddp, rank, it, 1)
        b2.average_gradients(ddp)
        opt.step()


def w_save(rank, size):
    """World 2: three steps, then a checkpoint (model + named state)."""
    net, ddp, opt = make(dict(lr=1e-2, weight_decay=0.01))[:3]
    _train(ddp, opt, rank, 0, 3)
    if rank == 0:
        save_checkpoint(os.environ["B2_ADAFACTOR_CKPT"], net, opt, step=3)
    ddp.remove_hooks()
    b2.barrier()


def w_load(rank, size):
    """World 3 with another bucket layout: the checkpoint's per-name state and step count load exactly, and training goes on
    with the replicas bit-identical."""
    net = Net()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=120)
    opt = FlatAdafactor(ddp, lr=1e-2, weight_decay=0.01, lr_schedule=SCHED)
    load_checkpoint(os.environ["B2_ADAFACTOR_CKPT"], net, opt)
    saved = torch.load(os.environ["B2_ADAFACTOR_CKPT"], weights_only=False)["optim_state"]
    mine = opt.named_state(net)
    assert opt.steps == 3 and mine.keys() == saved.keys()
    for n in mine:
        for key in mine[n]:
            assert torch.equal(mine[n][key], saved[n][key]), (n, key)
    _train(ddp, opt, rank, 3, 2)
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)
    ddp.remove_hooks()
    b2.barrier()


def w_torch_round_trip(rank, size):
    """named_state loads into a plain torch.optim.Adafactor (through the names), which continues bit for bit, and its
    state_dict loads back into a FlatAdafactor of another bucket layout."""
    hp = dict(lr=1e-2, weight_decay=0.01)
    net, ddp, opt, ref, topt, base, rbs, order = make(hp)
    _train(ddp, opt, rank, 0, 3)
    ref.load_state_dict(net.state_dict())
    t2 = torch.optim.Adafactor(ref.parameters(), foreach=False, **hp)
    named = opt.named_state(net)
    rnames = dict(ref.named_parameters())
    t2.load_state_dict({"state": {i: named[n] for i, (n, _) in enumerate(ref.named_parameters())},
                        "param_groups": [dict(t2.param_groups[0], params=list(range(len(rnames))))]})
    for gb in rbs:
        gb.zero_()
    _backward(ref, rank, 3, 1)
    for gb in rbs:
        gb.all_reduce_average_()
    t2.param_groups[0]["lr"] = SCHED.lr_at(hp["lr"], 3)
    t2.step()
    _train(ddp, opt, rank, 3, 1)
    compare(net, opt, ref, t2, "torch round trip")
    net3 = Net()
    ddp3 = DistributedDataParallel(net3, bucket_cap_bytes=150)
    opt3 = FlatAdafactor(ddp3, lr_schedule=SCHED, **hp)
    back = {n: t2.state[p] for n, p in ref.named_parameters()}
    assert opt3.load_named_state(net3, back) == len(back) and opt3.steps == 4
    mine = opt3.named_state(net3)
    for n in back:
        for key in back[n]:
            assert torch.equal(mine[n][key], back[n][key]), (n, key)
    for d in (ddp, ddp3):
        d.remove_hooks()
    b2.barrier()
