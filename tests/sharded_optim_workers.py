"""Workers of tests/test_sharded_optim_cpu.py (spawned processes, gloo @127.0.0.1): ``FlatSGD(sharded=True)`` without peer
memory -- the all-reduce, the update of the owned slice and the parameter all-gather with torch ops."""
import os

import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatSGD, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel

STEPS = 5
OPTS = dict(lr=0.2, momentum=0.9, weight_decay=0.01, nesterov=True,
            lr_schedule=LRSchedule(warmup_steps=2, decay="multistep", milestones=(3,), gamma=0.5))


def _mlp(seed=3):
    """221 + 17 + 187 + 11 + 55 + 5 parameters: with a 600-byte cap several buckets, none a multiple of 2 or 3 vectors."""
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(13, 17), nn.Tanh(), nn.Linear(17, 11), nn.Tanh(), nn.Linear(11, 5))


def _engine(sharded, **kw):
    net = _mlp()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
    return net, ddp, FlatSGD(ddp, sharded=sharded, **{**OPTS, **kw})


def _step(ddp, opt, rank, it, through_module=False):
    g = torch.Generator().manual_seed(1000 * it + rank)
    x, y = torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)
    opt.zero_grad()
    (ddp(x) - y).pow(2).mean().backward()
    b2.average_gradients(ddp.module if through_module else ddp)
    opt.step()


def _same(a: dict, b: dict):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k


def w_sharded_equals_unsharded(rank, size):
    net_u, ddp_u, opt_u = _engine(False)
    net_s, ddp_s, opt_s = _engine(True)
    assert len(opt_s.buckets) > 2 and any(gb.numel % (4 * size) for gb in opt_s.buckets)
    for k, gb in enumerate(opt_s.buckets):                       # momentum: the owned slice only
        per = opt_s.momentum_flats[k].numel()
        assert per == -(-(-(-gb.flat.numel() // 4)) // size) * 4 and per < gb.numel
        lo, hi = opt_s.shard_range(k)
        assert (lo, hi) == (min(rank * per, gb.numel), min((rank + 1) * per, gb.numel))
    assert opt_u.shard_range(0) == (0, opt_u.buckets[0].numel)
    for it in range(STEPS):
        _step(ddp_u, opt_u, rank, it)
        _step(ddp_s, opt_s, rank, it, through_module=it % 2 == 1)
        for (n, a), b in zip(net_u.named_parameters(), net_s.parameters()):
            assert torch.equal(a, b), (it, n)                    # bit-identical to the unsharded run
        for gb in opt_s.buckets:
            assert not gb.flat.any()                             # the exchange left the buckets zeroed
    assert opt_s.steps == opt_u.steps == STEPS and opt_s.lr_at() == opt_u.lr_at()
    flat = torch.cat([p.detach().reshape(-1) for p in net_s.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)              # replicas identical
    named_u, named_s = opt_u.named_momentum(net_u), opt_s.named_momentum(ddp_s)
    _same(named_u, named_s)
    assert any(v.abs().max() > 0 for v in named_s.values())

    # checkpoints: sharded -> unsharded -> sharded through the per-name form, and the training goes on identically
    net_a, ddp_a, opt_a = _engine(False)
    net_a.load_state_dict(net_s.state_dict())
    assert opt_a.load_named_momentum(net_a, named_s) == len(named_s)
    opt_a.steps = opt_s.steps
    net_b, ddp_b, opt_b = _engine(True)
    net_b.load_state_dict(net_a.state_dict())
    assert opt_b.load_named_momentum(net_b, opt_a.named_momentum(net_a)) == len(named_s)
    opt_b.steps = opt_a.steps
    for k in range(len(opt_s.buckets)):
        assert torch.equal(opt_b.momentum_flats[k], opt_s.momentum_flats[k])
    for it in range(STEPS, STEPS + 2):
        for ddp, opt in ((ddp_u, opt_u), (ddp_s, opt_s), (ddp_a, opt_a), (ddp_b, opt_b)):
            _step(ddp, opt, rank, it)
    for net in (net_s, net_a, net_b):
        for a, b in zip(net_u.parameters(), net.parameters()):
            assert torch.equal(a, b)

    # state_dict: whole buffers load into a sharded optimizer (each rank takes its slice); a shard loads on its own rank of
    # its own world size only
    net_c, ddp_c, opt_c = _engine(True)
    opt_c.load_state_dict(opt_u.state_dict())
    sd = opt_s.state_dict()
    assert sd["sharded"] is True and (sd["world"], sd["rank"]) == (size, rank) and "sharded" not in opt_u.state_dict()
    for k in range(len(opt_s.buckets)):
        assert torch.equal(opt_c.momentum_flats[k], opt_s.momentum_flats[k])
        assert sd["momentum_buffers"][k].numel() == opt_s.momentum_flats[k].numel()
    opt_c.load_state_dict(sd)
    assert opt_c.steps == opt_s.steps
    for bad in (dict(sd, rank=(rank + 1) % size), dict(sd, world=size + 1)):
        try:
            opt_c.load_state_dict(bad)
        except ValueError as e:
            assert "named_momentum" in str(e)
        else:
            raise AssertionError("a shard of another rank / world size was accepted")
    try:
        opt_u.load_state_dict(sd)
    except ValueError as e:
        assert "named_momentum" in str(e)
    else:
        raise AssertionError("an unsharded optimizer accepted a shard")
    b2.barrier()


def w_contract(rank, size):
    """max_grad_norm is refused; step() needs the step's exchange; one exchange per step; zero_grad=False; a plain module."""
    try:
        _engine(True, max_grad_norm=1.0)
    except ValueError as e:
        assert "sharded" in str(e)
    else:
        raise AssertionError("sharded=True accepted max_grad_norm")
    net, ddp, opt = _engine(True)
    try:
        opt.step()
    except RuntimeError as e:
        assert "average_gradients" in str(e)
    else:
        raise AssertionError("step() without an exchange passed")
    _step(ddp, opt, rank, 0)
    assert opt.steps == 1
    opt.zero_grad()
    (ddp(torch.ones(2, 13))).sum().backward()
    b2.average_gradients(ddp)
    try:
        b2.average_gradients(ddp)                                 # would apply every bucket's update a second time
    except RuntimeError as e:
        assert "twice" in str(e)
    else:
        raise AssertionError("a second exchange in one step passed")
    opt.step()
    # a module without the DDP wrapper (one bucket, exchanged by average_gradients), zero_grad=False: same parameters
    nets = []
    for sharded in (False, True):
        net = _mlp()
        opt = FlatSGD(net, sharded=sharded, zero_grad=False, **OPTS)
        for it in range(3):
            g = torch.Generator().manual_seed(77 * it + rank)
            opt.zero_grad()
            (net(torch.randn(4, 13, generator=g))).pow(2).mean().backward()
            b2.average_gradients(net)
            opt.step()
        assert net._grad_bucket.flat.any()                        # zero_grad=False: the gradients stay
        nets.append(net)
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        assert torch.equal(a, b)
    b2.barrier()


def w_save_named(rank, size):
    """Three sharded steps, then rank 0 writes the parameters and the per-name momentum for a world of another size."""
    net, ddp, opt = _engine(True)
    for it in range(3):
        _step(ddp, opt, rank, it)
    named = opt.named_momentum(ddp)                               # collective
    if rank == 0:
        torch.save({"model": net.state_dict(), "momentum": named, "steps": opt.steps}, os.environ["B2_SHARDED_CKPT"])
    b2.barrier()


def w_load_named(rank, size):
    blob = torch.load(os.environ["B2_SHARDED_CKPT"])
    net_s, ddp_s, opt_s = _engine(True)
    net_u, ddp_u, opt_u = _engine(False)
    for net, opt in ((net_s, opt_s), (net_u, opt_u)):
        net.load_state_dict(blob["model"])
        assert opt.load_named_momentum(net, blob["momentum"]) == len(blob["momentum"])
        opt.steps = blob["steps"]
    _same(opt_s.named_momentum(net_s), blob["momentum"])           # every rank's slice of a differently sized world
    for it in range(3, 5):
        _step(ddp_s, opt_s, rank, it)
        _step(ddp_u, opt_u, rank, it)
    for a, b in zip(net_u.parameters(), net_s.parameters()):
        assert torch.equal(a, b)
    _same(opt_s.named_momentum(net_s), opt_u.named_momentum(net_u))
    b2.barrier()


def w_world1(rank, size):
    """One rank: the flag changes nothing (the shard is everything, step() updates)."""
    nets = []
    for sharded in (False, True):
        net = _mlp()
        opt = FlatSGD(net, sharded=sharded, **OPTS)
        for it in range(3):
            (net(torch.randn(4, 13, generator=torch.Generator().manual_seed(it)))).pow(2).mean().backward()
            b2.average_gradients(net)
            opt.step()
        assert opt.shard_range(0) == (0, opt.buckets[0].numel) and "sharded" not in opt.state_dict()
        nets.append(net)
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        assert torch.equal(a, b)
