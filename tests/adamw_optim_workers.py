"""Workers of tests/test_adamw_cpu.py (spawned processes, gloo @127.0.0.1): ``FlatAdamW`` on CPU ranks, unsharded (torch's
single-tensor AdamW on the flats' views) and sharded (the all-reduce, AdamW on the owned slice and the parameter all-gather
with torch ops)."""
import os
import warnings

import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdamW, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel
from dist_tuto.pth_b200.utils.checkpoint import load_checkpoint, save_checkpoint

STEPS = 5
HP = dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1)
SCHED = LRSchedule(warmup_steps=2, decay="multistep", milestones=(3,), gamma=0.5)
# sharded and unsharded CPU runs do the same arithmetic per element, but torch's vectorised CPU kernels treat the last
# elements of a tensor in scalar code, and the slices start at other offsets: they agree to a few ulps
ATOL, RTOL = 1e-6, 1e-5


def _mlp(seed=3):
    """221 + 17 + 187 + 11 + 55 + 5 parameters: with a 600-byte cap several buckets, none a multiple of 2 or 3 vectors."""
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(13, 17), nn.Tanh(), nn.Linear(17, 11), nn.Tanh(), nn.Linear(11, 5))


def _engine(sharded, grad_dtype=None, **kw):
    net = _mlp()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600, grad_dtype=grad_dtype)
    return net, ddp, FlatAdamW(ddp, sharded=sharded, **{**HP, **kw})


def _backward(ddp, opt, rank, it):
    g = torch.Generator().manual_seed(1000 * it + rank)
    x, y = torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)
    opt.zero_grad()
    (ddp(x) - y).pow(2).mean().backward()


def _step(ddp, opt, rank, it):
    _backward(ddp, opt, rank, it)
    b2.average_gradients(ddp)
    opt.step()


def _bucket_grads(opt, net):
    """The averaged gradient of every parameter as the optimizer sees it (fp32 copies), by name."""
    names = {id(p): n for n, p in net.named_parameters()}
    return {names[id(p)]: gv.float().clone() for gb in opt.buckets for p, gv in zip(gb.params, gb.views)}


def _close(a, b):
    for (n, x), y in zip(a.named_parameters(), b.parameters()):
        assert torch.allclose(x, y, atol=ATOL, rtol=RTOL), n


def w_bit_equal_to_torch(rank, size):
    """Unsharded FlatAdamW is bit for bit torch.optim.AdamW(foreach=False) given the same averaged gradients: weight decay
    0 and > 0, an LRSchedule, max_grad_norm, and a bf16 bucket."""
    for kw, grad_dtype in ((dict(weight_decay=0.0), None), (dict(lr_schedule=SCHED), None), (dict(max_grad_norm=0.05), None),
                           ({}, torch.bfloat16)):
        net, ddp, opt = _engine(False, grad_dtype, zero_grad=False, **kw)
        ref = _mlp()
        topt = torch.optim.AdamW(ref.parameters(), foreach=False, **{**HP, **{k: v for k, v in kw.items() if k == "weight_decay"}})
        for it in range(STEPS):
            _backward(ddp, opt, rank, it)
            b2.average_gradients(ddp)
            grads = _bucket_grads(opt, net)
            for n, p in ref.named_parameters():
                p.grad = grads[n]
            if "max_grad_norm" in kw:                 # the norm sums the parameters in the buckets' order
                rp = dict(ref.named_parameters())
                tn = torch.nn.utils.clip_grad_norm_([rp[n] for n in grads], kw["max_grad_norm"], foreach=False)
            topt.param_groups[0]["lr"] = opt.lr_at()
            opt.step()
            topt.step()
            if "max_grad_norm" in kw:
                assert opt.grad_norm() == float(tn)
            for (n, a), b in zip(net.named_parameters(), ref.parameters()):
                assert torch.equal(a, b), (kw, grad_dtype, it, n)
        named = opt.named_state(net)
        for n, p in ref.named_parameters():
            st = topt.state[p]
            assert all(torch.equal(named[n][k], st[k]) for k in ("step", "exp_avg", "exp_avg_sq")), n
    b2.barrier()


def w_named_state_round_trip(rank, size):
    """named_state loads into torch.optim.AdamW and back, and the three runs continue identically."""
    net, ddp, opt = _engine(False)
    for it in range(3):
        _step(ddp, opt, rank, it)
    named = opt.named_state(net)
    ref = _mlp()
    ref.load_state_dict(net.state_dict())
    topt = torch.optim.AdamW(ref.parameters(), foreach=False, **HP)
    idx = {n: i for i, (n, _) in enumerate(ref.named_parameters())}
    sd = topt.state_dict()
    sd["state"] = {idx[n]: {k: v.clone() for k, v in s.items()} for n, s in named.items()}
    topt.load_state_dict(sd)
    net_b, ddp_b, opt_b = _engine(False)                                  # back: torch's state into a fresh FlatAdamW
    net_b.load_state_dict(ref.state_dict())
    back = {n: topt.state[p] for n, p in ref.named_parameters()}
    assert opt_b.load_named_state(net_b, back) == len(back) and opt_b.steps == 3
    for it in range(3, 5):
        _backward(ddp, opt, rank, it)
        b2.average_gradients(ddp)
        grads = _bucket_grads(opt, net)
        for n, p in ref.named_parameters():
            p.grad = grads[n]
        opt.step()
        topt.step()
        _step(ddp_b, opt_b, rank, it)
        for (n, a), b, c in zip(net.named_parameters(), ref.parameters(), net_b.parameters()):
            assert torch.equal(a, b) and torch.equal(a, c), (it, n)
    b2.barrier()


def w_sharded(rank, size):
    """Sharded: moments of the owned slice only, parameters bit-identical on every rank and within ATOL / RTOL of the
    unsharded run; state_dict shards, the per-name form across modes, and the refusals."""
    net_u, ddp_u, opt_u = _engine(False)
    net_s, ddp_s, opt_s = _engine(True)
    assert len(opt_s.buckets) > 2
    for k, gb in enumerate(opt_s.buckets):
        per = opt_s.exp_avg_flats[k].numel()
        assert per == opt_s.exp_avg_sq_flats[k].numel() < gb.numel
        assert opt_s.shard_range(k) == (min(rank * per, gb.numel), min((rank + 1) * per, gb.numel))
    for it in range(STEPS):
        _step(ddp_u, opt_u, rank, it)
        _step(ddp_s, opt_s, rank, it)
        _close(net_u, net_s)
        for gb in opt_s.buckets:
            assert not gb.flat.any()
    flat = torch.cat([p.detach().reshape(-1) for p in net_s.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)                      # replicas bit-identical
    su, ss = opt_u.named_state(net_u), opt_s.named_state(ddp_s)           # collective
    assert su.keys() == ss.keys()
    for n in su:
        assert torch.equal(su[n]["step"], ss[n]["step"])
        assert all(torch.allclose(su[n][k], ss[n][k], atol=ATOL, rtol=RTOL) for k in ("exp_avg", "exp_avg_sq")), n
    # state_dict: a shard loads on its own rank of its own world size only; whole buffers load as this rank's slice
    sd = opt_s.state_dict()
    assert sd["sharded"] is True and (sd["world"], sd["rank"]) == (size, rank) and "sharded" not in opt_u.state_dict()
    net_c, ddp_c, opt_c = _engine(True)
    opt_c.load_state_dict(sd)
    assert opt_c.steps == STEPS and all(torch.equal(a, b) for a, b in zip(opt_c.exp_avg_sq_flats, opt_s.exp_avg_sq_flats))
    opt_c.load_state_dict(opt_u.state_dict())
    for k in range(len(opt_s.buckets)):
        lo, hi = opt_c.shard_range(k)
        assert torch.equal(opt_c.exp_avg_flats[k][:hi - lo], opt_u.exp_avg_flats[k][lo:hi])
    for bad in (dict(sd, rank=(rank + 1) % size), dict(sd, world=size + 1)):
        try:
            opt_c.load_state_dict(bad)
        except ValueError as e:
            assert "named_state" in str(e)
        else:
            raise AssertionError("a shard of another rank / world size was accepted")
    # the per-name form: sharded -> unsharded -> sharded, and training goes on together
    net_a, ddp_a, opt_a = _engine(False)
    net_a.load_state_dict(net_s.state_dict())
    assert opt_a.load_named_state(net_a, ss) == len(ss) and opt_a.steps == STEPS
    net_b, ddp_b, opt_b = _engine(True)
    net_b.load_state_dict(net_a.state_dict())
    assert opt_b.load_named_state(net_b, opt_a.named_state(net_a)) == len(ss)
    for k in range(len(opt_s.buckets)):
        assert torch.equal(opt_b.exp_avg_flats[k], opt_s.exp_avg_flats[k])
        assert torch.equal(opt_b.exp_avg_sq_flats[k], opt_s.exp_avg_sq_flats[k])
    for it in range(STEPS, STEPS + 2):
        for ddp, opt in ((ddp_s, opt_s), (ddp_a, opt_a), (ddp_b, opt_b)):
            _step(ddp, opt, rank, it)
    for a, b in zip(net_s.parameters(), net_b.parameters()):
        assert torch.equal(a, b)
    _close(net_s, net_a)
    b2.barrier()


def w_contract(rank, size):
    """max_grad_norm is refused with sharded=True; step() needs the step's exchange; one exchange per step."""
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
    _backward(ddp, opt, rank, 1)
    b2.average_gradients(ddp)
    try:
        b2.average_gradients(ddp)                                 # would apply every bucket's update a second time
    except RuntimeError as e:
        assert "twice" in str(e)
    else:
        raise AssertionError("a second exchange in one step passed")
    opt.step()
    b2.barrier()


def w_save(rank, size):
    """Three sharded steps, then a checkpoint through utils.checkpoint (collective: named_state gathers the shards)."""
    net, ddp, opt = _engine(True)
    for it in range(3):
        _step(ddp, opt, rank, it)
    path = os.environ["B2_ADAMW_CKPT"]
    if rank == 0:
        save_checkpoint(path, net, opt, steps=opt.steps)
    else:
        opt.named_state(net)                                      # the gather is collective
    b2.barrier()


def w_load(rank, size):
    """The world-2 sharded checkpoint into world-3 sharded and unsharded optimizers: the shard does not fit, so the per-name
    state is loaded; both then train on together."""
    runs = []
    for sharded in (True, False):
        net, ddp, opt = _engine(sharded)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")                       # "does not fit this optimizer": the shard of world 2
            blob = load_checkpoint(os.environ["B2_ADAMW_CKPT"], net, opt)
        assert opt.steps == 3 and "optim_state" in blob and "momentum" not in blob
        got = opt.named_state(net)
        for n, s in blob["optim_state"].items():
            assert all(torch.equal(got[n][k], s[k]) for k in ("step", "exp_avg", "exp_avg_sq")), n
        for it in range(3, 5):
            _step(ddp, opt, rank, it)
        runs.append(net)
    _close(runs[0], runs[1])
    b2.barrier()


def w_world1(rank, size):
    """One rank: the flag changes nothing (the shard is everything, step() updates)."""
    nets = []
    for sharded in (False, True):
        net = _mlp()
        opt = FlatAdamW(net, sharded=sharded, **HP)
        for it in range(3):
            (net(torch.randn(4, 13, generator=torch.Generator().manual_seed(it)))).pow(2).mean().backward()
            b2.average_gradients(net)
            opt.step()
        assert opt.shard_range(0) == (0, opt.buckets[0].numel) and "sharded" not in opt.state_dict()
        nets.append(net)
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        assert torch.equal(a, b)
