"""Workers of tests/test_rmsprop_cpu.py (spawned processes, gloo @127.0.0.1): ``FlatRMSprop`` on CPU ranks against a
reference without DDP -- the same module and micro-batches, autograd's accumulation into ``p.grad``, an all-reduce average in
flat buffers laid out like the DDP buckets (gloo's ring adds three ranks' values in an order that depends on the position in
the buffer, so only the same layout gives the same bits), then ``torch.optim.RMSprop(foreach=False)``, driven by its own
``torch.amp.GradScaler("cpu")`` in the scaled cases."""
import os
import warnings

import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatEMA, FlatRMSprop, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel, GradBucket
from dist_tuto.pth_b200.utils.checkpoint import load_checkpoint, save_checkpoint

STEPS = 6
SCHED = LRSchedule(warmup_steps=2, decay="cosine", total_steps=7, min_factor=0.1)
POISON = {2: float("inf"), 4: float("nan")}        # step -> factor of rank 0's loss in the scaled cases
KEYS = ("step", "square_avg", "momentum_buffer", "grad_avg")
# sharded CPU runs update slices that start at other offsets than the per-tensor views: torch's vectorised CPU kernels treat
# the ends of a tensor in scalar code, so the two agree to a few ulps
ATOL, RTOL = 1e-6, 1e-5

# (name, FlatRMSprop kwargs, micro-batches per step, GradScaler): every momentum x centered combination, weight decay, groups,
# clipping and the schedule, accumulation and loss scaling; the sharded cases run the torch-op slice update
CASES = [
    ("plain", dict(lr=0.01, alpha=0.99, eps=1e-8), 1, False),
    ("momentum decay", dict(lr=0.01, alpha=0.9, eps=1e-3, momentum=0.9, weight_decay=0.01), 2, False),
    ("centered decay groups", dict(lr=0.01, alpha=0.9, eps=1e-3, centered=True, weight_decay=0.01, groups=True), 1, False),
    ("momentum centered clip groups", dict(lr=0.01, alpha=0.3, eps=1e-6, momentum=0.5, centered=True, weight_decay=0.05,
                                           max_grad_norm=0.05, groups=True), 2, False),
    ("recipe clip", dict(lr=0.01, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4, max_grad_norm=0.05), 1, False),
    ("recipe scaled", dict(lr=0.01, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4), 1, True),
    ("centered groups clip scaled", dict(lr=0.01, alpha=0.9, eps=1e-3, centered=True, weight_decay=0.01, groups=True,
                                         max_grad_norm=0.05), 2, True),
    ("sharded momentum centered groups", dict(lr=0.01, alpha=0.9, eps=1e-3, momentum=0.9, centered=True, weight_decay=0.01,
                                              groups=True, sharded=True), 2, False),
    ("sharded plain", dict(lr=0.01, alpha=0.99, eps=1e-8, sharded=True), 1, False),
]


class Net(nn.Module):
    """An MLP with a side branch that only the first micro-batch of a cycle uses (its bucket goes out from ``finish()``)."""

    def __init__(self, seed=3):
        super().__init__()
        torch.manual_seed(seed)
        self.body = nn.Sequential(nn.Linear(13, 17), nn.Tanh(), nn.Linear(17, 11), nn.LayerNorm(11), nn.Linear(11, 5))
        self.side = nn.Linear(13, 5)

    def forward(self, x, side=False):
        y = self.body(x)
        return y + self.side(x) if side else y


def _groups(net):
    return [{"params": [p for p in net.parameters() if p.ndim <= 1], "weight_decay": 0.0},
            {"params": [net.body[4].weight], "lr": 0.03}]


def _loss(model, rank, it, j, k, poison=1.0):
    g = torch.Generator().manual_seed(10007 * it + 101 * j + rank)
    x, y = torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)
    return (model(x, side=(j == 0)) - y).pow(2).mean() / k * poison


def make(hp, sharded=None):
    """(net, ddp, FlatRMSprop, reference net, torch.optim.RMSprop, base lr of each reference group, reference buckets, the
    parameter names in bucket order)."""
    hp = dict(hp)
    groups = hp.pop("groups", False)
    if sharded is not None:
        hp["sharded"] = sharded
    net = Net()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
    opt = FlatRMSprop(ddp, lr_schedule=SCHED, param_groups=_groups(net) if groups else None, **hp)
    ref = Net()
    t_hp = {k: v for k, v in hp.items() if k not in ("max_grad_norm", "sharded")}
    named = {id(q) for g in _groups(ref) for q in g["params"]}
    ref_groups = (_groups(ref) + [{"params": [p for p in ref.parameters() if id(p) not in named]}]) if groups \
        else [{"params": list(ref.parameters())}]
    topt = torch.optim.RMSprop(ref_groups, foreach=False, **t_hp)
    base = [g["lr"] for g in topt.param_groups]
    names = {id(p): n for n, p in net.named_parameters()}
    rp = dict(ref.named_parameters())
    order = [names[id(p)] for gb in ddp.buckets for p in gb.params]
    rbs = [GradBucket([rp[names[id(p)]] for p in gb.params], symmetric=False) for gb in ddp.buckets]
    return net, ddp, opt, ref, topt, base, rbs, order


def _backward(model, rank, it, k, scaler=None, poison=1.0):
    """k micro-batches, all but the last under no_sync() when ``model`` is a DDP wrapper."""
    for j in range(k):
        loss = _loss(model, rank, it, j, k, poison)
        loss = scaler.scale(loss) if scaler is not None else loss
        if j < k - 1 and hasattr(model, "no_sync"):
            with model.no_sync():
                loss.backward()
        else:
            loss.backward()


def _scaler():
    return torch.amp.GradScaler("cpu", init_scale=1000.0, growth_interval=3)


def _equal(a, b, exact):
    return torch.equal(a, b) if exact else torch.allclose(a, b, atol=ATOL, rtol=RTOL)


def compare(net, opt, ref, topt, exact, what):
    rp = dict(ref.named_parameters())
    for n, p in net.named_parameters():
        assert _equal(p, rp[n], exact), (what, n)
    mine = opt.named_state(net)                                    # collective when sharded
    for n, p in ref.named_parameters():
        st = topt.state[p]
        assert set(mine[n]) == set(st), (what, n, set(mine[n]), set(st))
        for key in st:
            assert _equal(mine[n][key], st[key], exact or key == "step"), (what, n, key)


def w_against_torch(rank, size, case):
    """One case of CASES for STEPS steps: parameters and every state bit for bit torch.optim.RMSprop(foreach=False) (within
    ATOL / RTOL on the sharded torch-op path), the scalers' scale and growth tracker equal, skipped steps skipped on every
    rank with the buckets zeroed, and the replicas identical."""
    name, hp, k, scaled = next(c for c in CASES if c[0] == case)
    exact = not hp.get("sharded", False) or size == 1
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
            assert scaler.get_scale() == rscaler.get_scale() and torch.equal(scaler._growth_tracker, rscaler._growth_tracker)
            assert skipped == (it in POISON), (it, skipped)
            if skipped:
                assert all(not gb.flat.any() for gb in opt.buckets), "a skipped step leaves the buckets zeroed"
        else:
            topt.step()
        applied += not skipped
        assert opt.steps == applied
        if "max_grad_norm" in hp and not skipped:
            assert opt.grad_norm() == float(tn), (name, it)
        compare(net, opt, ref, topt, exact, (name, it))
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)                        # replicas bit-identical
    ddp.remove_hooks()
    b2.barrier()


def w_all_cases(rank, size):
    """Every case of CASES, in one group of processes."""
    for case in CASES:
        w_against_torch(rank, size, case[0])


def w_ema(rank, size):
    """FlatEMA over FlatRMSprop (unsharded and sharded): the EMA equals torch._foreach_copy_ / _foreach_lerp_ over the
    reference's parameters driven by the same rule (copy at the first update, then lerp with 1 - decay)."""
    hp = dict(lr=0.01, alpha=0.9, eps=1e-3, momentum=0.9, centered=True, weight_decay=0.01)
    for sharded in (False, True):
        net, ddp, opt, ref, topt, base, rbs, order = make(hp, sharded=sharded)
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
        exact = not sharded or size == 1
        for (n, _), e in zip(ref.named_parameters(), rema):
            assert _equal(got[n], e, exact), (sharded, n)
        ddp.remove_hooks()
    b2.barrier()


def w_checkpoints(rank, size):
    """state_dict shards load on their own rank and world size only; whole buffers load into a sharded optimizer as this
    rank's slice; named_state crosses sharded -> unsharded -> sharded and training goes on together; a state_dict of another
    centered / momentum setting is refused."""
    hp = dict(lr=0.01, alpha=0.9, eps=1e-3, momentum=0.9, centered=True, weight_decay=0.01)

    def steps(ddp, opt, first, n):
        for it in range(first, first + n):
            opt.zero_grad()
            _backward(ddp, rank, it, 1)
            b2.average_gradients(ddp)
            opt.step()

    net_u, ddp_u, opt_u = make(hp, sharded=False)[:3]
    net_s, ddp_s, opt_s = make(hp, sharded=True)[:3]
    steps(ddp_u, opt_u, 0, 3)
    steps(ddp_s, opt_s, 0, 3)
    for k, gb in enumerate(opt_s.buckets):
        per = opt_s.square_avg_flats[k].numel()
        assert per == opt_s.grad_avg_flats[k].numel() == opt_s.momentum_buffer_flats[k].numel() < gb.numel
    sd = opt_s.state_dict()
    assert sd["sharded"] is True and (sd["world"], sd["rank"]) == (size, rank) and "sharded" not in opt_u.state_dict()
    net_c, ddp_c, opt_c = make(hp, sharded=True)[:3]
    opt_c.load_state_dict(sd)
    assert opt_c.steps == 3 and all(torch.equal(a, b) for a, b in zip(opt_c.grad_avg_flats, opt_s.grad_avg_flats))
    opt_c.load_state_dict(opt_u.state_dict())
    for k in range(len(opt_s.buckets)):
        lo, hi = opt_c.shard_range(k)
        assert torch.equal(opt_c.momentum_buffer_flats[k][:hi - lo], opt_u.momentum_buffer_flats[k][lo:hi])
    for bad in (dict(sd, rank=(rank + 1) % size), dict(sd, world=size + 1)):
        try:
            opt_c.load_state_dict(bad)
        except ValueError as e:
            assert "named_state" in str(e)
        else:
            raise AssertionError("a shard of another rank / world size was accepted")
    other = make(dict(hp, centered=False), sharded=True)[2]
    for bad_sd in (sd, dict(opt_u.state_dict(), momentum=0.0)):
        try:
            other.load_state_dict(bad_sd) if bad_sd is sd else opt_c.load_state_dict(bad_sd)
        except ValueError as e:
            assert "centered" in str(e)
        else:
            raise AssertionError("a state_dict of another centered / momentum setting was accepted")
    ss = opt_s.named_state(net_s)                                         # collective
    net_a, ddp_a, opt_a = make(hp, sharded=False)[:3]
    net_a.load_state_dict(net_s.state_dict())
    assert opt_a.load_named_state(net_a, ss) == len(ss) and opt_a.steps == 3
    net_b, ddp_b, opt_b = make(hp, sharded=True)[:3]
    net_b.load_state_dict(net_a.state_dict())
    assert opt_b.load_named_state(net_b, opt_a.named_state(net_a)) == len(ss)
    for k in range(len(opt_s.buckets)):
        for name in ("square_avg_flats", "grad_avg_flats", "momentum_buffer_flats"):
            assert torch.equal(getattr(opt_b, name)[k], getattr(opt_s, name)[k]), name
    try:
        make(dict(hp, centered=False, momentum=0.0), sharded=False)[2].load_named_state(net_a, {n: {"step": s["step"]}
                                                                                               for n, s in ss.items()})
    except ValueError as e:
        assert "square_avg" in str(e)
    else:
        raise AssertionError("a per-name state without square_avg was accepted")
    for ddp, opt in ((ddp_s, opt_s), (ddp_a, opt_a), (ddp_b, opt_b)):
        steps(ddp, opt, 3, 2)
    for a, b in zip(net_s.parameters(), net_b.parameters()):
        assert torch.equal(a, b)
    for a, b in zip(net_s.parameters(), net_a.parameters()):
        assert torch.allclose(a, b, atol=ATOL, rtol=RTOL)
    b2.barrier()


def w_named_state_round_trip(rank, size):
    """named_state loads into torch.optim.RMSprop and back, and the three runs continue identically."""
    hp = dict(lr=0.01, alpha=0.9, eps=1e-3, momentum=0.9, centered=True, weight_decay=0.01)
    net, ddp, opt = make(hp)[:3]
    for it in range(3):
        opt.zero_grad()
        _backward(ddp, rank, it, 1)
        b2.average_gradients(ddp)
        opt.step()
    named = opt.named_state(net)
    ref = Net()
    ref.load_state_dict(net.state_dict())
    topt = torch.optim.RMSprop(ref.parameters(), foreach=False, **hp)
    idx = {n: i for i, (n, _) in enumerate(ref.named_parameters())}
    sd = topt.state_dict()
    sd["state"] = {idx[n]: {k: v.clone() for k, v in s.items()} for n, s in named.items()}
    topt.load_state_dict(sd)
    net_b, ddp_b, opt_b = make(hp)[:3]                                    # back: torch's state into a fresh FlatRMSprop
    net_b.load_state_dict(ref.state_dict())
    back = {n: topt.state[p] for n, p in ref.named_parameters()}
    assert opt_b.load_named_state(net_b, back) == len(back) and opt_b.steps == 3
    names = {id(p): n for n, p in net.named_parameters()}
    for it in range(3, 5):
        for ddp_, opt_ in ((ddp, opt), (ddp_b, opt_b)):
            opt_.zero_grad()
            _backward(ddp_, rank, it, 1)
            b2.average_gradients(ddp_)
        grads = {names[id(p)]: gv.clone() for gb in opt.buckets for p, gv in zip(gb.params, gb.views)}
        for n, p in ref.named_parameters():
            p.grad = grads[n]
        topt.param_groups[0]["lr"] = SCHED.lr_at(hp["lr"], it)
        opt.step()
        opt_b.step()
        topt.step()
        for (n, a), b, c in zip(net.named_parameters(), ref.parameters(), net_b.parameters()):
            assert torch.equal(a, b) and torch.equal(a, c), (it, n)
    b2.barrier()


def w_save(rank, size):
    """Three sharded steps, then a checkpoint through utils.checkpoint (collective: named_state gathers the shards)."""
    net, ddp, opt = make(dict(lr=0.01, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4), sharded=True)[:3]
    for it in range(3):
        opt.zero_grad()
        _backward(ddp, rank, it, 1)
        b2.average_gradients(ddp)
        opt.step()
    path = os.environ["B2_RMSPROP_CKPT"]
    if rank == 0:
        save_checkpoint(path, net, opt, steps=opt.steps)
    else:
        opt.named_state(net)                                               # the gather is collective
    b2.barrier()


def w_load(rank, size):
    """The world-2 sharded checkpoint into world-3 sharded and unsharded optimizers: the shard does not fit, so the per-name
    state is loaded; both then train on together."""
    runs = []
    for sharded in (True, False):
        net, ddp, opt = make(dict(lr=0.01, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4), sharded=sharded)[:3]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")                                # "does not fit this optimizer": the shard of world 2
            blob = load_checkpoint(os.environ["B2_RMSPROP_CKPT"], net, opt)
        assert opt.steps == 3 and "optim_state" in blob
        got = opt.named_state(net)
        for n, s in blob["optim_state"].items():
            assert set(s) == {"step", "square_avg", "momentum_buffer"}
            assert all(torch.equal(got[n][k], s[k]) for k in s), n
        for it in range(3, 5):
            opt.zero_grad()
            _backward(ddp, rank, it, 1)
            b2.average_gradients(ddp)
            opt.step()
        runs.append(net)
    for a, b in zip(runs[0].parameters(), runs[1].parameters()):
        assert torch.allclose(a, b, atol=ATOL, rtol=RTOL)
    b2.barrier()


def w_contract(rank, size):
    """Sharded refusals inherited unchanged: clipping, a second exchange per step, step() without an exchange, and
    GradScaler over more than one rank."""
    try:
        make(dict(lr=0.01, max_grad_norm=1.0), sharded=True)
    except ValueError as e:
        assert "sharded" in str(e)
    else:
        raise AssertionError("sharded=True accepted max_grad_norm")
    net, ddp, opt = make(dict(lr=0.01, momentum=0.9), sharded=True)[:3]
    try:
        opt.step()
    except RuntimeError as e:
        assert "average_gradients" in str(e)
    else:
        raise AssertionError("step() without an exchange passed")
    _backward(ddp, rank, 0, 1)
    b2.average_gradients(ddp)
    try:
        b2.average_gradients(ddp)
    except RuntimeError as e:
        assert "twice" in str(e)
    else:
        raise AssertionError("a second exchange in one step passed")
    opt.step()
    net, ddp, opt = make(dict(lr=0.01, momentum=0.9), sharded=True)[:3]
    scaler = _scaler()
    _backward(ddp, rank, 0, 1, scaler)
    b2.average_gradients(ddp)
    try:
        scaler.step(opt)
    except RuntimeError as e:
        assert "sharded=False" in str(e) and "scaled gradient" in str(e), e
    else:
        raise AssertionError("a sharded GradScaler step over several ranks passed")
    assert opt.steps == 0
    b2.barrier()
