"""Workers of tests/test_param_groups_cpu.py (spawned processes, gloo @127.0.0.1): ``FlatSGD`` / ``FlatAdamW`` with
``param_groups`` on CPU ranks, unsharded and sharded (torch ops on the owned slice), against ``torch.optim.SGD`` /
``torch.optim.AdamW`` with the same groups."""
import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatSGD, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel

STEPS = 20
SCHED = LRSchedule(warmup_steps=3, decay="cosine", total_steps=16, min_factor=0.1)
CHANGE_AT = 11                    # param_groups[1]["lr"] is assigned before this update


def _mlp(seed=3):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(13, 17), nn.Tanh(), nn.Linear(17, 11), nn.LayerNorm(11), nn.Linear(11, 5))


def _groups(net):
    """Three groups: no decay on ndim <= 1, a 10x lr on the last layer's weight; the rest is the default group."""
    no_decay = [p for p in net.parameters() if p.ndim <= 1]
    return [{"params": no_decay, "weight_decay": 0.0}, {"params": [net[4].weight], "lr": 0.1}]


def _backward(ddp, net, rank, it):
    g = torch.Generator().manual_seed(1000 * it + rank)
    x, y = torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)
    (ddp(x) - y).pow(2).mean().backward()


def _bucket_grads(opt, net):
    names = {id(p): n for n, p in net.named_parameters()}
    return {names[id(p)]: gv.float().clone() for gb in opt.buckets for p, gv in zip(gb.params, gb.views)}


CASES = [("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01)),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True)),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.05)),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1)),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05))]


def _pair(kind, hp, sharded, grad_dtype=None):
    """(net, ddp, FlatX with groups, torch reference net, torch optimizer with the same groups)."""
    net = _mlp()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600, grad_dtype=grad_dtype)
    flat_hp = {k: v for k, v in hp.items()}
    Flat = FlatSGD if kind == "sgd" else FlatAdamW
    opt = Flat(ddp, sharded=sharded, zero_grad=False, lr_schedule=SCHED, param_groups=_groups(net), **flat_hp)
    ref = _mlp()
    t_hp = {k: v for k, v in hp.items() if k != "max_grad_norm"}
    Torch = torch.optim.SGD if kind == "sgd" else torch.optim.AdamW
    topt = Torch(_groups(ref) + [{"params": [p for p in ref.parameters() if not any(p is q for g in _groups(ref)
                                                                                   for q in g["params"])]}],
                 foreach=False, **t_hp)
    return net, ddp, opt, ref, topt


def _run_against_torch(rank, kind, hp, sharded, grad_dtype=None, exact=True):
    net, ddp, opt, ref, topt = _pair(kind, hp, sharded, grad_dtype)
    base = [g["lr"] for g in topt.param_groups]
    assert [g["lr"] for g in opt.param_groups] == base and len(opt.param_groups) == 3
    for it in range(STEPS):
        if it == CHANGE_AT:
            opt.param_groups[1]["lr"] = 0.02
            base[1] = 0.02
        opt.zero_grad()
        _backward(ddp, net, rank, it)
        b2.average_gradients(ddp)
        grads = _bucket_grads(opt, net)
        if sharded and opt._shard_mode is not None:       # the exchange applied the update; the bucket holds the average
            pass
        for n, p in ref.named_parameters():
            p.grad = grads[n]
        if "max_grad_norm" in hp:
            rp = dict(ref.named_parameters())
            torch.nn.utils.clip_grad_norm_([rp[n] for n in grads], hp["max_grad_norm"], foreach=False)
        for g, b in zip(topt.param_groups, base):
            g["lr"] = SCHED.lr_at(b, it)
        opt.step()
        topt.step()
        for (n, a), b in zip(net.named_parameters(), ref.parameters()):
            if exact:
                assert torch.equal(a, b), (kind, hp, sharded, it, n, (a - b).abs().max())
            else:
                assert torch.allclose(a, b, atol=1e-6, rtol=1e-5), (kind, hp, sharded, it, n)
    return net, opt


def w_bit_equal_to_torch(rank, size):
    """Unsharded FlatSGD (plain, Nesterov, clip) and FlatAdamW (plain, clip) with three groups, an LRSchedule and a mid-run
    lr change are bit for bit torch's optimizers with the same groups; so is sharded FlatSGD.  Sharded FlatAdamW: replicas
    bit-identical, within a few ulps of torch (torch's vectorised CPU kernels treat the slices' ends in scalar code)."""
    for kind, hp in CASES:
        _run_against_torch(rank, kind, hp, sharded=False)
        if "max_grad_norm" not in hp:
            net, _ = _run_against_torch(rank, kind, hp, sharded=True, exact=kind == "sgd")
            flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
            every = [torch.empty_like(flat) for _ in range(size)]
            b2.all_gather(every, flat)
            assert all(torch.equal(e, flat) for e in every)
    b2.barrier()


def w_no_decay_group(rank, size):
    """With lr 0 on the decayed groups' complement and weight_decay 0 on ndim <= 1, zero gradients leave the no-decay tensors
    exactly as they were (no decay applied) and shrink the others."""
    for Flat, hp in ((FlatSGD, dict(momentum=0.0)), (FlatAdamW, {})):
        for sharded in (False, True):
            net = _mlp()
            ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
            nd = [p for p in net.parameters() if p.ndim <= 1]
            opt = Flat(ddp, lr=0.1, weight_decay=0.5, sharded=sharded, param_groups=[{"params": nd, "weight_decay": 0.0}], **hp)
            before = {n: p.detach().clone() for n, p in net.named_parameters()}
            for _ in range(2):
                opt.zero_grad()
                b2.average_gradients(ddp)          # zero gradients
                opt.step()
            for n, p in net.named_parameters():
                if p.ndim <= 1:
                    assert torch.equal(p, before[n]), (Flat.__name__, sharded, n)
                else:
                    assert p.abs().sum() < before[n].abs().sum(), (Flat.__name__, sharded, n)
    b2.barrier()


def w_checkpoint(rank, size):
    """state_dict carries the groups by name; load_state_dict restores each group's lr / weight_decay, refuses other
    membership, and a state_dict without groups loads as before.  Grouped sharded -> grouped unsharded by name."""
    for Flat, hp in ((FlatSGD, dict(momentum=0.9)), (FlatAdamW, {})):
        net_s, ddp_s, _ = _mlp(), None, None
        ddp_s = DistributedDataParallel(net_s, bucket_cap_bytes=600)
        opt_s = Flat(ddp_s, lr=0.03, weight_decay=0.01, sharded=True, param_groups=_groups(net_s), **hp)
        for it in range(3):
            opt_s.zero_grad()
            _backward(ddp_s, net_s, rank, it)
            b2.average_gradients(ddp_s)
            opt_s.step()
        opt_s.param_groups[0]["lr"] = 0.5
        opt_s.param_groups[2]["weight_decay"] = 0.25
        sd = opt_s.state_dict()
        names = dict(net_s.named_parameters())
        assert [sorted(g["params"]) for g in sd["param_groups"]] == [
            sorted(n for n, p in names.items() if p.ndim <= 1), ["4.weight"],
            sorted(n for n, p in names.items() if p.ndim > 1 and n != "4.weight")]
        assert [g["lr"] for g in sd["param_groups"]] == [0.5, 0.1, 0.03]
        assert opt_s.weight_decay == 0.25 and sd["weight_decay"] == 0.25
        # into an unsharded grouped optimizer: groups from the state_dict, state by name
        net_u = _mlp()
        net_u.load_state_dict(net_s.state_dict())
        ddp_u = DistributedDataParallel(net_u, bucket_cap_bytes=600)
        opt_u = Flat(ddp_u, lr=0.03, weight_decay=0.01, param_groups=_groups(net_u), **hp)
        unsharded = dict(sd)
        for key in ("sharded", "world", "rank", "momentum_buffers", "exp_avg", "exp_avg_sq"):
            unsharded.pop(key, None)
        opt_u._load_group_state(unsharded)
        assert [(g["lr"], g["weight_decay"]) for g in opt_u.param_groups] == [(0.5, 0.0), (0.1, 0.01), (0.03, 0.25)]
        if Flat is FlatSGD:
            assert opt_u.load_named_momentum(net_u, opt_s.named_momentum(net_s)) > 0
        else:
            assert opt_u.load_named_state(net_u, opt_s.named_state(net_s)) > 0
        # the same groups in a sharded one of the same world: round trip
        net_c = _mlp()
        ddp_c = DistributedDataParallel(net_c, bucket_cap_bytes=600)
        opt_c = Flat(ddp_c, lr=0.03, weight_decay=0.01, sharded=True, param_groups=_groups(net_c), **hp)
        opt_c.load_state_dict(sd)
        assert [(g["lr"], g["weight_decay"]) for g in opt_c.param_groups] == [(0.5, 0.0), (0.1, 0.01), (0.03, 0.25)]
        assert opt_c.lr == 0.03 and opt_c.weight_decay == 0.25
        # other membership is refused; a state_dict without groups loads and keeps the groups as built
        net_d = _mlp()
        ddp_d = DistributedDataParallel(net_d, bucket_cap_bytes=600)
        opt_d = Flat(ddp_d, lr=0.03, weight_decay=0.01, sharded=True,
                     param_groups=[{"params": [net_d[0].weight], "lr": 0.5}], **hp)
        try:
            opt_d.load_state_dict(sd)
        except ValueError as e:
            assert "parameter groups" in str(e)
        else:
            raise AssertionError("a state_dict of other groups was accepted")
        plain = {k: v for k, v in sd.items() if k != "param_groups"}
        opt_d.load_state_dict(plain)
        assert opt_d.param_groups[0]["lr"] == 0.5 and opt_d.lr == 0.03
        # an ungrouped optimizer refuses a grouped state_dict of several groups
        net_e = _mlp()
        opt_e = Flat(DistributedDataParallel(net_e, bucket_cap_bytes=600), lr=0.03, sharded=True, **hp)
        assert len(opt_e.param_groups) == 1 and "param_groups" not in opt_e.state_dict()
        try:
            opt_e.load_state_dict(sd)
        except ValueError:
            pass
        else:
            raise AssertionError("an ungrouped optimizer took three groups")
    b2.barrier()


def w_world_change(rank, size):
    """A grouped sharded run of this world size continues as a grouped unsharded run from the per-name state: both stay
    together (SGD: bit for bit)."""
    net_s = _mlp()
    ddp_s = DistributedDataParallel(net_s, bucket_cap_bytes=600)
    opt_s = FlatSGD(ddp_s, lr=0.05, momentum=0.9, weight_decay=0.01, sharded=True, param_groups=_groups(net_s))
    for it in range(3):
        opt_s.zero_grad()
        _backward(ddp_s, net_s, rank, it)
        b2.average_gradients(ddp_s)
        opt_s.step()
    net_u = _mlp()
    net_u.load_state_dict(net_s.state_dict())
    ddp_u = DistributedDataParallel(net_u, bucket_cap_bytes=600)
    opt_u = FlatSGD(ddp_u, lr=0.05, momentum=0.9, weight_decay=0.01, param_groups=_groups(net_u))
    opt_u.load_named_momentum(net_u, opt_s.named_momentum(net_s))
    for it in range(3, 6):
        for ddp, net, opt in ((ddp_s, net_s, opt_s), (ddp_u, net_u, opt_u)):
            opt.zero_grad()
            _backward(ddp, net, rank, it)
            b2.average_gradients(ddp)
            opt.step()
    for a, b in zip(net_s.parameters(), net_u.parameters()):
        assert torch.equal(a, b)
    b2.barrier()
