"""Workers of tests/test_layerwise_cpu.py (gloo CPU ranks) and tests/test_gpu_layerwise.py (``backend="b200"``):
``FlatLAMB`` and ``FlatLARS`` through the public API, against a per-parameter torch-op reference
(tests/layerwise_model.py: the ratio, then LAMB's update or ``torch.optim.SGD(foreach=False)``)."""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
import layerwise_model as L
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatLAMB, FlatLARS, FlatSGD, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel
from dist_tuto.pth_b200.utils.checkpoint import load_checkpoint, save_checkpoint

STEPS = 5
HP = {"lamb": dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1),
      "lars": dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4)}
SCHED = LRSchedule(warmup_steps=2, decay="multistep", milestones=(3,), gamma=0.5)
CLS = {"lamb": FlatLAMB, "lars": FlatLARS}


def _mlp(seed=3):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(13, 17), nn.Tanh(), nn.Linear(17, 11), nn.Tanh(), nn.Linear(11, 5))


def _engine(kind, **kw):
    net = _mlp()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
    return net, ddp, CLS[kind](ddp, **{**HP[kind], **kw})


def _backward(ddp, opt, rank, it):
    g = torch.Generator().manual_seed(1000 * it + rank)
    x, y = torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)
    opt.zero_grad()
    (ddp(x) - y).pow(2).mean().backward()


def _step(ddp, opt, rank, it):
    _backward(ddp, opt, rank, it)
    b2.average_gradients(ddp)
    opt.step()


def _flat1(x):
    """1-D like the optimizer's slices of its flats where the layout allows; a channels_last tensor stays as it is."""
    return x.view(-1) if x.is_contiguous() else x


class RefOpt:
    """The per-parameter torch-op reference of both optimizers on plain parameters (any device)."""

    def __init__(self, named, kind, hp, exclude=None):
        self.named, self.kind, self.t = list(named), kind, 0
        self.hp = dict(hp)
        self.hp.setdefault("nesterov", False)
        ex = exclude or (lambda n, p: p.ndim <= 1)
        self.adapt = [not ex(n, p) for n, p in self.named]
        self.m = [_flat1(torch.zeros_like(p)) for _, p in self.named]      # the parameter's strides (channels_last)
        self.v = [_flat1(torch.zeros_like(p)) for _, p in self.named]
        self.ratios = {}

    def zero_grad(self):
        for _, p in self.named:
            p.grad = None

    @torch.no_grad()
    def step(self, lr=None):
        self.t += 1
        hp = dict(self.hp, lr=self.hp["lr"] if lr is None else lr)
        for (n, p), m, v, ad in zip(self.named, self.m, self.v, self.adapt):
            pf, gf = _flat1(p.data), _flat1(p.grad.float())
            if self.kind == "lamb":
                r = L.torch_lamb_tensor(pf, gf, m, v, ad, hp, self.t)
            else:
                r = L.torch_lars_ratio(pf, gf, ad, hp)
                L.torch_sgd(pf, L.torch_lars_direction(pf, gf, ad, hp, r), m, hp)
            self.ratios[n] = r


def _bucket_grads(opt, net):
    names = {id(p): n for n, p in net.named_parameters()}
    return {names[id(p)]: gv.float().clone() for gb in opt.buckets for p, gv in zip(gb.params, gb.views)}


def _replicas_identical(net, size):
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)


def _custom_exclude(name, p):
    return name.startswith("4.")          # the last layer, weight and bias


def w_bit_equal(rank, size):
    """FlatLAMB / FlatLARS are bit for bit the per-parameter reference with the same averaged gradients: with and
    without weight decay, an LRSchedule, clipping, Nesterov (LARS) and a custom exclude_from_adaptation."""
    for kind in ("lamb", "lars"):
        cases = [{}, dict(weight_decay=0.0), dict(lr_schedule=SCHED), dict(max_grad_norm=0.05),
                 dict(exclude_from_adaptation=_custom_exclude)]
        if kind == "lars":
            cases.append(dict(nesterov=True))
        for kw in cases:
            net, ddp, opt = _engine(kind, zero_grad=False, **kw)
            assert len(opt.buckets) > 2
            ref = _mlp()
            rhp = {**HP[kind], **{k: v for k, v in kw.items() if k in ("weight_decay", "nesterov")}}
            ropt = RefOpt(ref.named_parameters(), kind, rhp, kw.get("exclude_from_adaptation"))
            for it in range(STEPS):
                _backward(ddp, opt, rank, it)
                b2.average_gradients(ddp)
                grads = _bucket_grads(opt, net)
                for n, p in ref.named_parameters():
                    p.grad = grads[n]
                if "max_grad_norm" in kw:
                    rp = dict(ref.named_parameters())
                    tn = torch.nn.utils.clip_grad_norm_([rp[n] for n in grads], kw["max_grad_norm"], foreach=False)
                lr = opt.lr_at()
                opt.step()
                ropt.step(lr)
                if "max_grad_norm" in kw:
                    assert opt.grad_norm() == float(tn)
                for (n, a), b in zip(net.named_parameters(), ref.parameters()):
                    assert torch.equal(a, b), (kind, kw, it, n)
                assert opt.trust_ratios(ddp) == ropt.ratios, (kind, kw, it)
            rs = opt.trust_ratios(net)
            assert all(rs[n] == 1.0 for n, p in net.named_parameters()
                       if (_custom_exclude(n, p) if "exclude_from_adaptation" in kw else p.ndim <= 1))
            assert any(r != 1.0 for r in rs.values())
            _replicas_identical(net, size)
    b2.barrier()


def w_checkpoints(rank, size):
    """state_dict and the per-name forms round-trip; a LAMB state loads into FlatAdamW and LARS momentum into FlatSGD; all
    go on training together."""
    net, ddp, opt = _engine("lamb")
    for it in range(3):
        _step(ddp, opt, rank, it)
    sd, named = opt.state_dict(), opt.named_state(net)
    assert set(named[next(iter(named))]) == {"step", "exp_avg", "exp_avg_sq"}
    net_b, ddp_b, opt_b = _engine("lamb")
    net_b.load_state_dict(net.state_dict())
    opt_b.load_state_dict(sd)
    net_c, ddp_c, opt_c = _engine("lamb")
    net_c.load_state_dict(net.state_dict())
    assert opt_c.load_named_state(net_c, named) == len(named) and opt_c.steps == 3
    for it in range(3, 5):
        for d, o in ((ddp, opt), (ddp_b, opt_b), (ddp_c, opt_c)):
            _step(d, o, rank, it)
    for a, b, c in zip(net.parameters(), net_b.parameters(), net_c.parameters()):
        assert torch.equal(a, b) and torch.equal(a, c)
    net_a = _mlp()
    adam = FlatAdamW(DistributedDataParallel(net_a, bucket_cap_bytes=600))
    assert adam.load_named_state(net_a, opt.named_state(net)) == len(named) and adam.steps == 5
    adam.load_state_dict(opt.state_dict())
    got = adam.named_state(net_a)
    assert all(torch.equal(got[n][k], s[k]) for n, s in opt.named_state(net).items() for k in s)

    net, ddp, opt = _engine("lars", nesterov=True)
    for it in range(3):
        _step(ddp, opt, rank, it)
    sd, mom = opt.state_dict(), opt.named_momentum(net)
    assert sd["trust_coefficient"] == HP["lars"]["trust_coefficient"] and sd["nesterov"] is True
    net_b, ddp_b, opt_b = _engine("lars")
    net_b.load_state_dict(net.state_dict())
    opt_b.load_state_dict(sd)
    assert opt_b.nesterov and opt_b.steps == 3
    net_c, ddp_c, opt_c = _engine("lars", nesterov=True)
    net_c.load_state_dict(net.state_dict())
    assert opt_c.load_named_momentum(net_c, mom) == len(mom)
    for it in range(3, 5):
        for d, o in ((ddp, opt), (ddp_b, opt_b), (ddp_c, opt_c)):
            _step(d, o, rank, it)
    for a, b, c in zip(net.parameters(), net_b.parameters(), net_c.parameters()):
        assert torch.equal(a, b) and torch.equal(a, c)
    net_s = _mlp()
    sgd = FlatSGD(DistributedDataParallel(net_s, bucket_cap_bytes=600))
    assert sgd.load_named_momentum(net_s, opt.named_momentum(net)) == len(mom)
    assert all(torch.equal(sgd.named_momentum(net_s)[n], t) for n, t in opt.named_momentum(net).items())
    # utils.checkpoint carries both through its existing per-name forms
    path = os.path.join(os.environ["B2_LW_CKPT_DIR"], f"r{rank}.pt")
    for kind in ("lamb", "lars"):
        net, ddp, opt = _engine(kind)
        for it in range(2):
            _step(ddp, opt, rank, it)
        save_checkpoint(path, net, opt, steps=opt.steps)
        net_r, ddp_r, opt_r = _engine(kind)
        blob = load_checkpoint(path, net_r, opt_r)
        assert opt_r.steps == 2 and ("optim_state" in blob if kind == "lamb" else "momentum" in blob)
        _step(ddp, opt, rank, 2)
        _step(ddp_r, opt_r, rank, 2)
        for a, b in zip(net.parameters(), net_r.parameters()):
            assert torch.equal(a, b)
    b2.barrier()


def w_refusals(rank, size):
    for kind in ("lamb", "lars"):
        try:
            _engine(kind, sharded=True)
        except ValueError as e:
            assert "sharded" in str(e)
        else:
            raise AssertionError("sharded=True was accepted")
    bad = [("lamb", dict(lr=-1.0)), ("lamb", dict(betas=(1.0, 0.9))), ("lamb", dict(eps=-1.0)),
           ("lamb", dict(weight_decay=-0.1)), ("lars", dict(lr=-1.0)), ("lars", dict(momentum=-0.5)),
           ("lars", dict(trust_coefficient=0.0)), ("lars", dict(eps=-1.0)), ("lars", dict(weight_decay=-1.0)),
           ("lars", dict(momentum=0.0, nesterov=True)), ("lamb", dict(max_grad_norm=-1.0))]
    for kind, kw in bad:
        try:
            _engine(kind, **kw)
        except ValueError:
            pass
        else:
            raise AssertionError(f"{kind} accepted {kw}")
    b2.barrier()


# ----------------------------------------------------------------------------------------------- GPU (one rank)
def w_resnet(rank, size):
    """A ResNet-18 under bf16 autocast: FlatLAMB's and FlatLARS's losses stay close to the torch-op reference's, and
    step() never synchronises the host."""
    from dist_tuto.pth_b200.models.resnet import ResNet18
    dev = torch.device("cuda", torch.cuda.current_device())
    hps = {"lamb": dict(lr=2e-3), "lars": dict(lr=0.3, trust_coefficient=1e-2)}
    for kind in ("lamb", "lars"):
        losses = {}
        for flat in (False, True):
            torch.manual_seed(0)
            net = ResNet18().to(dev).to(memory_format=torch.channels_last)
            ddp = b2.DistributedDataParallel(net)
            opt =CLS[kind](ddp, **hps[kind]) if flat else RefOpt(net.named_parameters(), kind, _defaults(kind, hps[kind]))
            g = torch.Generator(device=dev).manual_seed(3)
            out = []
            for it in range(8):
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


def _defaults(kind, over):
    """The class defaults of the optimizer's hyper-parameters, overridden by ``over``."""
    import inspect
    sig = inspect.signature(CLS[kind].__init__)
    keys = ("lr", "betas", "eps", "weight_decay") if kind == "lamb" else ("lr", "momentum", "weight_decay",
                                                                          "trust_coefficient", "eps", "nesterov")
    return {**{k: sig.parameters[k].default for k in keys}, **over}
