"""Workers of the module-level tests of sharded FlatLAMB / FlatLARS on backend "b200" (tests/test_gpu_sharded_layerwise.py
at world 1, tests/test_gpu_sharded_layerwise_multi.py at 2 or more GPUs)."""
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2

CLS = {"lamb": b2.FlatLAMB, "lars": b2.FlatLARS}
HP = {"lamb": dict(lr=2e-3), "lars": dict(lr=0.3, trust_coefficient=1e-2)}


def _net(dev):
    from dist_tuto.pth_b200.models.resnet import ResNet18
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False   # the same gradients in every run
    torch.manual_seed(0)
    return ResNet18().to(dev)


def _train(kind, sharded, rank, steps, dev, accumulate=False, ema=False, check_sync=False):
    net = _net(dev)
    ddp = b2.DistributedDataParallel(net)
    opt = CLS[kind](ddp, sharded=sharded, **HP[kind])
    avg = b2.FlatEMA(opt, decay=0.9) if ema else None
    g = torch.Generator(device=dev).manual_seed(3 + rank)
    for it in range(steps):
        xs = [torch.randn(16, 3, 32, 32, generator=g, device=dev) for _ in range(2 if accumulate else 1)]
        ts = [torch.randint(0, 10, (16,), generator=g, device=dev) for _ in xs]
        if accumulate:
            with ddp.no_sync():
                F.cross_entropy(ddp(xs[0]), ts[0]).backward()
        if check_sync and it > 0:
            torch.cuda.set_sync_debug_mode("error")
        try:
            F.cross_entropy(ddp(xs[-1]), ts[-1]).backward()
            b2.average_gradients(ddp)
            opt.step()
            if avg is not None:
                avg.update()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return net, ddp, opt, avg


def _flat(net):
    return torch.cat([p.detach().reshape(-1).cpu() for p in net.parameters()])


def w_world1(rank, size):
    """World 1: sharded=True is the unsharded optimizer, bit for bit."""
    dev = torch.device("cuda", torch.cuda.current_device())
    for kind in ("lamb", "lars"):
        a = _train(kind, False, rank, 4, dev)
        b = _train(kind, True, rank, 4, dev)
        assert torch.equal(_flat(a[0]), _flat(b[0])), kind
        assert a[2].trust_ratios(a[0]) == b[2].trust_ratios(b[0]), kind
        for x in (a, b):
            x[1].remove_hooks()


def w_multi(rank, size):
    """W GPUs: sharded against unsharded for 20 steps, replicas and ratios identical on every rank, no host synchronisation
    in backward or step(), a named_state() checkpoint from the sharded optimizer into an unsharded one and back into a
    sharded one, and no_sync() accumulation with FlatEMA against the unsharded optimizer."""
    import torch.distributed as dist
    dev = torch.device("cuda", torch.cuda.current_device())
    for kind in ("lamb", "lars"):
        ref = _train(kind, False, rank, 20, dev)
        sh = _train(kind, True, rank, 20, dev, check_sync=True)
        assert sh[2]._shard_mode == "kernel", kind
        pr, ps = _flat(ref[0]), _flat(sh[0])
        err = float((pr - ps).abs().max())
        assert err <= 1e-3 * float(pr.abs().max()), (kind, err)
        everyone = [None] * size
        dist.all_gather_object(everyone, (ps.numpy().tobytes(), sh[2].trust_ratios(sh[0])))
        assert all(e == everyone[0] for e in everyone), f"{kind}: replicas or ratios differ between ranks"
        # checkpoint: sharded -> unsharded -> sharded, the per-name state unchanged at every hop
        get = (lambda o, net: o.named_state(net)) if kind == "lamb" else (lambda o, net: o.named_momentum(net))  # noqa: E731
        put = (lambda o, net, d: o.load_named_state(net, d)) if kind == "lamb" else (  # noqa: E731
            lambda o, net, d: o.load_named_momentum(net, d))
        named = get(sh[2], sh[0])
        fresh = _train(kind, False, rank, 0, dev)
        put(fresh[2], fresh[0], named)
        again = _train(kind, True, rank, 0, dev)
        put(again[2], again[0], get(fresh[2], fresh[0]))
        for back in (get(fresh[2], fresh[0]), get(again[2], again[0])):
            assert _same_state(named, back), kind
        # no_sync() accumulation with FlatEMA: sharded against unsharded, within the same bound as above
        acc = {s: _train(kind, s, rank, 3, dev, accumulate=True, ema=True) for s in (False, True)}
        ema = {}
        for s, (net, _, _, avg) in acc.items():
            with avg.average_parameters():
                ema[s] = _flat(net)
        for what, a, b in (("parameters", _flat(acc[False][0]), _flat(acc[True][0])), ("EMA", ema[False], ema[True])):
            err = float((a - b).abs().max())
            assert err <= 1e-3 * float(a.abs().max()), (kind, what, err)
        for x in (ref, sh, fresh, again, acc[False], acc[True]):
            x[1].remove_hooks()


def _same_state(a: dict, b: dict) -> bool:
    """Two per-name optimizer states (tensors, or dicts of tensors per name) hold the same bits."""
    if a.keys() != b.keys():
        return False
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, dict):
            if x.keys() != y.keys() or not all(torch.equal(torch.as_tensor(x[s]), torch.as_tensor(y[s])) for s in x):
                return False
        elif not torch.equal(torch.as_tensor(x), torch.as_tensor(y)):
            return False
    return True
