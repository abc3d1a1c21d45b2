"""Workers of tests/test_accumulation_cpu.py (gloo CPU ranks): gradient accumulation with ``DistributedDataParallel.no_sync()``
for every flat optimizer, against a reference without DDP -- the same module and micro-batches, autograd's accumulation into
``p.grad``, an all-reduce average, then ``torch.optim.SGD`` / ``AdamW(foreach=False)`` or the torch-op LAMB / LARS of
tests/layerwise_workers.py, applied once per k micro-batches.

The reference averages its gradients in flat buffers laid out like the DDP buckets (plain ``GradBucket``s, no hooks): gloo's
ring all-reduce adds three ranks' values in an order that depends on an element's position in the buffer, so only the same
layout gives the same bits at world size 3."""
import collections
import contextlib

import torch
import torch.nn as nn

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import FlatAdamW, FlatLAMB, FlatLARS, FlatSGD, LRSchedule
from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel, GradBucket
from layerwise_workers import RefOpt

STEPS = 5
KS = (1, 2, 4)
SCHED = LRSchedule(warmup_steps=2, decay="cosine", total_steps=6, min_factor=0.1)


class Net(nn.Module):
    """An MLP with a side branch that only the first micro-batch of a cycle uses: with k > 1 the last backward fires no
    hook for its parameters, so their bucket goes out from ``finish()``."""

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
            {"params": [net.body[4].weight], "lr": 0.1}]


# (name, kind, flat kwargs, exact): every optimizer and mode; the flat optimizers all take SCHED
CASES = [("sgd momentum wd groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, groups=True), True),
         ("sgd nesterov groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True, groups=True), True),
         ("sgd clip groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.05, groups=True), True),
         ("adamw groups", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, groups=True), True),
         ("adamw clip groups", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05,
                                             groups=True), True),
         ("sgd sharded groups", "sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, sharded=True, groups=True), True),
         # torch's vectorised CPU AdamW treats the ends of the shard slices in scalar code: a few ulps, as in its own tests
         ("adamw sharded groups", "adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, sharded=True,
                                                groups=True), False),
         ("lamb", "lamb", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1), True),
         ("lamb clip", "lamb", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05), True),
         ("lars nesterov", "lars", dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4,
                                         nesterov=True), True),
         ("lars clip", "lars", dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4,
                                     max_grad_norm=0.05), True)]
FLAT = {"sgd": FlatSGD, "adamw": FlatAdamW, "lamb": FlatLAMB, "lars": FlatLARS}


class Exchanges:
    """Counts ``GradBucket.exchange_`` calls per bucket (the all-reduce, or the sharded reduce-scatter + update + gather)."""

    def __init__(self):
        self.calls = collections.Counter()
        self._orig = GradBucket.exchange_
        counter = self

        def counting(gb, *a, **kw):
            counter.calls[id(gb)] += 1
            return counter._orig(gb, *a, **kw)
        GradBucket.exchange_ = counting

    def take(self) -> collections.Counter:
        out, self.calls = self.calls, collections.Counter()
        return out

    def close(self):
        GradBucket.exchange_ = self._orig


def micro_batch(rank, it, j):
    """Micro-batch j of step it: different on every rank."""
    g = torch.Generator().manual_seed(10007 * it + 101 * j + rank)
    return torch.randn(6, 13, generator=g), torch.randn(6, 5, generator=g)


def _loss(model, rank, it, j, k):
    x, y = micro_batch(rank, it, j)
    return (model(x, side=(j == 0)) - y).pow(2).mean() / k


def make(kind, hp):
    """(net, ddp, flat optimizer, reference net, reference optimizer, base lr of each reference group, reference buckets,
    the parameter names in bucket order)."""
    hp = dict(hp)
    groups = hp.pop("groups", False)
    net = Net()
    ddp = DistributedDataParallel(net, bucket_cap_bytes=600)
    kw = dict(lr_schedule=SCHED, **hp)
    if groups:
        kw["param_groups"] = _groups(net)
    opt = FLAT[kind](ddp, **kw)
    ref = Net()
    t_hp = {k: v for k, v in hp.items() if k not in ("max_grad_norm", "sharded")}
    if kind in ("sgd", "adamw"):
        named = {id(q) for g in _groups(ref) for q in g["params"]}
        ref_groups = (_groups(ref) + [{"params": [p for p in ref.parameters() if id(p) not in named]}]) if groups \
            else [{"params": list(ref.parameters())}]
        topt = (torch.optim.SGD if kind == "sgd" else torch.optim.AdamW)(ref_groups, foreach=False, **t_hp)
        base = [g["lr"] for g in topt.param_groups]
    else:
        topt = RefOpt(ref.named_parameters(), kind, t_hp)
        base = [hp["lr"]]
    names = {id(p): n for n, p in net.named_parameters()}
    rp = dict(ref.named_parameters())
    order = [names[id(p)] for gb in ddp.buckets for p in gb.params]
    rbs = [GradBucket([rp[names[id(p)]] for p in gb.params], symmetric=False) for gb in ddp.buckets]
    return net, ddp, opt, ref, topt, base, rbs, order


def ref_cycle(ref, topt, base, rbs, order, kind, hp, rank, it, k):
    """The reference: autograd accumulates the k micro-batches into p.grad, an all-reduce averages them, then the reference
    optimizer steps once (clipping the accumulated average first)."""
    for gb in rbs:
        gb.zero_()
    for j in range(k):
        _loss(ref, rank, it, j, k).backward()
    for gb in rbs:
        gb.all_reduce_average_()
    if "max_grad_norm" in hp:
        rp = dict(ref.named_parameters())
        torch.nn.utils.clip_grad_norm_([rp[n] for n in order], hp["max_grad_norm"], foreach=False)
    if kind in ("sgd", "adamw"):
        for g, b in zip(topt.param_groups, base):
            g["lr"] = SCHED.lr_at(b, it)
        topt.step()
    else:
        topt.step(SCHED.lr_at(base[0], it))


def flat_cycle(ddp, net, opt, rank, it, k, variant, ex):
    """One optimizer step of k micro-batches, the first k - 1 under no_sync().  Variants: "set_to_none" (the inner module's
    zero_grad(set_to_none=True) first), "nested" (nested no_sync), "finish" (all k under no_sync, then average_gradients
    exchanges every bucket), "inner" (average_gradients on the inner module).  Checks that no_sync backwards exchange
    nothing and the cycle exchanges every bucket exactly once."""
    if variant == "set_to_none":
        net.zero_grad(set_to_none=True)
        assert all(p.grad is None for p in net.parameters())
    n_quiet = k if variant == "finish" else k - 1
    for j in range(n_quiet):
        with ddp.no_sync():
            if variant == "nested":
                with ddp.no_sync():
                    _loss(ddp, rank, it, j, k).backward()
                assert not ddp.require_backward_grad_sync
            else:
                _loss(ddp, rank, it, j, k).backward()
        assert ddp.require_backward_grad_sync
        assert not ex.take(), (variant, j)
    if n_quiet < k:
        _loss(ddp, rank, it, k - 1, k).backward()
    b2.average_gradients(net if variant == "inner" else ddp)
    got = ex.take()
    assert sorted(got.values()) == [1] * len(opt.buckets) and set(got) == {id(gb) for gb in opt.buckets}, (variant, got)
    opt.step()


VARIANTS = ("plain", "set_to_none", "nested", "finish", "inner")


def _state(kind, opt, net):
    if kind in ("adamw", "lamb"):
        return {n: (s["exp_avg"], s["exp_avg_sq"]) for n, s in opt.named_state(net).items()}
    return {n: (m,) for n, m in opt.named_momentum(net).items()}


def _ref_state(kind, topt, ref):
    if isinstance(topt, RefOpt):
        if kind == "lamb":
            return {n: (m.view_as(p), v.view_as(p)) for (n, p), m, v in zip(topt.named, topt.m, topt.v)}
        return {n: (m.view_as(p),) for (n, p), m in zip(topt.named, topt.m)}
    st = {}
    for n, p in ref.named_parameters():
        s = topt.state[p]
        st[n] = (s["exp_avg"], s["exp_avg_sq"]) if kind == "adamw" else (s["momentum_buffer"],)
    return st


def _close(a, b, exact):
    return torch.equal(a, b) if exact else torch.allclose(a, b, atol=1e-6, rtol=1e-5)


def replicas_identical(net, size):
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    every = [torch.empty_like(flat) for _ in range(size)]
    b2.all_gather(every, flat)
    assert all(torch.equal(e, flat) for e in every)


def w_against_reference(rank, size):
    """Every optimizer and mode at k = 1, 2, 4 over STEPS steps (one variant per step): parameters and optimizer state
    equal the reference's (bit for bit where the optimizer's own tests are), ``steps`` counts optimizer steps, and the
    replicas are identical."""
    ex = Exchanges()
    try:
        for name, kind, hp, exact in CASES:
            for k in KS:
                net, ddp, opt, ref, topt, base, rbs, order = make(kind, hp)
                assert len(opt.buckets) > 2
                for it in range(STEPS):
                    flat_cycle(ddp, net, opt, rank, it, k, VARIANTS[it % len(VARIANTS)], ex)
                    ref_cycle(ref, topt, base, rbs, order, kind, hp, rank, it, k)
                    for (n, a), b in zip(net.named_parameters(), ref.parameters()):
                        assert _close(a, b, exact), (name, k, it, n, (a - b).abs().max())
                assert opt.steps == STEPS
                st, rst = _state(kind, opt, net), _ref_state(kind, topt, ref)
                for n in rst:
                    for a, b in zip(st[n], rst[n]):
                        assert _close(a, b, exact), (name, k, n)
                replicas_identical(net, size)
                ddp.remove_hooks()
    finally:
        ex.close()
    b2.barrier()


def w_errors(rank, size):
    """average_gradients inside no_sync() and step() after no_sync backwards only raise RuntimeError and exchange nothing;
    the cycle then completes correctly and equals the reference."""
    ex = Exchanges()
    try:
        for name, kind, hp, exact in [CASES[0], CASES[3], CASES[5], CASES[6], CASES[7]]:
            net, ddp, opt, ref, topt, base, rbs, order = make(kind, hp)
            k = 2
            for it in range(3):
                before = [p.detach().clone() for p in net.parameters()]
                with ddp.no_sync():
                    _loss(ddp, rank, it, 0, k).backward()
                    if it == 0:                  # average_gradients inside no_sync(), on the wrapper and the inner module
                        for m in (ddp, net):
                            with contextlib.suppress(RuntimeError):
                                b2.average_gradients(m)
                                raise AssertionError(f"{name}: average_gradients inside no_sync() was accepted")
                    if it == 1:
                        _loss(ddp, rank, it, 1, k).backward()
                if it == 1:                      # every micro-batch under no_sync, then step() without an exchange
                    msg = "were not exchanged" if opt._shard_mode is not None else "never exchanged"
                    try:
                        opt.step()
                    except RuntimeError as e:
                        assert msg in str(e), (name, str(e))
                    else:
                        raise AssertionError(f"{name}: step() after no_sync backwards only was accepted")
                    assert opt.steps == 1, name
                assert not ex.take(), name
                assert all(torch.equal(a, b) for a, b in zip(before, net.parameters())), name
                if it != 1:
                    _loss(ddp, rank, it, 1, k).backward()
                b2.average_gradients(ddp)
                assert sorted(ex.take().values()) == [1] * len(opt.buckets), name
                opt.step()
                ref_cycle(ref, topt, base, rbs, order, kind, hp, rank, it, k)
                for (n, a), b in zip(net.named_parameters(), ref.parameters()):
                    assert _close(a, b, exact), (name, it, n)
            assert opt.steps == 3
            replicas_identical(net, size)
            ddp.remove_hooks()
    finally:
        ex.close()
    b2.barrier()


# ----------------------------------------------------------------------------------------------- GPU (backend "b200")
def gpu_optimizers(sharded=False):
    """(name, constructor) of every optimizer on its CUDA kernel path (fp32 buckets); ``sharded``: FlatSGD and FlatAdamW
    with sharded=True, which cannot clip."""
    def groups(m):
        return [{"params": [p for p in m.parameters() if p.ndim <= 1], "weight_decay": 0.0, "lr": 0.02}]
    sched = LRSchedule(warmup_steps=2, decay="cosine", total_steps=8, min_factor=0.1)
    clip = {} if sharded else dict(max_grad_norm=0.5)
    out = [("sgd nesterov groups", lambda ddp, m: FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True,
                                                          param_groups=groups(m), lr_schedule=sched, sharded=sharded,
                                                          **clip)),
           ("adamw groups", lambda ddp, m: FlatAdamW(ddp, lr=3e-3, weight_decay=0.05, param_groups=groups(m),
                                                     lr_schedule=sched, sharded=sharded, **clip))]
    if not sharded:
        out += [("lamb", lambda ddp, m: FlatLAMB(ddp, lr=2e-3, lr_schedule=sched, **clip)),
                ("lars", lambda ddp, m: FlatLARS(ddp, lr=0.3, trust_coefficient=1e-2, lr_schedule=sched, **clip))]
    return out


def gpu_model(name, dev):
    """(module, micro-batch maker, loss) of "resnet" (ResNet-18, bf16 autocast, channels_last) or "net" (the tutorial's
    MNIST Net, fp32, dropout on)."""
    import torch.nn.functional as F
    from dist_tuto.pth_b200.models.convnet import Net as TutorialNet
    from dist_tuto.pth_b200.models.resnet import ResNet18

    torch.manual_seed(0)
    if name == "resnet":
        m = ResNet18().to(dev).to(memory_format=torch.channels_last)

        def data(g):
            return (torch.randn(16, 3, 32, 32, generator=g, device=dev).contiguous(memory_format=torch.channels_last),
                    torch.randint(0, 10, (16,), generator=g, device=dev))

        def loss(model, x, y):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return F.cross_entropy(model(x), y)
        return m, data, loss
    m = TutorialNet().to(dev)

    def data(g):
        return torch.randn(32, 1, 28, 28, generator=g, device=dev), torch.randint(0, 10, (32,), generator=g, device=dev)
    return m, data, lambda model, x, y: F.nll_loss(model(x), y)


def gpu_micro(data, dev, rank, it, j):
    return data(torch.Generator(device=dev).manual_seed(10007 * it + 101 * j + rank))


def accumulated_cycle(ddp, opt, data, loss_fn, dev, rank, it, k, debug_sync=False):
    """k micro-batches, the first k - 1 under no_sync(), average_gradients, step(); with ``debug_sync`` the backwards and
    step() run under ``torch.cuda.set_sync_debug_mode("error")``."""
    batches = [gpu_micro(data, dev, rank, it, j) for j in range(k)]
    if debug_sync:
        torch.cuda.set_sync_debug_mode("error")
    try:
        for j, (x, y) in enumerate(batches):
            torch.manual_seed(7 * it + j)                   # the reference's dropout masks
            with ddp.no_sync() if j < k - 1 else contextlib.nullcontext():
                (loss_fn(ddp, x, y) / k).backward()
        b2.average_gradients(ddp)
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)


def reference_cycle(ddp, opt, data, loss_fn, dev, rank, it, k):
    """The same optimizer applied once to the autograd-accumulated sum: each micro-batch's gradient from
    ``torch.autograd.grad`` (no hook fires) is added into ``p.grad`` in micro-batch order, as autograd accumulates, then
    ``average_gradients`` exchanges every bucket from ``finish()`` and ``step()`` updates.  The flat optimizer is the
    reference here because its CUDA kernels do not round like torch's optimizers; their own tests bound that."""
    params = [p for p in ddp.module.parameters() if p.requires_grad]
    for j in range(k):
        x, y = gpu_micro(data, dev, rank, it, j)
        torch.manual_seed(7 * it + j)
        grads = torch.autograd.grad(loss_fn(ddp, x, y) / k, params)
        with torch.no_grad():
            for p, g in zip(params, grads):
                p.grad.add_(g)
    b2.average_gradients(ddp)
    opt.step()


def gpu_state(m, opt):
    """Parameters, buffers and the optimizer's state flats (this rank's slices when sharded), as raw bytes."""
    flats = [f for name in ("momentum_flats", "exp_avg_flats", "exp_avg_sq_flats") for f in getattr(opt, name, [])]
    ts = [t.detach().reshape(-1) for t in m.state_dict().values()] + [f.reshape(-1) for f in flats]
    return [t.clone().view(torch.uint8) for t in ts]


def gpu_equal(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def w_gpu_against_reference(rank, size, models=("resnet", "net"), k=4, steps=3, sharded=(False,)):
    """Each model and optimizer on its kernel path: k-micro-batch cycles under no_sync() equal the reference bit for bit
    (fp32 buckets), with the micro-batches and step() under the sync debug mode from the second cycle on, and the
    replicated state is the same on every rank."""
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False   # two engines, one backward each
    try:
        for model_name in models:
            for sh in sharded:
                for name, make in gpu_optimizers(sh):
                    engines = []
                    for _ in range(2):
                        m, data, loss_fn = gpu_model(model_name, dev)
                        ddp = b2.DistributedDataParallel(m, bucket_cap_bytes=4 << 20)
                        engines.append((m, ddp, make(ddp, m)))
                    (ma, da, oa), (mb, db, ob) = engines
                    for it in range(steps):
                        accumulated_cycle(da, oa, data, loss_fn, dev, rank, it, k, debug_sync=it > 0)
                        reference_cycle(db, ob, data, loss_fn, dev, rank, it, k)
                        assert gpu_equal(gpu_state(ma, oa), gpu_state(mb, ob)), (model_name, name, sh, it, rank)
                    assert oa.steps == steps
                    if size > 1:
                        replicated = gpu_state(ma, oa)[:len(ma.state_dict())] + ([] if sh else gpu_state(ma, oa))
                        flat = torch.cat(replicated)
                        every = [torch.empty_like(flat) for _ in range(size)]
                        torch.distributed.all_gather(every, flat)
                        assert all(torch.equal(e, flat) for e in every), (model_name, name, sh)
                    da.remove_hooks()
                    db.remove_hooks()
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


def w_gpu_multi(rank, size):
    """Real ranks, overlap on: sharded and unsharded against the reference and across ranks, and a torch.profiler count
    of the exchange kernels: a k = 4 cycle launches as many as a k = 1 cycle, once per bucket per optimizer step."""
    w_gpu_against_reference(rank, size, models=("resnet",), k=4, steps=2, sharded=(False, True))
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda", rank)
    ex = Exchanges()
    try:
        for sh in (False, True):
            name, make = gpu_optimizers(sh)[0]
            m, data, loss_fn = gpu_model("resnet", dev)
            ddp = b2.DistributedDataParallel(m, bucket_cap_bytes=4 << 20)
            assert ddp.overlap
            opt = make(ddp, m)
            accumulated_cycle(ddp, opt, data, loss_fn, dev, rank, 0, 1)          # warm-up
            ex.take()
            counts = {}
            for it, k in ((1, 1), (2, 4)):
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    accumulated_cycle(ddp, opt, data, loss_fn, dev, rank, it, k)
                    torch.cuda.synchronize()
                assert sorted(ex.take().values()) == [1] * len(ddp.buckets), (sh, k)
                counts[k] = sum(e.count for e in prof.key_averages()
                                if "allreduce_" in e.key or "sharded_step_kernel" in e.key)
            assert counts[1] == counts[4] and counts[1] % len(ddp.buckets) == 0 and counts[1] > 0, (sh, counts)
            ddp.remove_hooks()
    finally:
        ex.close()


GRAPH_WARMUP = 3


def graph_cycles(make, n, graph, dev, k=4, warmup=GRAPH_WARMUP):
    """``warmup`` eager k-micro-batch cycles, then ``n`` more: eager, or replays of one captured cycle.  Model and
    optimizers of tests/capturable_workers.py (SyncBatchNorm, groups, clipping, schedules).  Returns (state, optimizer,
    the optimizer steps the replays or eager cycles added)."""
    import torch.nn.functional as F

    import capturable_workers as CW
    torch.manual_seed(7)
    m = CW.net().to(dev).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(m)
    opt = make(ddp, m, capturable=True)
    gen = torch.Generator().manual_seed(100)
    xs = [[torch.randn(8, 3, 12, 12, generator=gen).to(dev).contiguous(memory_format=torch.channels_last)
           for _ in range(k)] for _ in range(warmup + n)]
    ys = [[torch.randint(0, 10, (8,), generator=gen).to(dev) for _ in range(k)] for _ in range(warmup + n)]
    x, y = [t.clone() for t in xs[0]], [t.clone() for t in ys[0]]

    def load(i):
        for a, b in zip(x + y, xs[i] + ys[i]):
            a.copy_(b)

    def cycle():
        for j in range(k - 1):
            with ddp.no_sync():
                (F.cross_entropy(ddp(x[j]), y[j]) / k).backward()
        (F.cross_entropy(ddp(x[k - 1]), y[k - 1]) / k).backward()
        b2.average_gradients(ddp)
        opt.step()

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):                           # warm-up on a side stream, as torch requires before a capture
        for i in range(warmup):
            load(i)
            cycle()
    torch.cuda.current_stream(dev).wait_stream(s)
    before = opt.steps
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cycle()
        for i in range(warmup, warmup + n):
            load(i)
            g.replay()
    else:
        for i in range(warmup, warmup + n):
            load(i)
            cycle()
    torch.cuda.synchronize(dev)
    ddp.remove_hooks()
    return CW.state(m, opt), opt, opt.steps - before
