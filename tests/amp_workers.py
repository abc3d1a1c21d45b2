"""Workers of tests/test_amp_cpu.py (gloo CPU ranks): the flat optimizers driven by ``torch.amp.GradScaler("cpu")`` against
``torch.optim.SGD`` / ``AdamW(foreach=False)`` driven by their own scaler, on the module, micro-batches, bucket layout and
schedule of tests/accumulation_workers.py.  Rank 0's loss is multiplied by inf or NaN at some steps, so those steps overflow
on one rank only and every rank must skip them; ``init_scale`` is 1000, not a power of two, so unscaling rounds."""
import torch

import dist_tuto.pth_b200 as b2
from accumulation_workers import SCHED, _loss, _ref_state, _state, make, replicas_identical
from dist_tuto.pth_b200.ops.optim import FlatLAMB, FlatLARS

STEPS = 9
POISON = {2: float("inf"), 5: float("nan")}        # step -> factor of rank 0's loss at that step


def _scaler():
    return torch.amp.GradScaler("cpu", init_scale=1000.0, growth_interval=3)


def _poison(rank, it):
    return POISON.get(it, 1.0) if rank == 0 else 1.0


def _scaled_backward(model, scaler, rank, it, k):
    """k micro-batches (all but the last under no_sync() when ``model`` is a DDP wrapper), each loss scaled."""
    for j in range(k):
        loss = _loss(model, rank, it, j, k) * _poison(rank, it)
        if j < k - 1 and hasattr(model, "no_sync"):
            with model.no_sync():
                scaler.scale(loss).backward()
        else:
            scaler.scale(loss).backward()


def _snapshot(kind, opt, net):
    return ([p.detach().clone() for p in net.parameters()], _state(kind, opt, net), opt.steps)


def w_against_torch(rank, size, kind, hp, explicit, k):
    """``scaler.step(opt)`` (or, ``explicit``, ``scaler.unscale_(opt)``, ``clip_grad_norm_`` and ``scaler.step(opt)``) on a
    flat optimizer, against the torch optimizer with its own scaler; every step compares parameters, state, steps, the
    scale and the growth tracker bit for bit.  A skipped step leaves parameters, state and steps as they were, and the
    buckets zero."""
    hp = dict(hp)
    clip = hp.pop("max_grad_norm", None) if explicit else hp.get("max_grad_norm")
    net, ddp, opt, ref, topt, base, rbs, order = make(kind, hp)
    scaler, rscaler = _scaler(), _scaler()
    applied = 0
    for it in range(STEPS):
        before = _snapshot(kind, opt, net)
        _scaled_backward(ddp, scaler, rank, it, k)
        b2.average_gradients(ddp)
        if explicit:
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_([p for gb in opt.buckets for p in gb.params], clip, foreach=False)
        scaler.step(opt)
        scaler.update()
        # the reference: autograd into p.grad, the average in buckets laid out like DDP's, torch's scaler and optimizer
        for gb in rbs:
            gb.zero_()
        _scaled_backward(ref, rscaler, rank, it, k)
        for gb in rbs:
            gb.all_reduce_average_()
        if clip is not None:
            rscaler.unscale_(topt)
            rp = dict(ref.named_parameters())
            torch.nn.utils.clip_grad_norm_([rp[n] for n in order], clip, foreach=False)
        for g, b in zip(topt.param_groups, base):
            g["lr"] = SCHED.lr_at(b, applied)
        rscaler.step(topt)
        skipped = sum(float(v) for v in rscaler._found_inf_per_device(topt).values()) > 0
        rscaler.update()
        applied += not skipped
        assert skipped == (it in POISON), (it, skipped)
        assert opt.steps == applied, (it, opt.steps, applied)
        assert scaler.get_scale() == rscaler.get_scale() and torch.equal(scaler._growth_tracker, rscaler._growth_tracker)
        if skipped:
            after = _snapshot(kind, opt, net)
            assert all(torch.equal(a, b) for a, b in zip(before[0], after[0])), it
            assert all(torch.equal(x, y) for n in before[1] for x, y in zip(before[1][n], after[1][n])), it
            assert before[2] == after[2]
            assert all(not gb.flat.any() for gb in opt.buckets), "a skipped step leaves the buckets zeroed"
        rp = dict(ref.named_parameters())
        for n, p in net.named_parameters():
            assert torch.equal(p, rp[n]), (kind, hp, it, n)
        want = _ref_state(kind, topt, ref)
        for n, got in _state(kind, opt, net).items():
            for a, b in zip(got, want[n]):
                assert torch.equal(a, b.view_as(a)), (kind, hp, it, n)
    replicas_identical(net, size)
    ddp.remove_hooks()


def w_layerwise(rank, size, kind, hp):
    """FlatLAMB / FlatLARS with the scaler against the same optimizer without one, fed the unscaled gradient (torch's
    ``g * fp32(1 / double(S))``) and skipping where the scaler skips: parameters, state, trust ratios and grad_norm agree
    bit for bit."""
    net, ddp, opt, _, _, _, _, _ = make(kind, hp)
    twin, tddp, topt, _, _, _, _, _ = make(kind, hp)
    scaler = _scaler()
    flat = FlatLAMB if kind == "lamb" else FlatLARS
    assert isinstance(opt, flat) and [len(g["params"]) for g in opt.param_groups] == [len(list(net.parameters()))]
    assert opt.param_groups[0]["lr"] == hp["lr"] and opt.param_groups[0]["weight_decay"] == hp["weight_decay"]
    for it in range(STEPS):
        _scaled_backward(ddp, scaler, rank, it, 1)
        b2.average_gradients(ddp)
        inv = scaler._scale.double().reciprocal().float()
        for gb, tgb in zip(opt.buckets, tddp.buckets):
            tgb.flat.copy_(gb.flat * inv)
        finite = all(torch.isfinite(gb.flat).all() for gb in tddp.buckets)
        scaler.step(opt)
        scaler.update()
        if finite:
            topt.step()
        else:
            tddp.zero_grad()
        tddp._reset()
        assert opt.steps == topt.steps
        for p, q in zip(net.parameters(), twin.parameters()):
            assert torch.equal(p, q), (kind, it)
        assert opt.trust_ratios(net) == topt.trust_ratios(twin)
        assert opt.grad_norm() == topt.grad_norm()
    assert opt.steps == STEPS - len(POISON)
    ddp.remove_hooks()
    tddp.remove_hooks()


def w_sharded_refused(rank, size, kind):
    """sharded=True over several ranks: GradScaler's step raises before anything changes."""
    net, ddp, opt, _, _, _, _, _ = make(kind, dict(lr=0.01, sharded=True))
    scaler = _scaler()
    _scaled_backward(ddp, scaler, rank, 0, 1)
    b2.average_gradients(ddp)
    try:
        scaler.step(opt)
    except RuntimeError as e:
        assert "sharded=False" in str(e) and "scaled gradient" in str(e), e
    else:
        raise AssertionError("sharded=True with GradScaler did not raise")
    assert opt.steps == 0
    ddp.remove_hooks()


# (kind, flat kwargs, explicit unscale_ + clip_grad_norm_, micro-batches per step)
CASES = [("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, groups=True), False, 1),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, nesterov=True, groups=True), False, 1),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.05, groups=True), False, 1),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.05), True, 1),
         ("sgd", dict(lr=0.05, momentum=0.9, weight_decay=0.01), False, 2),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, groups=True), False, 1),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05, groups=True), False, 1),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05), True, 1),
         ("adamw", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1), False, 2)]
LAYERWISE = [("lamb", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1)),
             ("lamb", dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1, max_grad_norm=0.05)),
             ("lars", dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4, nesterov=True)),
             ("lars", dict(lr=0.1, momentum=0.9, weight_decay=1e-2, trust_coefficient=2e-2, eps=1e-4, max_grad_norm=0.05))]


def w_all(rank, size):
    """Every case of CASES and LAYERWISE; sharded=True trains like sharded=False at world size 1 and raises above it."""
    for kind, hp, explicit, k in CASES:
        w_against_torch(rank, size, kind, hp, explicit, k)
    for kind, hp in LAYERWISE:
        w_layerwise(rank, size, kind, hp)
    for kind in ("sgd", "adamw"):
        if size == 1:
            w_against_torch(rank, size, kind, dict(CASES[0 if kind == "sgd" else 5][1], sharded=True), False, 1)
        else:
            w_sharded_refused(rank, size, kind)


def w_gpu_multi(rank, size):
    """Real ranks (backend b200): rank 0's loss overflows at some steps, every rank skips them, and the replicas stay
    bit-identical, with eager steps and with replays of a captured step."""
    import torch.nn.functional as F

    from dist_tuto.pth_b200.models.resnet import ResNet18
    from dist_tuto.pth_b200.ops.optim import FlatAdamW
    from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    for graph in (False, True):
        torch.manual_seed(5)
        m = ResNet18(num_classes=100).to(dev).to(memory_format=torch.channels_last)
        ddp = DistributedDataParallel(m)
        opt = FlatAdamW(ddp, lr=1e-3, max_grad_norm=5.0, capturable=graph)
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
        gen = torch.Generator().manual_seed(100 + rank)
        x = torch.randn(8, 3, 64, 64, generator=gen).to(dev).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 100, (8,), generator=gen).to(dev)
        poison = torch.ones((), device=dev)

        def step():
            with torch.autocast("cuda", dtype=torch.float16):
                loss = F.cross_entropy(ddp(x), y) * poison
            scaler.scale(loss).backward()
            b2.average_gradients(ddp)
            scaler.step(opt)
            scaler.update()

        g = None
        if graph:
            s = torch.cuda.Stream(dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                for _ in range(3):
                    step()
            torch.cuda.current_stream(dev).wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
        base, skips = opt.steps, []
        for it in range(8):
            poison.fill_(float("inf") if rank == 0 and it in (2, 5) else 1.0)
            x.normal_()
            before = float(scaler._scale)
            g.replay() if g is not None else step()
            skips.append(float(scaler._scale) < before)   # GradScaler backs off only after a step it skipped
        torch.cuda.synchronize(dev)
        assert skips[2] and skips[5], skips
        assert opt.steps == base + 8 - sum(skips), (graph, opt.steps, base, skips)
        mine = torch.tensor(skips, dtype=torch.float32, device=dev)
        every = [torch.empty_like(mine) for _ in range(size)]
        b2.all_gather(every, mine)
        assert all(torch.equal(e, mine) for e in every), every
        replicas_identical(m, size)
        ddp.remove_hooks()
