"""capturable=True on one H100: the scalar block against the CPU model, every capturable unsharded instance against its
existing instance fed the same scalars, no host synchronisation in step(), and captured DDP steps against eager ones."""
import pytest
import torch

import capturable_model as CM
import capturable_workers as WK
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops.optim import LRSchedule, schedule_tuple
from emulated_ranks import C, _untouched, _with_sentinel  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

MU, BETAS, EPS = 0.9, (0.9, 0.999), 1e-8
LRS, WDS = [0.1, 3e-3, 1.7e-4], [0.0, 0.01, 0.25]
SCHEDULES = [None, LRSchedule(warmup_steps=7, decay="multistep", milestones=(20, 1000), gamma=0.5),
             LRSchedule(warmup_steps=3, decay="cosine", total_steps=2 ** 41, min_factor=0.1)]


def _state(C):
    lay = C.flat_scalars_layout()
    return (torch.zeros(lay["table_bytes"], dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"),
            torch.zeros(lay["block_bytes"], dtype=torch.uint8, device="cuda"), lay)


def _block_at(C, st, s, lrs=LRS, wds=WDS, sched=None):
    """The block of the update at counter s, reached by a sync to s - 1 and one advance (s = 0: the sync alone)."""
    table, counter, block, _ = st
    C.flat_scalars_sync(table, counter, block, lrs, wds, *BETAS, EPS, schedule_tuple(sched), steps=max(s - 1, 0))
    if s:
        C.flat_scalars_advance(table, counter, block)
    assert int(counter.item()) == s
    return block.view(torch.float32).cpu().tolist()


@pytest.mark.parametrize("sched", SCHEDULES, ids=["none", "warmup multistep", "warmup cosine"])
def test_block_equals_the_model(C, sched):
    st = _state(C)
    lay = st[3]
    for s in [0, 1, 2, 3, 6, 7, 19, 20, 21, 999, 1000, 12345, 2 ** 40 + 3]:
        blk = _block_at(C, st, s, sched=sched)
        for g, (lr, wd) in enumerate(zip(LRS, WDS)):
            lr_t = float(C.lr_schedule_eval(schedule_tuple(sched), lr, torch.tensor([s], device="cuda"))[0])
            host = sched.lr_at(lr, s) if sched is not None else CM.f32(lr)
            assert CM.ulps(lr_t, host) <= (1 if sched is not None and sched.decay == "cosine" else 0), (s, g)
            want = CM.block(lr_t, wd, BETAS, EPS, s)
            got = (blk[lay["sgd_lr"] + g], blk[lay["sgd_wd"] + g], blk[lay["decay"] + g], blk[lay["step_size"] + g])
            assert got == (want["lr"], want["wd"], want["decay"], want["step_size"]), (s, g)
        assert (blk[lay["lr"]], blk[lay["wd"]]) == (want["lr"], want["wd"]) and blk[lay["adamw"]:lay["adamw"] + 7] == want["adamw"], s


def test_block_follows_the_squaring_order(C):
    """beta2 = 1 - 1e-8: at these counters a block computed with pow(beta, t) differs from the squaring order in some fp32
    field; the device equals the squaring order bit for bit at every one of them."""
    betas = (0.9, 0.99999999)
    LR32 = CM.f32(1e-3)                        # the device rounds the base lr to fp32 first
    counters = [s for s in range(2000)
                if CM.block(LR32, 0.0, betas, EPS, s)["adamw"] != CM.block(LR32, 0.0, betas, EPS, s, pow_fn=pow)["adamw"]]
    assert counters
    table, counter, block, lay = _state(C)
    for s in counters:
        C.flat_scalars_sync(table, counter, block, [1e-3], [0.0], *betas, EPS, None, steps=s)
        blk = block.view(torch.float32).cpu().tolist()
        assert blk[lay["adamw"]:lay["adamw"] + 7] == CM.block(LR32, 0.0, betas, EPS, s)["adamw"], s


def test_uploads_are_refused_inside_a_capture():
    m = WK.net().cuda()
    ddp = b2.DistributedDataParallel(m)
    opt = b2.FlatSGD(ddp, capturable=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match="capture"):
            with torch.cuda.graph(g, stream=s):
                opt.sync_hyperparameters()
    torch.cuda.synchronize()
    assert not hasattr(b2.FlatLAMB, "sync_hyperparameters") and not hasattr(b2.FlatLARS, "sync_hyperparameters")
    ddp.remove_hooks()


def test_real_rank_worker_at_world_one():
    """The worker of tests/test_gpu_capturable_multi.py, on backend "b200" at world size 1."""
    b2.launch(WK.w_graph_equals_eager, size=1, backend="b200", join_timeout_s=600)


def _host_scalars(C, st, s):
    blk = _block_at(C, st, s)
    lay = st[3]
    ng = len(LRS)
    return (blk[lay["lr"]], blk[lay["wd"]], blk[lay["adamw"]:lay["adamw"] + 7], blk[lay["sgd_lr"]:lay["sgd_lr"] + ng],
            blk[lay["sgd_wd"]:lay["sgd_wd"] + ng], blk[lay["decay"]:lay["decay"] + ng], blk[lay["step_size"]:lay["step_size"] + ng])


@pytest.mark.parametrize("n", [1, 3, 4, 7, 1024, 1027, 256 * 4 + 5, 200003])
@pytest.mark.parametrize("kind", ["sgd", "sgd_nesterov", "adamw"])
def test_capturable_instances_equal_the_existing_ones(C, n, kind):
    st = _state(C)
    lr, wd, sc, glr, gwd, gdec, gstep = _host_scalars(C, st, 4)
    gen = torch.Generator().manual_seed(n)
    gmap = torch.randint(0, len(LRS), ((n + 3) // 4,), generator=gen, dtype=torch.uint8).cuda()
    p0, g0, m0, v0 = (torch.randn(n, generator=gen) for _ in range(4))
    v0 = v0.abs()
    nesterov = kind == "sgd_nesterov"
    for grouped in (False, True):
        for clip in (None, 0.05):
            a = {k: _with_sentinel(x) for k, x in (("p", p0), ("g", g0), ("m", m0), ("v", v0))}
            b = {k: x.clone() for k, x in a.items()}
            kw, rkw = {}, {}
            if clip is not None:
                sq = torch.zeros(1, dtype=torch.float64, device="cuda")
                C.grad_sqnorm(a["g"][:n], sq, 0, torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda"))
                kw = dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=torch.zeros(1, device="cuda"))
                rkw = dict(max_grad_norm=clip, sqnorms=sq, grad_norm_out=torch.zeros(1, device="cuda"))
            f, r = {k: x[:n] for k, x in a.items()}, {k: x[:n] for k, x in b.items()}
            gm = gmap if grouped else None
            if kind == "adamw":
                C.adamw_flat_cap(f["p"], f["m"], f["v"], f["g"], gm, st[2], True, **kw)
                if grouped:
                    C.adamw_flat_grouped(r["p"], r["m"], r["v"], r["g"], gmap, sc, gdec, gstep, True, **rkw)
                else:
                    C.adamw_flat(r["p"], r["m"], r["v"], r["g"], sc, True, **rkw)
            else:
                C.sgd_flat_cap(f["p"], f["m"], f["g"], gm, st[2], MU, True, nesterov, **kw)
                if grouped:
                    C.sgd_flat_grouped(r["p"], r["m"], r["g"], gmap, glr, gwd, MU, True, nesterov, **rkw)
                else:
                    C.sgd_flat(r["p"], r["m"], r["g"], lr, MU, wd, True, nesterov, **rkw)
            torch.cuda.synchronize()
            for k in ("p", "m", "g", "v"):
                assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), (kind, n, grouped, clip, k)
                assert _untouched(a[k][n:]), (kind, n, grouped, clip, k)
            if clip is not None:
                assert torch.equal(kw["grad_norm_out"], rkw["grad_norm_out"])


def _model():
    return torch.nn.Sequential(torch.nn.Linear(12, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4)).cuda()


def test_refusals_on_cuda():
    net = _model()
    ddp = b2.DistributedDataParallel(net, grad_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="fp32 gradient buckets"):
        b2.FlatAdamW(ddp, capturable=True)
    ddp.remove_hooks()


@pytest.mark.parametrize("name,make", WK.optimizers(), ids=[n for n, _ in WK.optimizers()])
def test_eager_step_does_not_synchronise(name, make):
    m = WK.net().cuda()
    ddp = b2.DistributedDataParallel(m)
    opt = make(ddp, m, capturable=True)
    x, y = torch.randn(4, 3, 8, 8, device="cuda"), torch.randint(0, 10, (4,), device="cuda")
    for it in range(3):
        torch.nn.functional.cross_entropy(ddp(x), y).backward()
        b2.average_gradients(ddp)
        if it == 2:
            # a changed group value is uploaded from pinned memory with non-blocking copies (the debug mode sees torch's
            # own synchronisations only; the upload has no other)
            opt.param_groups[0]["lr"] *= 0.5
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert opt.steps == 3
    ddp.remove_hooks()


@pytest.mark.parametrize("name,make", WK.optimizers(), ids=[n for n, _ in WK.optimizers()])
def test_graph_replays_equal_eager_steps(name, make):
    dev = torch.device("cuda", 0)
    n = 12
    eager = WK.state(*WK.run(make, n, False, dev))
    m, opt = WK.run(make, n, True, dev)
    graph = WK.state(m, opt)
    assert WK.same(eager, graph), name
    assert graph[3] == n and graph[2] is not None
    lrs = [opt.lr_at(s) for s in range(WK.WARMUP, n)]
    assert len(set(lrs)) > 1, "the lr must change across the replays"
    # a checkpoint after the replays loads into a fresh capturable optimizer with the same counter and scalars
    sd = opt.state_dict()
    m2 = WK.net().cuda()
    ddp2 = b2.DistributedDataParallel(m2)
    opt2 = make(ddp2, m2, capturable=True)
    opt2.load_state_dict(sd)
    assert opt2.steps == n and torch.equal(opt2._cap_block, opt._cap_block)
    ddp2.remove_hooks()


def test_capturable_sgd_equals_the_non_capturable_optimizer():
    """With a schedule whose lr the host and the device compute alike (warmup, multistep), capturable FlatSGD is bit for
    bit today's FlatSGD."""
    def make(ddp, m, **kw):
        return b2.FlatSGD(ddp, lr=0.05, momentum=0.9, weight_decay=0.01, max_grad_norm=0.5,
                          lr_schedule=LRSchedule(warmup_steps=3, decay="multistep", milestones=(6,), gamma=0.3), **kw)
    dev = torch.device("cuda", 0)
    a = WK.state(*WK.run(make, 9, False, dev, capturable=False))
    b = WK.state(*WK.run(make, 9, True, dev, capturable=True))
    assert WK.same(a, b)
