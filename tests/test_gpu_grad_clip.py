"""GPU tier: gradient-norm clipping in the optimizer kernels (the clip instances of csrc/sgd.cu, csrc/sgd_device.cuh).

* ``allreduce_sgd`` in both exchange flavours at emulated worlds 1-8 (the harness of tests/emulated_ranks.py): the
  norm is bit-identical on every rank and within grad_clip_model.NORM_REL_TOL of the fp64 norm of the model's averaged
  gradient, and parameters, momentum, aux and buckets are bit-equal to the model given that norm; a huge max norm equals
  the instance without clipping; the uint32 epoch wrap; sizes where a thread has several vectors; an inf gradient;
* every engine path -- the one-GPU slot path, the cluster path, ``deterministic=True``, the batched engine and
  ``sgd_flat`` + ``grad_sqnorm`` over several buckets -- bit for bit against the fp32 model applied to the gradient the
  engine itself averaged, with the norm checked against fp64;
* graph replays, ``run_native`` and eager steps agree bit for bit; a resumed checkpoint continues bit-equal; two GPUs.
"""
import pytest
import torch

import comm_model as M
import grad_clip_model as GM
import grad_clip_workers as GW
import sgd_options_model as SM
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200 import LRSchedule
from dist_tuto.pth_b200 import data as D
from emulated_ranks import SERIALIZED, C, World, sms  # noqa: F401
from engine_paths import Spy, _batches, _slot_trainer, _state

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900),
              pytest.mark.skipif(SERIALIZED,
                                 reason="serialized launches: every emulated rank's grid would spin alone until it traps")]

SCHED = LRSchedule(warmup_steps=4, decay="multistep", milestones=[7], gamma=0.5)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _same_bits_or_both_nan(what, got, want):
    got, want = got.cpu(), want.cpu()
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), (what, "NaN positions differ")
    assert torch.equal(got[~gn].view(torch.int32), want[~wn].view(torch.int32)), what


# --------------------------------------------------------------------------------------------- emulated ranks
def clip_run(C, sms, world, exchange, zero_grads, wd, nesterov, c, n=None, steps=3, step0=0, seed=0, plant_inf=False,
             against_plain=False):
    from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC
    n = NPAR_ALLOC if n is None else n
    nv = n // 4
    mu, lr, scale = 0.5, 0.125, 1.0 / world
    two = exchange != "barrier1"
    push = exchange.startswith("push")
    bf16 = exchange == "push_bf16"
    blocks = M.sgd_grid_blocks(n)
    W = World(world, sms)
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    m = torch.randn(n, generator=g) * 0.1
    params = [p.cuda() for _ in range(world)]
    mom = [m.cuda() for _ in range(world)]
    grads = [torch.zeros((2 if two else 1) * n, device="cuda") for _ in range(world)]
    step = [torch.full((1,), step0, dtype=torch.int64, device="cuda") for _ in range(world)]
    done = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(world)]
    aux0 = torch.full((M.AUX_N,), -3.0)
    aux = [aux0.cuda() for _ in range(world)]
    inbox = [torch.zeros(2 * world * nv * 8, dtype=torch.int32, device="cuda") for _ in range(world)] if push else []
    ws = [torch.zeros(C.clip_workspace_numel(n), device="cuda") for _ in range(world)]
    norm = [torch.zeros(1, device="cuda") for _ in range(world)]
    gptr = [t.data_ptr() for t in grads]
    iptr = [t.data_ptr() for t in inbox]
    if against_plain:                   # the same steps through the instance without clipping
        pp, mp = [t.clone() for t in params], [t.clone() for t in mom]
        stp = [t.clone() for t in step]
    clipped = 0
    for it in range(steps):
        st = step0 + it
        cur = (st & 1) if two else 0
        gs = [torch.randn(n, generator=g) for _ in range(world)]
        if plant_inf:
            gs[world - 1][7] = float("inf")
        for r in range(world):
            grads[r][cur * n:cur * n + n].copy_(gs[r])
            if two:
                grads[r][(cur ^ 1) * n:(cur ^ 1) * n + n].fill_(7.0)
        before = [t.cpu() for t in grads]
        W.launch(blocks, lambda r: C.allreduce_sgd(gptr, W.sig_ptrs, params[r], mom[r], step[r], lr, mu, scale, r, world,
                                                   zero_grads, n if two else 0, done[r], aux[r], iptr, bf16,
                                                   weight_decay=wd, nesterov=nesterov, max_grad_norm=c,
                                                   clip_workspace=ws[r], grad_norm_out=norm[r]))
        what = f"clip {exchange} world {world} wd {wd} nesterov {nesterov} zero_grads {zero_grads} c {c} step {st}"
        nk = [float(t.item()) for t in norm]
        assert all(x == nk[0] or (x != x and nk[0] != nk[0]) for x in nk), (what, nk)      # the same bits on every rank
        gavg = M.reduce_scaled([M.bf16_rn(t) if push and bf16 and world > 1 else t for t in gs], scale)
        if plant_inf:
            assert nk[0] == float("inf"), (what, nk[0])
        else:
            GM.assert_norm_close(what, nk[0], GM.norm64(gavg))
        clipped += nk[0] > c
        p, m = GM.clip_update(gavg, p, m, mu, lr, wd, nesterov, nk[0], c)
        for r in range(world):
            _same_bits_or_both_nan(what + f": params rank {r}", params[r], p)
            _same_bits_or_both_nan(what + f": momentum rank {r}", mom[r], m)
            _same_bits_or_both_nan(what + f": aux rank {r}", aux[r], M.aux_model(p, aux0))
        M.assert_bits_equal(what + ": gradient buckets", grads, [M.bucket_model(b, n, cur, zero_grads, two) for b in before], 4)
        for r in range(world):
            assert int(step[r].item()) == st + 1 and int(done[r].item()) == 0, (what, r)
        if against_plain:
            for r in range(world):
                grads[r][cur * n:cur * n + n].copy_(gs[r])
            W.launch(blocks, lambda r: C.allreduce_sgd(gptr, W.sig_ptrs, pp[r], mp[r], stp[r], lr, mu, scale, r, world,
                                                       zero_grads, n if two else 0, done[r], None, iptr, bf16,
                                                       weight_decay=wd, nesterov=nesterov))
            for r in range(world):
                assert torch.equal(pp[r], params[r]) and torch.equal(mp[r], mom[r]), (what, "differs from no clipping")
    return clipped


@pytest.mark.parametrize("wd,nesterov", [(0.0, False), (2.0 ** -6, True)], ids=["plain", "wd+nesterov"])
@pytest.mark.parametrize("zero_grads", [True, False], ids=["zero", "keep"])
@pytest.mark.parametrize("exchange", ["barrier1", "barrier2", "push_fp32", "push_bf16"])
@pytest.mark.parametrize("world", range(1, 9))
def test_allreduce_sgd_clip_matches_the_model(C, sms, world, exchange, zero_grads, wd, nesterov):
    # randn gradients of NPAR_ALLOC elements averaged over `world` ranks: norm ~ 148 / sqrt(world) > 10
    assert clip_run(C, sms, world, exchange, zero_grads, wd, nesterov, 10.0, seed=world) == 3


@pytest.mark.parametrize("world,exchange", [(1, "barrier1"), (2, "barrier2"), (2, "push_fp32"), (3, "push_bf16")])
def test_huge_max_norm_equals_no_clipping(C, sms, world, exchange):
    assert clip_run(C, sms, world, exchange, True, 2.0 ** -6, True, 1e30, seed=40 + world, against_plain=True) == 0


@pytest.mark.parametrize("world,exchange", [(2, "push_fp32"), (3, "push_bf16"), (8, "push_fp32"), (4, "barrier2")])
def test_clip_across_the_uint32_epoch_wrap(C, sms, world, exchange):
    clip_run(C, sms, world, exchange, True, 2.0 ** -5, True, 10.0, steps=4, step0=2 ** 32 - 2, seed=100 + world)


@pytest.mark.parametrize("world,exchange", [(1, "barrier1"), (2, "barrier2"), (2, "push_fp32"), (2, "push_bf16")])
def test_clip_with_several_vectors_per_thread(C, sms, world, exchange):
    n = 4 * (64 * 512 * 2 + 100)               # 65636 vectors over 64 CTAs x 512 threads: two or three per thread
    assert M.sgd_grid_blocks(n) == 64
    clip_run(C, sms, world, exchange, False, 2.0 ** -6, False, 50.0, n=n, steps=2, seed=7)


@pytest.mark.parametrize("world,exchange", [(1, "barrier1"), (2, "push_fp32"), (3, "barrier2")])
def test_an_inf_gradient_follows_torch(C, sms, world, exchange):
    """n = inf: coef = c / inf = 0, so every finite gradient becomes 0 and the inf one NaN, as clip_grad_norm_ does."""
    clip_run(C, sms, world, exchange, True, 0.0, False, 1.0, steps=1, seed=3, plant_inf=True)
    g = torch.zeros(8)
    g[1] = float("inf")
    t = torch.nn.Parameter(torch.zeros(8))
    t.grad = g.clone()
    assert float(torch.nn.utils.clip_grad_norm_([t], 1.0, foreach=False)) == float("inf")
    assert torch.isnan(t.grad[1]) and bool((t.grad[[0, 2, 3, 4, 5, 6, 7]] == 0).all())


# --------------------------------------------------------------------------------------------- engine paths
class ClipSpy(Spy):
    """Spy (tests/engine_paths.py) that also reads the norm each optimizer launch reported."""

    def __init__(self, tr):
        super().__init__(tr)
        self.norms = []

    def allreduce_sgd(self, *a, **k):
        super().allreduce_sgd(*a, **k)
        torch.cuda.current_stream().synchronize()
        self.norms.append(float(k["grad_norm_out"].item()))

    def reduce_sgd(self, *a, **k):
        super().reduce_sgd(*a, **k)
        torch.cuda.current_stream().synchronize()
        self.norms.append(float(k["grad_norm_out"].item()))


def _check_clip_oracle(tr, spy, lr, sched, wd, nesterov, c):
    torch.cuda.synchronize()
    clipped = 0
    for i, (p0, m0, g, st) in enumerate(spy.log):
        nk = spy.norms[i]
        GM.assert_norm_close(f"step {st}: norm", nk, GM.norm64(g))
        clipped += nk > c
        p_want, m_want = GM.clip_update(g.cpu(), p0.cpu(), m0.cpu(), tr.mu, lr if sched is None else sched.lr_at(lr, st), wd,
                                        nesterov, nk, c)
        nxt = spy.log[i + 1] if i + 1 < len(spy.log) else (tr.params, tr.momentum)
        M.assert_bits_equal(f"step {st}: params", [nxt[0]], [p_want], 4)
        M.assert_bits_equal(f"step {st}: momentum", [nxt[1]], [m_want], 4)
    assert tr.grad_norm() == spy.norms[-1]
    assert clipped >= len(spy.log) // 2, spy.norms


@pytest.mark.parametrize("path", ["slot", "cluster", "deterministic"])
def test_fused_engine_paths_clip_like_the_model(dev, path):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    kw = dict(weight_decay=1e-2, nesterov=True, lr_schedule=SCHED, max_grad_norm=0.5)
    if path == "slot":
        tr, raw = FusedTrainer(128, lr=0.05, seed=11, device=dev, raw_uint8=True, **kw), True
    else:
        tr, raw = FusedTrainer(32, lr=0.05, seed=3, device=dev, deterministic=path == "deterministic", **kw), False
        assert tr.cluster > 1
    spy = ClipSpy(tr)
    for x, y in _batches(10, tr.bsz, 5, raw):
        tr.step(x.to(dev), y.to(dev))
    assert len(spy.log) == 10
    _check_clip_oracle(tr, spy, 0.05, SCHED, 1e-2, True, 0.5)


def test_batched_engine_clips_like_the_model(dev):
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    tr = BatchedTrainer(2048, lr=0.3, seed=3, device=dev, raw_uint8=True, lr_schedule=SCHED, max_grad_norm=0.05)
    spy = ClipSpy(tr)
    for x, y in _batches(8, 2048, 7):
        tr.step_device(x.to(dev), y.to(dev))
    assert len(spy.log) == 8
    _check_clip_oracle(tr, spy, 0.3, SCHED, 0.0, False, 0.05)


@pytest.mark.parametrize("nesterov", [False, True], ids=["momentum", "nesterov"])
def test_sgd_flat_and_grad_sqnorm_over_several_buckets(C, nesterov):
    sizes = [4096, 1003, 70001]
    g = torch.Generator().manual_seed(5)
    ps = [torch.randn(k, generator=g) for k in sizes]
    ms = [torch.zeros(k) for k in sizes]
    pd, md = [t.cuda() for t in ps], [t.cuda() for t in ms]
    sq = torch.zeros(len(sizes), dtype=torch.float64, device="cuda")
    ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
    out = torch.zeros(1, device="cuda")
    c, wd = 20.0, 1e-2
    for step in range(4):
        grads = [torch.randn(k, generator=g) for k in sizes]
        gd = [t.cuda() for t in grads]
        for k, t in enumerate(gd):
            C.grad_sqnorm(t, sq, k, ws)
        for k in range(len(sizes)):
            C.sgd_flat(pd[k], md[k], gd[k], 0.05, 0.9, wd, True, nesterov, max_grad_norm=c, sqnorms=sq, grad_norm_out=out)
        torch.cuda.synchronize()
        for k, t in enumerate(grads):
            want = float((t.double() ** 2).sum())
            assert abs(float(sq[k]) - want) <= 2 * GM.NORM_REL_TOL * want, (k, float(sq[k]), want)
        nk = float(out.item())
        GM.assert_norm_close(f"sgd_flat step {step}", nk, GM.norm64(grads))
        assert nk > c
        coef = torch.tensor(float(GM.coef32(nk, c)), dtype=torch.float32)
        for k in range(len(sizes)):
            gg = SM.fma32(wd, ps[k], grads[k] * coef)         # sgd_flat_kernel applies fmaf(wd, p, g) whatever wd is
            ps[k], ms[k] = SM.sgd_update(gg, ps[k], ms[k], 0.9, 0.05, 0.0, nesterov)
            M.assert_bits_equal(f"sgd_flat step {step} bucket {k}: params", [pd[k]], [ps[k]], 4)
            M.assert_bits_equal(f"sgd_flat step {step} bucket {k}: momentum", [md[k]], [ms[k]], 4)
            assert bool((gd[k] == 0).all())
    assert int(ws[C.grad_sqnorm_workspace_numel() - 4:].view(torch.int32)[0]) == 0      # the ticket is back at zero


def test_flat_sgd_kernel_path_reports_the_norm(dev):
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(64, 32), torch.nn.ReLU(), torch.nn.Linear(32, 10)).to(dev)
    from dist_tuto.pth_b200.ops.optim import FlatSGD
    opt = FlatSGD(net, lr=0.1, momentum=0.9, max_grad_norm=0.01)
    x = torch.randn(16, 64, device=dev)
    net(x).square().mean().backward()
    want = GM.norm64([p.grad.detach().cpu() for p in net.parameters()])
    opt.step()
    GM.assert_norm_close("FlatSGD", opt.grad_norm(), want)


# --------------------------------------------------------------------------------------------- launch paths
def test_graph_native_and_eager_steps_are_bit_equal_with_clipping(dev):
    ds = D.SyntheticMNIST(n=12 * 128, seed=4)
    part = D.Partition(ds, list(range(12 * 128)))
    mk = lambda: D.NativeBatchLoader(part, 128, seed=9, raw_uint8=True, pin_memory=True, num_buffers=6)   # noqa: E731
    kw = dict(weight_decay=1e-2, nesterov=True, lr_schedule=SCHED, max_grad_norm=0.3)
    graph = _slot_trainer(dev, **kw)
    for x, y in mk():
        graph.step(x, y)
    native = _slot_trainer(dev, **kw)
    done, finished = native.run_native(mk())
    assert done == 12 and finished
    eager = _slot_trainer(dev, **kw)
    for x, y in mk():
        eager.step(x.to(dev), y.to(dev))
    plain = _slot_trainer(dev, weight_decay=1e-2, nesterov=True, lr_schedule=SCHED)
    for x, y in mk():
        plain.step(x, y)
    a, b, c, d = _state(graph), _state(native), _state(eager), _state(plain)
    assert a[3] == b[3] == c[3] == 12
    for other in (b, c):
        assert torch.equal(a[0], other[0]) and torch.equal(a[1], other[1]) and a[2] == other[2]
    assert graph.grad_norm() == native.grad_norm() == eager.grad_norm() > 0.3
    assert not torch.equal(a[0], d[0])                     # the clip did change the run
    assert plain.grad_norm() is None


def test_checkpoint_resume_continues_bit_equal_with_clipping(dev):
    batches = [(x.pin_memory(), y.pin_memory()) for x, y in _batches(16, 128, 12)]
    kw = dict(weight_decay=5e-4, lr_schedule=SCHED, max_grad_norm=0.3)
    straight = _slot_trainer(dev, **kw)
    for x, y in batches:
        straight.step(x, y)
    first = _slot_trainer(dev, **kw)
    for x, y in batches[:7]:
        first.step(x, y)
    sd = first.state_dict()
    assert sd["max_grad_norm"] == 0.3 and sd["steps"] == 7
    second = _slot_trainer(dev, **kw)
    second.load_state_dict(sd)
    for x, y in batches[7:]:
        second.step(x, y)
    a, b = _state(straight), _state(second)
    assert a[3] == b[3] == 16 and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert straight.grad_norm() == second.grad_norm()
    third = _slot_trainer(dev)                             # load_state_dict keeps the constructor's max_grad_norm
    third.load_state_dict(sd)
    assert third.max_grad_norm is None


@pytest.mark.parametrize("engine,batch", [("fused", 128), ("batched", 4096)])
def test_train_takes_max_grad_norm(dev, engine, batch):
    out = b2.train(0, 1, b2.TrainConfig(epochs=2, max_steps=6, global_batch=batch, engine=engine, device="cuda:0",
                                        max_grad_norm=0.25, dataset=D.SyntheticMNIST(n=4 * batch, seed=2),
                                        log=lambda *a: None))
    assert out["steps"] == 6 and out["model"].max_grad_norm == 0.25
    assert len(out["grad_norm"]) == 2 and all(n > 0 for n in out["grad_norm"])


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_push_exchange_clips():
    b2.launch(GW.w_two_gpu_clip, size=2, backend="b200", join_timeout_s=600)
