"""GPU tier: weight decay and Nesterov momentum in the optimizer kernels (csrc/sgd_device.cuh, csrc/sgd.cu).

* both exchange flavours of ``allreduce_sgd`` at emulated worlds 1-8 (the harness of tests/emulated_ranks.py),
  bit for bit against the model, through the uint32 epoch wrap;
* every engine path -- the one-GPU slot path, the cluster path, ``deterministic=True``, the batched engine and
  ``sgd_flat`` -- bit for bit against an fp32 oracle that applies the update with exact fmaf to the gradient the engine
  itself averaged, and within a stated bound of fp64 ``torch.optim.SGD`` on the same gradients;
* graph replays, ``run_native`` and eager steps agree bit for bit, with and without an lr schedule; explicit defaults
  equal no options; a resumed checkpoint continues bit-equal; two GPUs over the push exchange.
"""
import pytest
import torch

import comm_model as M
import sgd_options_model as SM
import sgd_options_workers as SW
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200 import LRSchedule
from dist_tuto.pth_b200 import data as D
from emulated_ranks import SERIALIZED, C, World, sms  # noqa: F401
from engine_paths import Spy, _batches, _slot_trainer, _state

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900),
              pytest.mark.skipif(SERIALIZED,
                                 reason="serialized launches: every emulated rank's grid would spin alone until it traps")]

OPTIONS = [(1e-2, False), (0.0, True), (1e-2, True)]
OPT_IDS = ["wd", "nesterov", "wd+nesterov"]
SCHED = LRSchedule(warmup_steps=4, decay="multistep", milestones=[7], gamma=0.5)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


# --------------------------------------------------------------------------------------------- emulated ranks
def sgd_model(grads, params, mom, scale, mu, lr, wd, nesterov, bf16_terms):
    """comm_model.sgd_model with weight decay and Nesterov: the exchange of comm_model, then the update of
    sgd_options_model.  With mu, lr and wd powers of two it equals comm_model's fp64 model where that one applies."""
    g = M.reduce_scaled([M.bf16_rn(t) if bf16_terms else t for t in grads], scale)
    return SM.sgd_update(g, params, mom, mu, lr, wd, nesterov)


def options_run(C, sms, world, exchange, zero_grads, wd, nesterov, steps=3, step0=0, seed=0):
    from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC
    n, nv = NPAR_ALLOC, NPAR_ALLOC // 4
    mu, lr, scale = 0.5, 0.125, 1.0 / world
    assert M.is_pow2(mu) and M.is_pow2(lr) and (wd == 0 or M.is_pow2(wd))
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
    gptr = [t.data_ptr() for t in grads]
    iptr = [t.data_ptr() for t in inbox]
    for it in range(steps):
        st = step0 + it
        cur = (st & 1) if two else 0
        gs = [torch.randn(n, generator=g) for _ in range(world)]
        for r in range(world):
            grads[r][cur * n:cur * n + n].copy_(gs[r])
            if two:
                grads[r][(cur ^ 1) * n:(cur ^ 1) * n + n].fill_(7.0)
        before = [t.cpu() for t in grads]
        W.launch(blocks, lambda r: C.allreduce_sgd(gptr, W.sig_ptrs, params[r], mom[r], step[r], lr, mu, scale, r, world,
                                                   zero_grads, n if two else 0, done[r], aux[r], iptr, bf16,
                                                   weight_decay=wd, nesterov=nesterov))
        p, m = sgd_model(gs, p, m, scale, mu, lr, wd, nesterov, bf16_terms=push and bf16 and world > 1)
        what = f"allreduce_sgd {exchange} world {world} wd {wd} nesterov {nesterov} zero_grads {zero_grads} step {st}"
        M.assert_bits_equal(what + ": params", params, [p] * world, 4)
        M.assert_bits_equal(what + ": momentum", mom, [m] * world, 4)
        M.assert_bits_equal(what + ": aux", aux, [M.aux_model(p, aux0)] * world, 4)
        M.assert_bits_equal(what + ": gradient buckets", grads,
                            [M.bucket_model(b, n, cur, zero_grads, two) for b in before], 4)
        for r in range(world):
            assert int(step[r].item()) == st + 1 and int(done[r].item()) == 0, (what, r)


@pytest.mark.parametrize("wd,nesterov", OPTIONS, ids=OPT_IDS)
@pytest.mark.parametrize("zero_grads", [True, False], ids=["zero", "keep"])
@pytest.mark.parametrize("exchange", ["barrier1", "barrier2", "push_fp32", "push_bf16"])
@pytest.mark.parametrize("world", range(1, 9))
def test_allreduce_sgd_options_match_the_model_bit_for_bit(C, sms, world, exchange, zero_grads, wd, nesterov):
    options_run(C, sms, world, exchange, zero_grads, 2.0 ** -6 if wd else 0.0, nesterov, seed=world)


def test_model_equals_comm_model_without_options():
    g = torch.Generator().manual_seed(1)
    gs = [torch.randn(4096, generator=g) for _ in range(3)]
    p, m = torch.randn(4096, generator=g), torch.randn(4096, generator=g)
    a = sgd_model(gs, p, m, 1 / 3, 0.5, 0.125, 0.0, False, True)
    b = M.sgd_model(gs, p, m, 1 / 3, 0.5, 0.125, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("world,exchange", [(2, "push_fp32"), (3, "push_bf16"), (8, "push_fp32"), (4, "barrier2")])
def test_options_across_the_uint32_epoch_wrap(C, sms, world, exchange):
    options_run(C, sms, world, exchange, True, 2.0 ** -5, True, steps=4, step0=2 ** 32 - 2, seed=100 + world)


# --------------------------------------------------------------------------------------------- engine paths
def _check_against_oracles(tr, spy, lr, sched, wd, nesterov):
    """Each logged launch against the exact fp32 update (bit for bit), and the whole run against fp64 torch.optim.SGD on
    the same gradients: |p - p64| <= 2^-16 * (|p64| + 1) after the run's steps (fp32 rounding of every operation, with
    momentum carrying it across steps)."""
    torch.cuda.synchronize()
    for i, (p0, m0, g, st) in enumerate(spy.log):
        p_want, m_want = SM.sgd_update(g, p0, m0, tr.mu, lr if sched is None else sched.lr_at(lr, st), wd, nesterov)
        nxt = spy.log[i + 1] if i + 1 < len(spy.log) else (tr.params, tr.momentum)
        M.assert_bits_equal(f"step {st}: params", [nxt[0]], [p_want.cpu()], 4)
        M.assert_bits_equal(f"step {st}: momentum", [nxt[1]], [m_want.cpu()], 4)
    lrs = [lr if sched is None else sched.lr_at(lr, st) for *_, st in spy.log]
    ref = SM.torch_sgd_fp64(spy.log[0][0], [e[2] for e in spy.log], lrs, tr.mu, wd, nesterov)
    err = (tr.params.double() - ref).abs()
    assert bool((err <= 2.0 ** -16 * (ref.abs() + 1)).all()), float(err.max())
    assert any(not torch.equal(a[2], spy.log[0][2]) for a in spy.log[1:])          # the gradients did change


@pytest.mark.parametrize("wd,nesterov", OPTIONS, ids=OPT_IDS)
@pytest.mark.parametrize("path", ["slot", "cluster", "deterministic"])
def test_fused_engine_paths_match_the_fp32_oracle(dev, path, wd, nesterov):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    if path == "slot":
        tr, raw = FusedTrainer(128, lr=0.05, seed=11, device=dev, raw_uint8=True, weight_decay=wd, nesterov=nesterov,
                               lr_schedule=SCHED), True
    else:
        tr, raw = FusedTrainer(32, lr=0.05, seed=3, device=dev, weight_decay=wd, nesterov=nesterov, lr_schedule=SCHED,
                               deterministic=path == "deterministic"), False
        assert tr.cluster > 1
    spy = Spy(tr)
    for x, y in _batches(10, tr.bsz, 5, raw):
        tr.step(x.to(dev), y.to(dev))                     # device tensors: eager steps
    assert len(spy.log) == 10 and int(tr.step_counter.item()) == 10
    _check_against_oracles(tr, spy, 0.05, SCHED, wd, nesterov)


@pytest.mark.parametrize("wd,nesterov", OPTIONS, ids=OPT_IDS)
def test_batched_engine_matches_the_fp32_oracle(dev, wd, nesterov):
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    tr = BatchedTrainer(2048, lr=0.3, seed=3, device=dev, raw_uint8=True, weight_decay=wd, nesterov=nesterov,
                        lr_schedule=SCHED)
    spy = Spy(tr)
    for x, y in _batches(8, 2048, 7):
        tr.step_device(x.to(dev), y.to(dev))
    assert len(spy.log) == 8
    _check_against_oracles(tr, spy, 0.3, SCHED, wd, nesterov)


@pytest.mark.parametrize("wd,nesterov", [(0.0, False)] + OPTIONS, ids=["plain"] + OPT_IDS)
@pytest.mark.parametrize("n", [4096, 1003])
def test_sgd_flat_matches_the_fp32_oracle(C, n, wd, nesterov):
    g = torch.Generator().manual_seed(n)
    p, m = torch.randn(n, generator=g), torch.zeros(n)
    pd, md = p.cuda(), m.cuda()
    grads = [torch.randn(n, generator=g) for _ in range(5)]
    for k, gr in enumerate(grads):
        gd = gr.cuda()
        C.sgd_flat(pd, md, gd, 0.05, 0.9, wd, True, nesterov)
        torch.cuda.synchronize()
        # sgd_flat_kernel applies fmaf(wd, p, g) whatever wd is (FlatSGD's kernel path, unchanged by this option)
        gg = SM.fma32(wd, p, gr)
        p, m = SM.sgd_update(gg, p, m, 0.9, 0.05, 0.0, nesterov)
        M.assert_bits_equal(f"sgd_flat step {k}: params", [pd], [p], 4)
        M.assert_bits_equal(f"sgd_flat step {k}: momentum", [md], [m], 4)
        assert bool((gd == 0).all())
    with pytest.raises(RuntimeError, match="nesterov"):
        C.sgd_flat(pd, md, gd, 0.05, 0.0, wd, True, True)


# --------------------------------------------------------------------------------------------- launch paths
@pytest.mark.parametrize("sched", [None, SCHED], ids=["const", "schedule"])
def test_graph_native_and_eager_steps_are_bit_equal(dev, sched):
    ds = D.SyntheticMNIST(n=12 * 128, seed=4)
    part = D.Partition(ds, list(range(12 * 128)))
    mk = lambda: D.NativeBatchLoader(part, 128, seed=9, raw_uint8=True, pin_memory=True, num_buffers=6)   # noqa: E731
    kw = dict(weight_decay=1e-2, nesterov=True, lr_schedule=sched)
    graph = _slot_trainer(dev, **kw)
    for x, y in mk():
        graph.step(x, y)
    native = _slot_trainer(dev, **kw)
    done, finished = native.run_native(mk())
    assert done == 12 and finished
    eager = _slot_trainer(dev, **kw)
    for x, y in mk():
        eager.step(x.to(dev), y.to(dev))
    plain = _slot_trainer(dev, lr_schedule=sched)
    for x, y in mk():
        plain.step(x, y)
    a, b, c, d = _state(graph), _state(native), _state(eager), _state(plain)
    assert a[3] == b[3] == c[3] == 12
    for other in (b, c):
        assert torch.equal(a[0], other[0]) and torch.equal(a[1], other[1]) and a[2] == other[2]
    assert not torch.equal(a[0], d[0])                     # the options did change the run


def test_explicit_defaults_are_bit_equal_to_no_options(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    batches = [(x.pin_memory(), y.pin_memory()) for x, y in _batches(6, 128, 8)]
    res = []
    for kw in ({}, dict(weight_decay=0.0, nesterov=False)):
        tr = _slot_trainer(dev, **kw)
        for x, y in batches:
            tr.step(x, y)
        det = FusedTrainer(16, lr=0.05, seed=3, device=dev, deterministic=True, **kw)
        for x, y in batches:
            det.step((x[:16].float() / 255.0).pin_memory(), y[:16].pin_memory())
        res.append((_state(tr), _state(det)))
    for a, b in zip(*res):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


def test_checkpoint_resume_continues_bit_equal(dev):
    batches = [(x.pin_memory(), y.pin_memory()) for x, y in _batches(16, 128, 12)]
    kw = dict(weight_decay=5e-4, nesterov=True, lr_schedule=SCHED)
    straight = _slot_trainer(dev, **kw)
    for x, y in batches:
        straight.step(x, y)
    first = _slot_trainer(dev, **kw)
    for x, y in batches[:7]:
        first.step(x, y)
    sd = first.state_dict()
    assert sd["weight_decay"] == 5e-4 and sd["nesterov"] is True and sd["steps"] == 7
    second = _slot_trainer(dev, **kw)
    second.load_state_dict(sd)
    for x, y in batches[7:]:
        second.step(x, y)
    a, b = _state(straight), _state(second)
    assert a[3] == b[3] == 16 and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # load_state_dict keeps the constructor's options, as it keeps the lr and the schedule
    third = _slot_trainer(dev)
    third.load_state_dict(sd)
    assert (third.weight_decay, third.nesterov) == (0.0, False)


def test_train_fused_engine_takes_the_options(dev):
    out = b2.train(0, 1, b2.TrainConfig(epochs=1, max_steps=4, global_batch=128, engine="fused", device="cuda:0",
                                        weight_decay=5e-4, nesterov=True, dataset=D.SyntheticMNIST(n=1024, seed=2),
                                        log=lambda *a: None))
    assert out["steps"] == 4 and (out["model"].weight_decay, out["model"].nesterov) == (5e-4, True)


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_push_exchange_applies_the_options():
    b2.launch(SW.w_two_gpu_options, size=2, backend="b200", join_timeout_s=600)
