"""FlatAdamW's kernels on one GPU: ``adamw_flat`` (csrc/adamw.cu) and the AdamW instance of the sharded kernel
(csrc/sharded_sgd.cu) bit for bit against tests/adamw_model.py, the kernel against ``torch.optim.AdamW`` on CUDA and fp64,
the sharded kernel at emulated worlds 1-8 (the harness of tests/emulated_ranks.py), and a ResNet-18 trained
through ``DistributedDataParallel`` + ``FlatAdamW`` under bf16 autocast."""
import math

import pytest
import torch
import torch.nn.functional as F

import adamw_model as A
import comm_model as M
import sharded_sgd_model as S
from emulated_ranks import CO_RESIDENT, C, World, _bits, _untouched, _with_sentinel, sms  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HP = dict(lr=0.01, betas=(0.8, 0.95), eps=1e-6, wd=0.1)
SIZES = [1, 2, 3, 4, 5, 6, 7, 1023, 1024, 1025, 1026, 1027, 256 * 4 * 7 + 3, 1 << 20, (1 << 20) + 1, 3 * 1000003]


def _sc(t, hp=HP):
    return A.scalars64(hp["lr"], hp["betas"], hp["eps"], hp["wd"], t)


def _state(n, seed):
    g = torch.Generator().manual_seed(seed)
    p, grad = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1
    m, v = torch.randn(n, generator=g) * 0.01, torch.rand(n, generator=g) * 1e-3
    z = torch.rand(n, generator=g) < 0.1                  # zero-gradient elements with empty moments: den == eps
    grad[z], m[z], v[z] = 0, 0, 0
    return p, grad, m, v


@pytest.mark.parametrize("n", SIZES)
def test_adamw_flat_matches_the_model_bit_for_bit(C, n):
    p, g, m, v = _state(n, n)
    for zero_grad in (True, False):
        bufs = [_with_sentinel(x) for x in (p, m, v, g)]
        dp, dm, dv, dg = bufs
        for t in (1, 2):
            C.adamw_flat(dp[:n], dm[:n], dv[:n], dg[:n], _sc(t), zero_grad)
            want = A.adamw_update(g, p if t == 1 else want[0], m if t == 1 else want[1], v if t == 1 else want[2],
                                  HP["lr"], HP["betas"], HP["eps"], HP["wd"], t)
            for name, got, w in zip("pmv", (dp, dm, dv), want):
                assert _bits(got[:n], w), f"n {n} t {t} zero_grad {zero_grad}: {name}"
            assert all(_untouched(b[n:]) for b in bufs), f"n {n}: a sentinel behind a buffer changed"
            if zero_grad:
                assert not dg[:n].any()
                dg[:n].copy_(g)
            else:
                assert _bits(dg[:n], g)


@pytest.mark.parametrize("n", [5, 1027, (1 << 20) + 3])
def test_clip_instance_with_a_coefficient_below_one(C, n):
    p, g, m, v = _state(n, 3 * n)
    dp, dm, dv, dg = (x.cuda() for x in (p, m, v, g))
    sq = torch.zeros(2, dtype=torch.float64, device="cuda")
    ws = torch.zeros(C.grad_sqnorm_workspace_numel(), device="cuda")
    other = torch.randn(4096, device="cuda")                # a second bucket's squares count towards the norm
    C.grad_sqnorm(dg, sq, 0, ws)
    C.grad_sqnorm(other, sq, 1, ws)
    norm = torch.zeros(1, device="cuda")
    c = 0.5
    C.adamw_flat(dp, dm, dv, dg, _sc(3), True, max_grad_norm=c, sqnorms=sq, grad_norm_out=norm)
    coef = A.clip_coef(sq.cpu().tolist(), c)
    assert coef < 1.0
    want = A.adamw_update(g * torch.tensor(coef, dtype=torch.float32), p, m, v, HP["lr"], HP["betas"], HP["eps"], HP["wd"], 3)
    for name, got, w in zip("pmv", (dp, dm, dv), want):
        assert _bits(got, w), name
    assert not dg.any()
    assert float(norm) == A.f32(math.sqrt(sum(sq.cpu().tolist())))


def test_kernel_error_against_fp64_is_within_4x_torch_fp32():
    """50 updates with fresh gradients; the kernel (through FlatAdamW) and torch.optim.AdamW on CUDA from the same inputs."""
    from dist_tuto.pth_b200 import FlatAdamW
    n, steps = 50001, 50
    gen = torch.Generator().manual_seed(5)
    p0 = torch.randn(n, generator=gen)
    grads = [torch.randn(n, generator=gen) * 0.1 for _ in range(steps)]
    lin = torch.nn.Linear(n, 1, bias=False).cuda()
    with torch.no_grad():
        lin.weight.copy_(p0.view(1, n))
    opt = FlatAdamW(lin, lr=HP["lr"], betas=HP["betas"], eps=HP["eps"], weight_decay=HP["wd"])
    w = torch.nn.Parameter(p0.clone().cuda())
    topt = torch.optim.AdamW([w], lr=HP["lr"], betas=HP["betas"], eps=HP["eps"], weight_decay=HP["wd"])
    for g in grads:
        lin._grad_bucket.flat[:n].copy_(g)
        opt.step()
        w.grad = g.cuda()
        topt.step()
    ref = A.adamw_fp64(p0, grads, [HP["lr"]] * steps, HP["betas"], HP["eps"], HP["wd"])
    e_k = float((lin.weight.detach().view(-1).double().cpu() - ref).abs().max())
    e_t = float((w.detach().double().cpu() - ref).abs().max())
    big = ref.abs().max().float()
    ulp = float(torch.nextafter(big, torch.tensor(float("inf"))) - big)
    assert e_k <= 4 * e_t + ulp, (e_k, e_t, ulp)


# ----------------------------------------------------------------------------------------------- emulated ranks
def _sharded_model(gs, params, ms, vs, scale, t):
    """Every rank's parameter flat, moment shards and bucket after one sharded AdamW step (as sharded_sgd_model)."""
    world, n = len(gs), gs[0].numel()
    new_p, new_m, new_v = [p.clone() for p in params], [m.clone() for m in ms], [v.clone() for v in vs]
    for r in range(world):
        lo, hi = S.slice_of(r, world, n)
        g = M.reduce_scaled([x[lo:hi].float() for x in gs], scale)
        p, new_m[r], new_v[r] = A.adamw_update(g, params[r][lo:hi], ms[r], vs[r], HP["lr"], HP["betas"], HP["eps"], HP["wd"], t)
        for q in range(world):
            new_p[q][lo:hi] = p
    return new_p, new_m, new_v


def run_sharded(C, W, n_vec, max_blocks, wire, zero_grad, seed, steps=3, against_kernels=False, t0=1):
    world = W.world
    epv = M.elems_per_vec(wire)
    n, per = n_vec * epv, n_vec * epv // world
    scale = 1.0 / world
    blocks = S.grid_blocks(n_vec, world, max_blocks)
    p0, m0, m_full = S.make_state(world, n, seed)
    v_full = m_full.abs() * 0.01
    v0 = [v_full[r * per:(r + 1) * per].clone() for r in range(world)]
    params = [_with_sentinel(p) for p in p0]
    ms, vs = [_with_sentinel(m) for m in m0], [_with_sentinel(v) for v in v0]
    grads = [_with_sentinel(torch.zeros(n), wire) for _ in range(world)]
    gp, pp = [g.data_ptr() for g in grads], [p.data_ptr() for p in params]
    what = f"sharded_adamw world {world} n_vec {n_vec} max_blocks {max_blocks} {wire} zero_grad {zero_grad}"
    if against_kernels:
        ref = [p0[0].cuda(), m_full.cuda(), v_full.cuda()]
    for it in range(steps):
        t = t0 + it
        gs = M.make_inputs(world, n, wire, 7919 * seed + it, specials=False)
        for r in range(world):
            if zero_grad and it > 0:
                assert not bool(grads[r][:n].any()), f"{what} step {it}: rank {r}'s bucket was not left zeroed"
            grads[r][:n].copy_(gs[r])
        if against_kernels:
            bufs = [g[:n].clone() for g in grads]
            bptr = [b.data_ptr() for b in bufs]
            W.launch(M.grid_blocks(M.TWOSHOT, n_vec, world, max_blocks),
                     lambda r: C.allreduce(M.TWOSHOT, False, bptr, W.sig_ptrs, 0, None, None, n_vec, scale, r, world, max_blocks))
            C.adamw_flat(ref[0], ref[1], ref[2], bufs[0], _sc(t), False)
        W.launch(blocks, lambda r: C.sharded_adamw(wire == torch.bfloat16, gp, pp, W.sig_ptrs, ms[r][:per], vs[r][:per], n_vec,
                                                   _sc(t), scale, zero_grad, r, world, max_blocks))
        wp, wm, wv = _sharded_model(gs, p0, m0, v0, scale, t)
        M.assert_bits_equal(f"{what} step {it}: params", [p[:n] for p in params], wp, 4)
        M.assert_bits_equal(f"{what} step {it}: exp_avg", [m[:per] for m in ms], wm, 4)
        M.assert_bits_equal(f"{what} step {it}: exp_avg_sq", [v[:per] for v in vs], wv, 4)
        M.assert_bits_equal(f"{what} step {it}: gradient buckets", [g[:n] for g in grads],
                            [torch.zeros_like(g) if zero_grad else g.clone() for g in gs], epv)
        for r in range(world):
            assert _untouched(params[r][n:]) and _untouched(ms[r][per:]) and _untouched(vs[r][per:]) and \
                _untouched(grads[r][n:]), f"{what} step {it}: rank {r} wrote behind one of its buffers"
        if against_kernels:
            name = f"{what} step {it}: two-shot all-reduce + adamw_flat"
            M.assert_bits_equal(name + ": params", [p[:n] for p in params], [ref[0].cpu()] * world, 4)
            M.assert_bits_equal(name + ": exp_avg", [torch.cat([m[:per] for m in ms])], [ref[1].cpu()], 4)
            M.assert_bits_equal(name + ": exp_avg_sq", [torch.cat([v[:per] for v in vs])], [ref[2].cpu()], 4)
        p0, m0, v0 = wp, wm, wv


def _cases(world, sms):
    out = []
    for m, mb in enumerate([1, 3, sms // world]):
        tail = M.THREADS * mb                 # one pass of the AdamW instance's loop (unroll 1) at mb CTAs
        for i, sl in enumerate([1, 511, 513, tail - 1, tail + 1, 3 * tail + 1]):
            k = 6 * m + i
            out.append((world * sl, mb, torch.bfloat16 if k % 2 else torch.float32, (k // 2) % 2 == 0))
    return out


@CO_RESIDENT
@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_adamw_matches_the_model_bit_for_bit(C, sms, world):
    for k, (n_vec, mb, wire, zero_grad) in enumerate(_cases(world, sms)):
        run_sharded(C, World(world, sms), n_vec, mb, wire, zero_grad, seed=100 * world + k)


@CO_RESIDENT
@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_adamw_fp32_equals_allreduce_then_adamw_flat(C, sms, world):
    big = (524288 + world - 1) // world * world
    for k, (n_vec, mb) in enumerate([(world * 513, 1), (world * 3073, 3), (big, sms // world)]):
        run_sharded(C, World(world, sms), n_vec, mb, torch.float32, k % 2 == 0, seed=50 * world + k, against_kernels=True)


@CO_RESIDENT
@pytest.mark.parametrize("world", [1, 3, 8])
def test_sharded_adamw_epochs_wrap_through_zero(C, sms, world):
    W = World(world, sms, pad_start=2 ** 32 - 5)
    run_sharded(C, W, world * 1500, 3, torch.bfloat16, True, seed=9 * world, steps=6)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all()) and int(ep[0, 0]) == 7


def test_refusals(C):
    pad = torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda")
    g, p, m, v = (torch.zeros(64, device="cuda") for _ in range(4))
    one = lambda t, k: [t.data_ptr()] * k          # noqa: E731
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.sharded_adamw(False, one(g, 3), one(p, 3), one(pad, 3), m, v, 16, _sc(1), 1.0, True, 0, 3)
    with pytest.raises(RuntimeError, match="world"):
        C.sharded_adamw(False, one(g, 9), one(p, 9), one(pad, 9), m, v, 18, _sc(1), 1.0, True, 0, 9)
    with pytest.raises(RuntimeError, match="exp_avg"):
        C.sharded_adamw(False, one(g, 2), one(p, 2), one(pad, 2), m[:8], v, 16, _sc(1), 1.0, True, 0, 2)
    with pytest.raises(RuntimeError, match="scalars"):
        C.sharded_adamw(False, one(g, 2), one(p, 2), one(pad, 2), m, v, 16, _sc(1)[:6], 1.0, True, 0, 2)
    with pytest.raises(RuntimeError, match="one size"):
        C.adamw_flat(p, m, v[:60], g, _sc(1), True)


# ----------------------------------------------------------------------------------------------- module level
def test_ddp_resnet18_trains_like_torch_adamw_under_bf16_autocast():
    import dist_tuto.pth_b200 as b2
    import adamw_gpu_workers as WK
    b2.launch(WK.w_resnet, size=1, backend="b200", join_timeout_s=600)


def test_world_one_sharded_is_the_unsharded_path():
    import dist_tuto.pth_b200 as b2
    import adamw_gpu_workers as WK
    b2.launch(WK.w_world1, size=1, backend="b200", join_timeout_s=600)
