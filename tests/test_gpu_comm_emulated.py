"""The all-reduce and gradient-exchange kernels (csrc/allreduce.cu, csrc/sgd.cu) on ONE GPU, with W emulated ranks.

The harness is tests/emulated_ranks.py's: each rank gets its own data, signal pad, inbox and stream, and its own launch,
and no case runs more CTAs than the GPU has SMs.  That runs the arithmetic, indexing, padding, parity and epoch protocol of
the one-shot, two-shot and LL all-reduce and of both exchange flavours of ``allreduce_sgd`` at worlds 1-8, and every result
is compared bit for bit with the model of tests/comm_model.py.  What it cannot cover (the memory model across NVLink, NVLS
and the IPC / VMM mappings) stays in tests/test_gpu_multi.py.
"""
import pytest
import torch

import comm_model as M
from emulated_ranks import (C, SENT_VECS, WRAP, World, _typed_sentinel, _untouched, allreduce_cases,  # noqa: F401
                            pytestmark, sms)


# ---------------------------------------------------------------------------------------------------------- all-reduce
def allreduce_call(C, W, variant, n_vec, max_blocks, wire, mode, local, scale, seed):
    """One all-reduce over the emulated world with fresh inputs; checks every rank's output, its symmetric buffer and the
    sentinels behind them against the model."""
    world = W.world
    epv = M.elems_per_vec(wire)
    n = n_vec * epv
    xs = M.make_inputs(world, n, local, seed)
    want = M.allreduce_model(variant, xs, wire, scale, local, staged=mode != "inplace")
    bufs = [_typed_sentinel(n + SENT_VECS * epv, wire) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
    else:
        src = [torch.cat([xs[r], _typed_sentinel(SENT_VECS * epv, local, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [_typed_sentinel(n + SENT_VECS * epv, local) for _ in range(world)]
    buf_ptrs = [b.data_ptr() for b in bufs]
    ll = variant == M.LL
    blocks = M.grid_blocks(variant, n_vec, world, max_blocks)
    W.launch(blocks, lambda r: C.allreduce(variant, wire == torch.bfloat16, buf_ptrs, W.sig_ptrs, 0, src[r], dst[r], n_vec,
                                           scale, r, world, max_blocks, W.inbox_ptrs if ll else [],
                                           M.LL_CAP_VEC if ll else 0))
    what = (f"{M.VARIANT_NAMES[variant]} world {world} n_vec {n_vec} max_blocks {max_blocks} wire {wire} {mode} "
            f"{local} scale {scale}")
    outs = [(bufs[r] if mode == "inplace" else dst[r])[:n] for r in range(world)]
    M.assert_bits_equal(what + ": output", outs, want["out"], epv)
    M.assert_bits_equal(what + ": replicas", outs, [outs[0].cpu()] * world, epv)
    for r in range(world):
        assert _untouched(bufs[r][n:]), f"{what}: rank {r} wrote behind n_vec in its symmetric buffer"
        if mode == "staged":
            assert _untouched(dst[r][n:]), f"{what}: rank {r} wrote behind n_vec in dst"
        elif mode == "alias":
            assert _untouched(dst[r][n:]), f"{what}: rank {r} wrote behind n_vec in src / dst"
        if want["buf"][r] is None:
            assert _untouched(bufs[r]), f"{what}: rank {r}'s symmetric buffer was written"
    M.assert_bits_equal(what + ": symmetric buffers", [b[:n] for b in bufs], want["buf"], epv)


@pytest.mark.parametrize("variant", [M.ONESHOT, M.TWOSHOT, M.LL], ids=["oneshot", "twoshot", "ll"])
@pytest.mark.parametrize("world", range(1, 9))
def test_allreduce_matches_the_model_bit_for_bit(C, sms, world, variant):
    for k, (n_vec, mb, (wire, mode, local), scale) in enumerate(allreduce_cases(variant, world, sms)):
        W = World(world, sms)                     # fresh pads and inboxes: the cap does not change on one buffer here
        allreduce_call(C, W, variant, n_vec, mb, wire, mode, local, scale, seed=1000 * world + 100 * variant + k)


@pytest.mark.parametrize("world", range(1, 9))
def test_epochs_wrap_through_zero_in_every_variant(C, sms, world):
    """Every pad's per-block epoch and flag words start at 2^32 - 5; twelve calls mixing the variants, the barrier kernel and
    block counts carry them through 0 (block 0 reaches epoch 0 in an LL call, whose flag is then 1)."""
    W = World(world, sms, pad_start=WRAP)
    f32, b16 = torch.float32, torch.bfloat16
    calls = [(M.LL, 1000, 3, f32, "inplace", f32), (M.ONESHOT, 3000, 3, f32, "staged", f32), "barrier",
             (M.LL, 4096, 1, b16, "staged", f32), (M.TWOSHOT, world * 700, 2, b16, "inplace", b16),
             (M.ONESHOT, 600, 1, b16, "alias", f32), (M.LL, 513, 3, f32, "alias", f32), "barrier",
             (M.TWOSHOT, world * 1500, 3, f32, "staged", f32), (M.LL, 2000, 3, b16, "inplace", b16),
             (M.ONESHOT, 5000, 2, f32, "inplace", f32), (M.LL, 4096, 3, b16, "alias", b16)]
    for k, c in enumerate(calls):
        if c == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
            continue
        variant, n_vec, mb, wire, mode, local = c
        allreduce_call(C, W, variant, n_vec, mb, wire, mode, local, 1.0 / world, seed=77 * world + k)
    # block 0 went through 0 and, like every other block, agrees on its epoch across ranks
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 100


@pytest.mark.parametrize("world", [2, 5, 8])
def test_ll_allreduce_with_a_cap_that_changes_between_calls(C, sms, world):
    """LL calls on one set of pads and inboxes with max_blocks 2, 1, 2 (n_vec 1024, 700, 700) and different data each time.
    If the cap decided the grid, vector 600 would be handled by block 0 in the second call and by block 1 in the third, both
    at epoch 2 and parity 0, and the third call could accept the second call's line."""
    W = World(world, sms)
    for k, (n_vec, mb) in enumerate([(1024, 2), (700, 1), (700, 2)]):
        allreduce_call(C, W, M.LL, n_vec, mb, torch.float32, "inplace", torch.float32, 1.0, seed=5 * world + k)


# ------------------------------------------------------------------------------------------------------------ SGD
def sgd_run(C, sms, world, exchange, zero_grads, steps=4, step0=0, seed=0):
    """``steps`` calls of allreduce_sgd over the emulated world.  exchange: "barrier1" (one bucket, grad_stride 0),
    "barrier2" (two buckets), "push_fp32" / "push_bf16" (push exchange, two buckets)."""
    from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC
    n, nv = NPAR_ALLOC, NPAR_ALLOC // 4
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
                                                   zero_grads, n if two else 0, done[r], aux[r], iptr, bf16))
        p, m = M.sgd_model(gs, p, m, scale, mu, lr, bf16_terms=push and bf16 and world > 1)
        what = f"allreduce_sgd {exchange} world {world} zero_grads {zero_grads} step {st}"
        M.assert_bits_equal(what + ": params", params, [p] * world, 4)
        M.assert_bits_equal(what + ": momentum", mom, [m] * world, 4)
        M.assert_bits_equal(what + ": aux", aux, [M.aux_model(p, aux0)] * world, 4)
        M.assert_bits_equal(what + ": gradient buckets", grads,
                            [M.bucket_model(b, n, cur, zero_grads, two) for b in before], 4)
        for r in range(world):
            assert int(step[r].item()) == st + 1 and int(done[r].item()) == 0, (what, r)


@pytest.mark.parametrize("zero_grads", [True, False], ids=["zero", "keep"])
@pytest.mark.parametrize("exchange", ["barrier1", "barrier2", "push_fp32", "push_bf16"])
@pytest.mark.parametrize("world", range(1, 9))
def test_allreduce_sgd_matches_the_model_bit_for_bit(C, sms, world, exchange, zero_grads):
    sgd_run(C, sms, world, exchange, zero_grads, seed=world)


@pytest.mark.parametrize("world,exchange", [(2, "push_fp32"), (2, "push_bf16"), (5, "push_bf16"), (8, "push_fp32")])
def test_push_exchange_across_the_uint32_epoch_wrap(C, sms, world, exchange):
    """Step counter 2^32 - 2 .. 2^32 + 1 on a zeroed inbox: at step 2^32 - 1 the push epoch (uint32)(step + 1) is 0, the
    value of a line nobody wrote; the kernel must use another flag there."""
    sgd_run(C, sms, world, exchange, True, step0=2 ** 32 - 2, seed=100 + world)
