"""The sharded optimizer kernel (csrc/sharded_sgd.cu) on ONE GPU, with W emulated ranks.

``C.sharded_sgd`` takes raw per-rank pointers, so W "ranks" are W sets of buffers on one device, each with its own gradient
bucket, parameter flat, momentum shard, signal pad and stream, and its own launch.  That runs the slice mapping, the rank-order
reduction, the update, the peer stores, the zeroing and the epoch protocol at worlds 1-8, and every buffer is compared bit for
bit with the model of tests/sharded_sgd_model.py and, for fp32 buckets, with the existing kernels (``C.allreduce`` then
``C.sgd_flat``) run on the same inputs.  What it cannot cover (the memory model across NVLink and the symmetric mappings) is
in tests/test_gpu_sharded_sgd_multi.py.

The W grids of one call must be co-resident; tests/emulated_ranks.py's ``World`` issues them back to back on W streams and
asserts ``world x blocks <= SM count`` before any launch.
"""
import pytest
import torch

import comm_model as M
import sharded_sgd_model as S
from emulated_ranks import C, WRAP, World, _untouched, _with_sentinel, pytestmark, sms  # noqa: F401

OPTIONS = [(0.0, False), (0.01, False), (0.0, True), (0.01, True)]  # (weight decay, nesterov)
LR, MU = 0.07, 0.9


def run_steps(C, W, n_vec, max_blocks, wire, wd, nesterov, zero_grad, seed, steps=3, against_kernels=False):
    """``steps`` sharded steps over the emulated world with fresh gradients each; after each, every rank's parameter flat,
    momentum shard and gradient bucket and the sentinels behind them are checked against the model.  ``against_kernels``
    (fp32): the parameters and momentum also equal, bit for bit, the two-shot and the one-shot all-reduce of the same
    gradients followed by sgd_flat."""
    world = W.world
    epv = M.elems_per_vec(wire)
    n, per = n_vec * epv, n_vec * epv // world
    scale = 1.0 / world
    blocks = S.grid_blocks(n_vec, world, max_blocks)
    p0, m0, m_full = S.make_state(world, n, seed)
    params = [_with_sentinel(p) for p in p0]
    mom = [_with_sentinel(m) for m in m0]
    grads = [_with_sentinel(torch.zeros(n), wire) for _ in range(world)]
    gp, pp = [g.data_ptr() for g in grads], [p.data_ptr() for p in params]
    what = (f"sharded_sgd world {world} n_vec {n_vec} max_blocks {max_blocks} {wire} wd {wd} nesterov {nesterov} "
            f"zero_grad {zero_grad}")
    if against_kernels:
        assert wire == torch.float32
        ref_p = {v: p0[0].cuda() for v in (M.TWOSHOT, M.ONESHOT)}
        ref_m = {v: m_full.cuda() for v in (M.TWOSHOT, M.ONESHOT)}
    for it in range(steps):
        gs = M.make_inputs(world, n, wire, 7919 * seed + it, specials=False)
        for r in range(world):
            if zero_grad and it > 0:
                assert not bool(grads[r][:n].any()), f"{what} step {it}: rank {r}'s bucket was not left zeroed"
            grads[r][:n].copy_(gs[r])
        if against_kernels:
            for v in (M.TWOSHOT, M.ONESHOT):
                bufs = [g[:n].clone() for g in grads]
                bptr = [b.data_ptr() for b in bufs]
                W.launch(M.grid_blocks(v, n_vec, world, max_blocks),
                         lambda r: C.allreduce(v, False, bptr, W.sig_ptrs, 0, None, None, n_vec, scale, r, world, max_blocks))
                C.sgd_flat(ref_p[v], ref_m[v], bufs[0], LR, MU, wd, False, nesterov)
        W.launch(blocks, lambda r: C.sharded_sgd(wire == torch.bfloat16, gp, pp, W.sig_ptrs, mom[r][:per], n_vec, LR, MU, wd,
                                                 nesterov, scale, zero_grad, r, world, max_blocks))
        want = S.sharded_sgd_model(gs, p0, m0, scale, LR, MU, wd, nesterov, zero_grad)
        M.assert_bits_equal(f"{what} step {it}: params", [p[:n] for p in params], want["params"], 4)
        M.assert_bits_equal(f"{what} step {it}: momentum", [m[:per] for m in mom], want["momentum"], 4)
        M.assert_bits_equal(f"{what} step {it}: gradient buckets", [g[:n] for g in grads], want["grads"], epv)
        for r in range(world):
            assert _untouched(params[r][n:]) and _untouched(mom[r][per:]) and _untouched(grads[r][n:]), (
                f"{what} step {it}: rank {r} wrote behind one of its buffers")
        if against_kernels:
            for v in (M.TWOSHOT, M.ONESHOT):
                name = f"{what} step {it}: {M.VARIANT_NAMES[v]} all-reduce + sgd_flat"
                M.assert_bits_equal(name + ": params", [p[:n] for p in params], [ref_p[v].cpu()] * world, 4)
                M.assert_bits_equal(name + ": momentum", [torch.cat([m[:per] for m in mom])], [ref_m[v].cpu()], 4)
        p0, m0 = want["params"], want["momentum"]


def cases(world, sms):
    """(n_vec, max_blocks, wire, wd, nesterov, zero_grad): per max_blocks (1, 3, SMs // world) slices of 1, 511, 512, 513
    vectors and one and three full passes of the unrolled loop +- 1; the options, zero_grad and the wire dtype rotate so that
    every combination occurs in every world."""
    out = []
    for m, mb in enumerate([1, 3, sms // world]):
        tail = M.UNROLL * M.THREADS * mb              # one full pass of the unrolled loop at mb CTAs
        for i, sl in enumerate([1, 511, 512, 513, tail - 1, tail + 1, 3 * tail - 1, 3 * tail + 1]):
            k = 8 * m + i
            wd, nesterov = OPTIONS[k % 4]
            out.append((world * sl, mb, torch.bfloat16 if (k // 4) % 2 else torch.float32, wd, nesterov, (k // 8 + i) % 2 == 0))
    return out


@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_sgd_matches_the_model_bit_for_bit(C, sms, world):
    for k, (n_vec, mb, wire, wd, nesterov, zero_grad) in enumerate(cases(world, sms)):
        run_steps(C, World(world, sms), n_vec, mb, wire, wd, nesterov, zero_grad, seed=100 * world + k)


@pytest.mark.parametrize("world", range(1, 9))
def test_fp32_equals_the_allreduce_kernels_followed_by_sgd_flat(C, sms, world):
    """Also the 8 MB bucket of a ResNet-18 step (524288 vectors, rounded up to the world), at SMs // world CTAs."""
    big = (524288 + world - 1) // world * world
    for k, (n_vec, mb) in enumerate([(world * 513, 1), (world * 3073, 3), (big, sms // world)]):
        wd, nesterov = OPTIONS[(world + k) % 4]
        run_steps(C, World(world, sms), n_vec, mb, torch.float32, wd, nesterov, k % 2 == 0, seed=50 * world + k,
                  against_kernels=True)


@pytest.mark.parametrize("world", [2, 8])
def test_bf16_8mb_bucket(C, sms, world):
    run_steps(C, World(world, sms), 524288, sms // world, torch.bfloat16, 0.01, True, True, seed=world, steps=2)


@pytest.mark.parametrize("world", range(1, 9))
def test_epochs_wrap_through_zero(C, sms, world):
    """Every pad's per-block epoch and flag words start at 2^32 - 5; six steps (two barriers each) carry them through 0."""
    W = World(world, sms, pad_start=WRAP)
    run_steps(C, W, world * 1500, 3, torch.float32, 0.01, True, True, seed=9 * world, steps=6)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all()) and int(ep[0, 0]) == 7


def test_refusals(C):
    pad = torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda")
    g, p, m = (torch.zeros(64, device="cuda") for _ in range(3))
    one = lambda t, k: [t.data_ptr()] * k          # noqa: E731
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.sharded_sgd(False, one(g, 3), one(p, 3), one(pad, 3), m, 16, 0.1, 0.5, 0.0, False, 1.0, True, 0, 3)
    with pytest.raises(RuntimeError, match="world"):
        C.sharded_sgd(False, one(g, 9), one(p, 9), one(pad, 9), m, 18, 0.1, 0.5, 0.0, False, 1.0, True, 0, 9)
    with pytest.raises(RuntimeError, match="one gradient bucket"):
        C.sharded_sgd(False, one(g, 2), one(p, 1), one(pad, 2), m, 16, 0.1, 0.5, 0.0, False, 1.0, True, 0, 2)
    with pytest.raises(RuntimeError, match="momentum"):
        C.sharded_sgd(False, one(g, 2), one(p, 2), one(pad, 2), m[:8], 16, 0.1, 0.5, 0.0, False, 1.0, True, 0, 2)
    with pytest.raises(RuntimeError, match="nesterov"):
        C.sharded_sgd(False, one(g, 2), one(p, 2), one(pad, 2), m, 16, 0.1, 0.0, 0.0, True, 1.0, True, 0, 2)
