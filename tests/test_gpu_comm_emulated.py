"""The all-reduce and gradient-exchange kernels (csrc/allreduce.cu, csrc/sgd.cu) on ONE GPU, with W emulated ranks.

The kernels take raw per-rank pointers, so W "ranks" can be W sets of buffers on one device: each rank gets its own data,
signal pad, inbox and stream, and its own launch.  That runs the arithmetic, indexing, padding, parity and epoch protocol of
the one-shot, two-shot and LL all-reduce and of both exchange flavours of ``allreduce_sgd`` at worlds 1-8, and every result
is compared bit for bit with the model of tests/comm_model.py.  What it cannot cover (the memory model across NVLink, NVLS
and the IPC / VMM mappings) stays in tests/test_gpu_multi.py.

Every CTA of these kernels spins on its peers, so the W grids of one call must all be resident at once:

* the W launches are issued back to back on W streams between two device synchronisations, never one after another with a
  wait in between.  With serialized launches (CUDA_LAUNCH_BLOCKING=1, or a tool that serializes kernels) the first rank's
  grid spins alone until B2_SPIN_LIMIT and traps, so this file is skipped under CUDA_LAUNCH_BLOCKING=1 and is not part of
  tools/sanitize.sh;
* the budget is one CTA per SM for all ranks together (``allreduce_oneshot_kernel<false>`` uses 128 registers x 512
  threads, the whole register file of an SM): the harness computes each launch's grid as the launcher does and refuses
  any case with ``world x blocks > SM count``.
"""
import os

import pytest
import torch

import comm_model as M

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900),
              pytest.mark.skipif(os.environ.get("CUDA_LAUNCH_BLOCKING") == "1",
                                 reason="serialized launches: every rank's grid would spin alone until it traps")]

SENT_VECS = 3                                   # sentinel vectors behind every buffer
SENTINEL = {torch.float32: 0x5EADBEEF, torch.bfloat16: 0x5EAD}     # finite bit patterns no kernel result can produce here
WRAP = 2 ** 32 - 5                              # epoch-wrap test: every pad's epoch and flag words start here


@pytest.fixture(scope="module")
def C():
    from dist_tuto.pth_b200.ops import _ext
    return _ext.C()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sentinel(n, dtype, dev="cuda"):
    bits = torch.full((n,), SENTINEL[dtype], dtype=torch.int32 if dtype == torch.float32 else torch.int16, device=dev)
    return bits.view(dtype)


def _untouched(t):
    ib = torch.int32 if t.dtype == torch.float32 else torch.int16
    return bool((t.view(ib) == SENTINEL[t.dtype]).all())


class World:
    """W emulated ranks on cuda:0: a zeroed signal pad (uint32 [B2_SIGNAL_WORDS]), an LL inbox
    ([2 parities][W sources][LL_CAP_VEC][2 lines of 16 B]) and a stream per rank."""

    def __init__(self, world, sms, pad_start=0):
        self.world, self.sms = world, sms
        self.pads = [torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda") for _ in range(world)]
        if pad_start:
            for p in self.pads:                   # per-block epoch words and every flag word
                p[:M.EPOCH_WORD0 + M.MAX_BLOCKS] = pad_start - 2 ** 32 if pad_start >= 2 ** 31 else pad_start
        self.inbox = [torch.zeros(2 * world * M.LL_CAP_VEC * 8, dtype=torch.int32, device="cuda") for _ in range(world)]
        self.streams = [torch.cuda.Stream() for _ in range(world)]
        self.sig_ptrs = [p.data_ptr() for p in self.pads]
        self.inbox_ptrs = [b.data_ptr() for b in self.inbox]

    def launch(self, blocks, fn):
        """fn(r) issues rank r's kernel.  All W launches go out back to back, each on its own stream."""
        assert self.world * blocks <= self.sms, (
            f"{self.world} ranks x {blocks} CTAs would not be co-resident on {self.sms} SMs; not launched")
        torch.cuda.synchronize()
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                fn(r)
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- all-reduce
# (wire dtype, mode, local dtype): in place on the symmetric buffers; src / dst; src aliasing dst (parallel/symm.py's
# staged path)
COMBOS = [(torch.float32, "inplace", torch.float32), (torch.float32, "staged", torch.float32),
          (torch.float32, "alias", torch.float32), (torch.bfloat16, "inplace", torch.bfloat16),
          (torch.bfloat16, "staged", torch.bfloat16), (torch.bfloat16, "staged", torch.float32),
          (torch.bfloat16, "alias", torch.float32), (torch.bfloat16, "alias", torch.bfloat16)]


def allreduce_call(C, W, variant, n_vec, max_blocks, wire, mode, local, scale, seed):
    """One all-reduce over the emulated world with fresh inputs; checks every rank's output, its symmetric buffer and the
    sentinels behind them against the model."""
    world = W.world
    epv = M.elems_per_vec(wire)
    n = n_vec * epv
    xs = M.make_inputs(world, n, local, seed)
    want = M.allreduce_model(variant, xs, wire, scale, local, staged=mode != "inplace")
    bufs = [_sentinel(n + SENT_VECS * epv, wire) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
    else:
        src = [torch.cat([xs[r], _sentinel(SENT_VECS * epv, local, "cpu")]).cuda() for r in range(world)]
        dst = src if mode == "alias" else [_sentinel(n + SENT_VECS * epv, local) for _ in range(world)]
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


def allreduce_cases(variant, world, sms):
    """(n_vec, max_blocks, combo, scale) per case: every size at max_blocks 1, 3 and SMs // world; every (wire, mode, local)
    combination once per max_blocks and so with every scale."""
    scales = [1.0, 1.0 / world, 0.3]
    out = []
    for m, mb in enumerate([1, 3, sms // world]):
        tail = 2 * M.THREADS * mb                 # one full pass of the unrolled peer-load loop at mb CTAs
        if variant == M.LL:
            sizes = [1, 511, 512, 513, 1023, 1025, 4095, M.LL_CAP_VEC]
        elif variant == M.ONESHOT:
            sizes = [1, 511, 512, 513, tail - 1, tail + 1, M.LL_CAP_VEC, 3 * tail + 700]
        else:                                     # two-shot: slices, several of them not multiples of 512
            sizes = [world * s for s in (1, 511, 512, 513, tail - 1, tail + 1, 700, 3 * tail + 300)]
        for i, n_vec in enumerate(sizes):
            out.append((n_vec, mb, COMBOS[(i + m) % len(COMBOS)], scales[m]))
    return out


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
