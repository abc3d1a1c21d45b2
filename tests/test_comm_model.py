"""CPU checks of tests/comm_model.py, the bit-exact model the emulated-world GPU tests compare the communication kernels
with: the model agrees with an fp64 all-reduce within its error bound, its launch constants are the kernel sources', and
the bit checker reports the first wrong rank and vector for faults that the 1e-5 / 2e-2 tolerances of the multi-GPU tests
would let through."""
import os

import pytest
import torch

import comm_model as M

F32, B16 = torch.float32, torch.bfloat16
# (wire, local dtype, staged): in place in the wire dtype, src / dst in the wire dtype, fp32 src / dst over a bf16 wire
COMBOS = [(F32, F32, False), (F32, F32, True), (B16, B16, False), (B16, B16, True), (B16, F32, True)]


def test_launch_constants_are_the_kernel_sources():
    k = M.kernel_constants()
    assert k == {"threads": M.THREADS, "unroll": M.UNROLL, "max_blocks": M.MAX_BLOCKS, "max_ranks": M.MAX_RANKS,
                 "sgd_threads": M.THREADS}


@pytest.mark.parametrize("variant", [M.ONESHOT, M.TWOSHOT, M.LL], ids=["oneshot", "twoshot", "ll"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("combo", COMBOS, ids=["f32-inplace", "f32-staged", "b16-inplace", "b16-staged", "f32-over-b16"])
def test_model_agrees_with_fp64_within_its_bound(variant, world, combo):
    wire, local, staged = combo
    for scale in (1.0, 1.0 / world, 0.3):
        xs = M.make_inputs(world, 4096, local, seed=world * 31 + variant)
        want = M.allreduce_model(variant, xs, wire, scale, local, staged)
        out = want["out"][0]
        assert out.dtype == local
        rounded = wire == B16 and (variant == M.TWOSHOT or local == B16)
        M.check_against_fp64(f"{variant} {combo} {scale}", out, xs, scale, wire, rounded)
        assert all(torch.equal(o.view(torch.int16 if o.dtype == B16 else torch.int32),
                               out.view(torch.int16 if o.dtype == B16 else torch.int32)) for o in want["out"])


def test_inputs_hold_ties_signed_zeros_and_infinities():
    xs = M.make_inputs(3, 4096, F32, seed=1)
    bits = torch.stack([x.view(torch.int32) for x in xs])
    assert bool(((bits & 0xFFFF) == 0x8000).any())                       # exact bf16 ties
    assert bool((torch.stack(xs) == 0).any() and torch.signbit(torch.stack(xs)[torch.stack(xs) == 0]).any())
    inf = torch.isinf(torch.stack(xs))
    assert bool(inf.any()) and int(inf.sum(0).max()) == 1                  # one rank per position: never Inf - Inf
    tie = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8])                  # halfway cases: RN-even goes down, then up
    assert M.bf16_rn(tie).tolist() == [1.0, 1.0 + 2 ** -6]


def test_sgd_model_is_the_fp32_fma_for_power_of_two_mu_and_lr():
    g = torch.Generator().manual_seed(3)
    grads = [torch.randn(4096, generator=g) for _ in range(3)]
    p, m = torch.randn(4096, generator=g), torch.randn(4096, generator=g)
    mu, lr, scale = 0.5, 0.125, 1.0 / 3
    for bf16 in (False, True):
        p1, m1 = M.sgd_model(grads, p, m, scale, mu, lr, bf16)
        gs = torch.zeros(4096)
        for t in grads:
            gs = gs + (t.to(B16).float() if bf16 else t)
        gs = gs * torch.tensor(scale, dtype=F32)
        m2 = m * mu + gs                   # mu * m is exact in fp32: one rounding, as fmaf
        p2 = p - m2 * lr
        assert torch.equal(m1.view(torch.int32), m2.view(torch.int32)) and torch.equal(p1.view(torch.int32), p2.view(torch.int32))
    with pytest.raises(AssertionError):
        M.sgd_model(grads, p, m, scale, 0.9, lr, False)


def test_aux_slots_are_distinct_and_inside_aux():
    w2f, w2b = M.aux_index()
    assert sorted(w2f.tolist()) == list(range(5000))
    assert len(set(w2b.tolist())) == 5000 and 5000 <= int(w2b.min()) and int(w2b.max()) < M.AUX_N
    assert set((w2b - 5000).remainder(8).tolist()) == {0, 1, 2, 3, 4}       # slots 5..7 of each group of 8 stay free


# ---------------------------------------------------------------------------------------------------- planted faults
def _loose_equal(a, b, wire):
    tol = 2e-2 if wire == B16 else 1e-5
    return torch.allclose(a.float(), b.float(), rtol=tol, atol=tol)


def _mismatch(got, want, wire, expect_rank=None, expect_vec=None):
    m = M.first_mismatch(got, want, M.elems_per_vec(wire))
    assert m is not None, "the planted fault went unnoticed"
    if expect_rank is not None:
        assert m[0] == expect_rank, m
    if expect_vec is not None:
        assert m[1] == expect_vec, m
    with pytest.raises(AssertionError, match=f"rank {m[0]}, vector {m[1]} "):
        M.assert_bits_equal("fault", got, want, M.elems_per_vec(wire))
    return m


def _sum(terms, scale):
    return M.reduce_scaled(terms, scale)


def test_reversed_and_rotated_rank_order_are_caught():
    world, wire = 5, F32
    xs = M.make_inputs(world, 8192, F32, seed=11, specials=False)
    want = M.allreduce_model(M.ONESHOT, xs, wire, 1.0, F32, False)["out"]
    rev = [_sum(xs[::-1], 1.0)] * world
    assert all(_loose_equal(a, b, wire) for a, b in zip(rev, want))
    _mismatch(rev, want, wire, expect_rank=0)
    rot = [_sum(xs[r:] + xs[:r], 1.0) for r in range(world)]                # each rank starts with its own term
    assert all(_loose_equal(a, b, wire) for a, b in zip(rot, want))
    _mismatch(rot, want, wire, expect_rank=1)                              # rank 0's order is the right one


def test_skipped_or_doubled_bf16_rounding_is_caught():
    world, wire = 4, B16
    xs = M.make_inputs(world, 8192, F32, seed=12)
    want = M.allreduce_model(M.ONESHOT, xs, wire, 0.3, F32, True)["out"]
    skipped = [_sum(xs, 0.3)] * world                                      # fp32 src sent without the bf16 rounding
    assert all(_loose_equal(a, b, wire) for a, b in zip(skipped, want))
    _mismatch(skipped, want, wire)
    xb = M.make_inputs(world, 8192, B16, seed=13)
    want = M.allreduce_model(M.TWOSHOT, xb, wire, 0.3, B16, False)["out"]
    acc = _sum([x.float() for x in xb], 1.0)
    twice = [(M.bf16_rn(acc) * M.fp32_scale(0.3)).to(B16)] * world        # rounded before the scale, and again after
    assert all(_loose_equal(a, b, wire) for a, b in zip(twice, want))
    _mismatch(twice, want, wire)


def test_scale_before_the_sum_is_caught():
    world, wire = 3, F32
    xs = M.make_inputs(world, 8192, F32, seed=14, specials=False)
    want = M.allreduce_model(M.LL, xs, wire, 0.3, F32, False)["out"]
    early = [_sum([x * M.fp32_scale(0.3) for x in xs], 1.0)] * world
    assert all(_loose_equal(a, b, wire) for a, b in zip(early, want))
    _mismatch(early, want, wire)


def test_twoshot_with_one_shot_rounding_is_caught():
    """Two-shot packs the reduced slice to the wire dtype, so an fp32 dst over a bf16 wire gets bf16 values."""
    world, wire = 4, B16
    xs = M.make_inputs(world, 8192, F32, seed=15)
    want = M.allreduce_model(M.TWOSHOT, xs, wire, 1.0 / world, F32, True)["out"]
    oneshot = M.allreduce_model(M.ONESHOT, xs, wire, 1.0 / world, F32, True)["out"]
    assert all(_loose_equal(a, b, wire) for a, b in zip(oneshot, want))
    _mismatch(oneshot, want, wire)


def test_unreduced_tail_vectors_are_caught():
    world, wire, k = 3, F32, 700
    n_vec = world * k + 2                                          # a two-shot slice of n_vec // world leaves 2 vectors
    xs = M.make_inputs(world, n_vec * 4, F32, seed=16, specials=False)
    want = M.allreduce_model(M.ONESHOT, xs, wire, 1.0, F32, False)["out"]
    got = [w.clone() for w in want]
    for r in range(world):
        got[r][world * k * 4:] = xs[r][world * k * 4:]             # in place: those vectors keep the rank's own data
    _mismatch(got, want, wire, expect_rank=0, expect_vec=world * k)


def test_unreduced_last_grid_stride_pass_is_caught():
    world, wire, mb = 2, F32, 3
    per_pass = M.UNROLL * M.THREADS * mb                           # one pass of the one-shot loop at mb CTAs
    n_vec = 3 * per_pass + 5
    xs = M.make_inputs(world, n_vec * 4, F32, seed=17, specials=False)
    want = M.allreduce_model(M.ONESHOT, xs, wire, 1.0, F32, False)["out"]
    last = (n_vec - 1) // per_pass * per_pass
    got = [w.clone() for w in want]
    for r in range(world):
        got[r][last * 4:] = xs[r][last * 4:]
    _mismatch(got, want, wire, expect_rank=0, expect_vec=last)


def test_zeroing_the_wrong_parity_bucket_is_caught():
    n = 4096
    bucket = torch.randn(2 * n, generator=torch.Generator().manual_seed(18))
    for cur in (0, 1):
        want = M.bucket_model(bucket, n, cur, True, True)
        assert torch.equal(want[cur * n:(cur + 1) * n], bucket[cur * n:(cur + 1) * n])
        wrong = M.bucket_model(bucket, n, cur ^ 1, True, True)
        _mismatch([wrong], [want], F32, expect_rank=0, expect_vec=0)


# ---------------------------------------------------------------------------------------------------- launcher input checks
# The bindings refuse what the kernels would silently get wrong, before anything is launched (the messages are the
# checks', not a launch error; no pointer here is ever dereferenced).
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def _allreduce(C, variant=M.ONESHOT, n_vec=64, rank=0, world=2, bufs=None, sigs=None, inbox=None):
    bufs = [0x1000 * (i + 1) for i in range(world)] if bufs is None else bufs
    sigs = [0x2000 * (i + 1) for i in range(world)] if sigs is None else sigs
    inbox = ([0x3000 * (i + 1) for i in range(world)] if variant == M.LL else []) if inbox is None else inbox
    C.allreduce(variant, False, bufs, sigs, 0, None, None, n_vec, 1.0, rank, world, 1, inbox, M.LL_CAP_VEC)


@pytest.mark.parametrize("variant", [M.TWOSHOT, M.NVLS], ids=["twoshot", "nvls"])
def test_allreduce_refuses_a_slice_remainder(variant):
    with pytest.raises(RuntimeError, match="n_vec must be a multiple of world"):
        _allreduce(_C(), variant, n_vec=3 * 100 + 1, world=3)


@pytest.mark.parametrize("rank,world", [(0, 0), (0, 9), (-1, 2), (2, 2)])
def test_comm_bindings_refuse_a_bad_world_or_rank(rank, world):
    C = _C()
    n = max(world, 1)
    with pytest.raises(RuntimeError, match="world must be in 1..8|is outside"):
        _allreduce(C, rank=rank, world=world, bufs=[0x1000] * n, sigs=[0x2000] * n)
    with pytest.raises(RuntimeError, match="world must be in 1..8|is outside"):
        C.barrier([0x2000] * n, rank, world)
    with pytest.raises(RuntimeError, match="world must be in 1..8|is outside"):
        C.allreduce_sgd([0x1000] * n, [0x2000] * n, torch.zeros(64), torch.zeros(64), None, 0.125, 0.5, 1.0, rank, world, True)


@pytest.mark.parametrize("variant", [-1, 4, 7])
def test_allreduce_refuses_an_unknown_variant(variant):
    with pytest.raises(RuntimeError, match="variant must be 0"):
        _allreduce(_C(), variant)


def test_comm_bindings_refuse_pointer_lists_of_the_wrong_length():
    C = _C()
    with pytest.raises(RuntimeError, match="one buffer and one signal pad per rank"):
        _allreduce(C, world=3, bufs=[0x1000, 0x2000])
    with pytest.raises(RuntimeError, match="one buffer and one signal pad per rank"):
        _allreduce(C, world=3, sigs=[0x1000, 0x2000, 0x3000, 0x4000])
    with pytest.raises(RuntimeError, match="one LL inbox per rank"):
        _allreduce(C, M.LL, world=3, inbox=[0x1000, 0x2000])
    with pytest.raises(RuntimeError, match="one LL inbox per rank"):
        _allreduce(C, M.LL, world=3, inbox=[])
    with pytest.raises(RuntimeError, match="one signal pad per rank"):
        C.barrier([0x2000], 0, 2)
    p = torch.zeros(64)
    with pytest.raises(RuntimeError, match="one gradient bucket and one signal pad per rank"):
        C.allreduce_sgd([0x1000], [0x2000, 0x3000], p, p.clone(), None, 0.125, 0.5, 1.0, 0, 2, True)
    with pytest.raises(RuntimeError, match="one gradient bucket and one signal pad per rank"):
        C.allreduce_sgd([0x1000, 0x2000], [0x2000], p, p.clone(), None, 0.125, 0.5, 1.0, 0, 2, True)
