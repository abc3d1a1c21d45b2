"""Scatter from a root and gather to a root (csrc/allreduce.cu) on ONE GPU with W emulated ranks, bit for bit against
tests/scatter_gather_model.py.

The harness is tests/emulated_ranks.py's: each rank has its own buffers, signal pad, LL inbox and stream, the W
launches go out back to back, and no case runs more CTAs than the GPU has SMs.  Outputs, symmetric buffers, the sentinels
behind them and every src are compared whole, so "a non-root leaves its output alone", "a non-root's src is never read" and
"src is left untouched" are checked too.  The last tests drive ``SymmWorld.scatter_`` / ``gather_`` for W ranks built over
the emulated buffers, one rank per stream.
"""
import pytest
import torch

import collectives_model as CM
import comm_model as M
import emulated_ranks as E
from emulated_ranks import (C, VARIANT_IDS, VARIANTS, _raw, _unaligned, gather_call, pytestmark,  # noqa: F401
                            scatter_call, sms)


def segment_sizes(kind, variant, world, mb):
    """Per-rank vectors: across the LL inbox's block boundaries up to LL_CAP_VEC, and across every grid and unroll tail of
    the loop each variant runs (one-shot gather: the world x larger output; one-shot scatter: one segment; two-shot: one
    slice)."""
    tail = 2 * M.THREADS * mb                     # one full pass of the unrolled loop at mb CTAs
    if variant == M.LL:
        return [1, 511, 512, 513, 1025, 4095, M.LL_CAP_VEC]
    if variant == M.ONESHOT and kind == "gather":
        return [1, 511, 513, max(tail // world - 1, 1), tail // world + 1, 700, (3 * tail + 700) // world]
    return [1, 511, 512, 513, tail - 1, tail + 1, 700, 3 * tail + 300]


def _cases(kind, variant, world, sms):
    roots = [0, world - 1, world // 2]
    k = 0
    for m, mb in enumerate([1, 3, sms // world]):
        for seg_vec in segment_sizes(kind, variant, world, mb):
            yield seg_vec, mb, ["inplace", "staged"][(k + m) % 2], roots[(k // 2) % 3], k
            k += 1


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_gather_matches_the_model_bit_for_bit(C, sms, world, variant):
    for seg_vec, mb, mode, root, k in _cases("gather", variant, world, sms):
        gather_call(C, E.World(world, sms), variant, seg_vec, mb, mode, root, seed=11000 * world + 100 * variant + k)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_scatter_matches_the_model_bit_for_bit(C, sms, world, variant):
    for seg_vec, mb, mode, root, k in _cases("scatter", variant, world, sms):
        scatter_call(C, E.World(world, sms), variant, seg_vec, mb, mode, root, seed=13000 * world + 100 * variant + k)


# ---------------------------------------------------------------------------------------------------------- sequences
@pytest.mark.parametrize("world", range(1, 9))
def test_scatter_and_gather_share_pads_and_inboxes_with_every_kind_through_the_epoch_wrap(C, sms, world):
    """One set of pads and inboxes, starting 5 before the uint32 wrap, runs scatters and gathers in every variant, mode and
    root between all-reduces, reduces, broadcasts, all-gathers and barriers; every call matches the model and the per-block
    epochs agree on every rank at the end."""
    W = E.World(world, sms, pad_start=E.WRAP)
    f32, b16 = torch.float32, torch.bfloat16
    last, mid = world - 1, world // 2
    calls = [("sc", M.LL, 1000, 3, "inplace", last), ("ga", M.ONESHOT, 600, 2, "staged", 0),
             ("ar", M.LL, CM.MAX, 1000, 3, f32, "inplace", -1), ("ga", M.LL, 4096, 1, "staged", mid), "barrier",
             ("sc", M.TWOSHOT, 700, 3, "staged", 0), ("ag", M.LL, 513, 2, "inplace"),
             ("sc", M.ONESHOT, 3000, 2, "inplace", mid), ("ga", M.TWOSHOT, 1500, 3, "inplace", last),
             ("bc", M.LL, 700, 1, "staged", last), ("sc", M.LL, 4096, 3, "staged", 0),
             ("ar", M.ONESHOT, CM.PRODUCT, 3000, 3, b16, "staged", mid), ("ga", M.LL, 513, 3, "inplace", 0), "barrier",
             ("sc", M.ONESHOT, 513, 1, "staged", last), ("ag", M.TWOSHOT, 300, 2, "staged"),
             ("ga", M.ONESHOT, 2000, 3, "inplace", mid), ("sc", M.TWOSHOT, 1025, 2, "inplace", mid),
             ("ar", M.TWOSHOT, CM.SUM, world * 900, 3, f32, "staged", mid), ("ga", M.TWOSHOT, 300, 1, "staged", 0),
             ("sc", M.LL, 2000, 2, "inplace", 0)]
    for k, c in enumerate(calls):
        seed = 97 * world + k
        if c == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
        elif c[0] == "ar":
            _, variant, op, n_vec, mb, wire, mode, root = c
            E.reduce_call(C, W, variant, op, n_vec, mb, wire, mode, wire, root, seed)
        elif c[0] == "bc":
            _, variant, n_vec, mb, mode, root = c
            E.broadcast_call(C, W, variant, n_vec, mb, mode, root, seed)
        elif c[0] == "ag":
            _, variant, seg_vec, mb, mode = c
            E.allgather_call(C, W, variant, seg_vec, mb, mode, seed)
        else:
            kind, variant, seg_vec, mb, mode, root = c
            (scatter_call if kind == "sc" else gather_call)(C, W, variant, seg_vec, mb, mode, root, seed)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 100


# ---------------------------------------------------------------------------------------------------------- SymmWorld
def _lists(world, numel, dtype, block):
    """world outputs per rank: views of one block, or separate tensors."""
    if block:
        return [list(torch.zeros(world * numel, dtype=dtype, device="cuda").view(world, numel).unbind(0))
                for _ in range(world)]
    return [[torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)] for _ in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_scatter_and_gather_route_stage_and_copy_out(C, sms, world):
    """int64 / bf16 / uint8 at sizes on both sides of the LL and one-shot thresholds and ragged ones, block and separate
    lists, aligned and unaligned tensors; roots given as global ranks of a group whose ranks are not 0..W-1.  A non-root's
    list is never read or written."""
    globals_ = [10 + 3 * r for r in range(world)]
    worlds, keep = E.symm_worlds(world, sms, globals_)
    for k, numel in enumerate([5, 1024, 3001, 12288, 40000, 24000, 60001]):
        dtype = [torch.int64, torch.bfloat16, torch.uint8][k % 3]
        root = [0, world - 1, world // 2][k % 3]
        block = k % 2 == 0
        unaligned = k % 4 == 1
        segs = [_raw(dtype, numel, 1000 * world + 10 * k + r) for r in range(world)]
        # scatter: the root's list holds the segments; every other rank's list holds decoys that must stay as they are
        lists = _lists(world, numel, dtype, block)
        decoy = _raw(dtype, numel, 7)
        for r in range(world):
            for s in range(world):
                lists[r][s].copy_(segs[s] if r == root else decoy)
        ts = [torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)]
        if unaligned:
            ts = [_unaligned(t) for t in ts]
        E.on_ranks(worlds, lambda r, w: w.scatter_(ts[r], lists[r], globals_[root]))
        for r in range(world):
            assert E._bits_equal(ts[r], segs[r]), ("scatter", dtype, numel, block, unaligned, r)
            for s in range(world):
                assert E._bits_equal(lists[r][s], segs[s] if r == root else decoy), ("scatter: list written", numel, r, s)
        # gather: rank r's tensor lands in the root's list; the others' lists are left alone
        ins = [segs[r].cuda() for r in range(world)]
        if unaligned:
            ins = [_unaligned(x) for x in ins]
        outs = _lists(world, numel, dtype, block)
        for r in range(world):
            for s in range(world):
                outs[r][s].copy_(decoy)
        E.on_ranks(worlds, lambda r, w: w.gather_(ins[r], outs[r] if r == root else None, globals_[root]))
        for r in range(world):
            for s in range(world):
                assert E._bits_equal(outs[r][s], segs[s] if r == root else decoy), ("gather", dtype, numel, block, r, s)
            assert E._bits_equal(ins[r], segs[r]), ("gather: input changed", numel, r)
    del keep


def test_symm_world_refuses_a_bad_root_list_before_any_launch(C, sms):
    """World 1: the root's list of the wrong length, dtype or size raises (as torch does), and so does a root outside the
    world; nothing is launched."""
    worlds, keep = E.symm_worlds(1, sms, [4])
    w = worlds[0]
    t = torch.zeros(8, dtype=torch.int64, device="cuda")
    for fn in (w.scatter_, w.gather_):
        with pytest.raises(ValueError, match="needs 1 tensors on the root"):
            fn(t, [t.clone(), t.clone()], 4)
        with pytest.raises(ValueError, match="needs 1 tensors on the root"):
            fn(t, None, 4)
        with pytest.raises(ValueError, match="dtype and size"):
            fn(t, [torch.zeros(8, dtype=torch.int32, device="cuda")], 4)
        with pytest.raises(ValueError, match="dtype and size"):
            fn(t, [torch.zeros(9, dtype=torch.int64, device="cuda")], 4)
        with pytest.raises(TypeError, match="contiguous CUDA"):
            fn(t, [torch.zeros(8, dtype=torch.int64)], 4)
        with pytest.raises(ValueError, match="not in this world"):
            fn(t, [t.clone()], 0)
    x = torch.arange(8, dtype=torch.int64, device="cuda")
    out = [torch.zeros_like(x)]
    w.gather_(x, out, 4)
    assert torch.equal(out[0], x)
    y = torch.zeros_like(x)
    w.scatter_(y, [x], 4)
    assert torch.equal(y, x)
    del keep
