"""Reduce-scatter and all-to-all (csrc/allreduce.cu segments_pull_kernel / segments_ll_kernel) on ONE GPU with W emulated
ranks, bit for bit against tests/reduce_scatter_alltoall_model.py.

The harness is tests/emulated_ranks.py's: each rank has its own buffers, signal pad, LL inbox and stream, the W
launches go out back to back, and no case runs more CTAs than the GPU has SMs.  Outputs, symmetric buffers, the sentinels
behind them and every src are compared whole.  The reduce-scatter is also compared with the all-reduce kernels' slice on the
same inputs, the new calls share pads and inboxes with every other kind of call through the uint32 epoch wrap, and the last
tests drive ``SymmWorld.reduce_scatter_`` / ``all_to_all_`` for W ranks built over the emulated buffers.
"""
import pytest
import torch

import collectives_model as CM
import comm_model as M
import emulated_ranks as E
import reduce_dtypes_model as RM
import reduce_scatter_alltoall_model as RS
from emulated_ranks import (C, _any_nan, _bytes_cpu, _grid, _raw, _unaligned, alltoall_call, pytestmark,  # noqa: F401
                            reduce_scatter_call, sms)

VARIANTS = [M.ONESHOT, M.LL]                     # pull (what one-shot, two-shot and NVLS run here) and LL
VARIANT_IDS = ["pull", "ll"]
OPS = [CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN]


def segment_sizes(variant, mb):
    """Vectors per segment: across the LL inbox's block boundaries up to LL_CAP_VEC, and across every grid and unroll tail
    of the pull loop at mb CTAs, including LL_CAP_VEC + 1 (the first segment LL cannot take)."""
    tail = 2 * M.THREADS * mb
    if variant == M.LL:
        return [1, 511, 512, 513, 1025, 4095, M.LL_CAP_VEC]
    return [1, 511, 512, 513, tail - 1, tail + 1, M.LL_CAP_VEC + 1, 3 * tail + 300]


def _cases(variant, world, sms):
    k = 0
    for m, mb in enumerate([1, 3, sms // world]):
        for seg_vec in segment_sizes(variant, mb):
            yield seg_vec, mb, k, m
            k += 1


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_reduce_scatter_matches_the_model_bit_for_bit(C, sms, world, variant):
    for seg_vec, mb, k, m in _cases(variant, world, sms):
        dtype = RS.DTYPES[(k + 2 * m) % len(RS.DTYPES)]
        reduce_scatter_call(C, E.World(world, sms), variant, dtype, OPS[(k + m) % 4], seg_vec, mb,
                            ["inplace", "staged"][(k + m) % 2], seed=21000 * world + 100 * variant + k)


@pytest.mark.parametrize("dtype", RS.DTYPES, ids=[RS.NAMES[d] for d in RS.DTYPES])
def test_every_op_of_each_dtype(C, sms, dtype):
    """Each (dtype, op, variant, mode) once at world 4, at a size with a partial last block."""
    world = 4
    for variant in VARIANTS:
        for op in OPS:
            for mode in ("inplace", "staged"):
                reduce_scatter_call(C, E.World(world, sms), variant, dtype, op, 1000, 3, mode, seed=17 * variant + 5 * op)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_alltoall_matches_the_model_bit_for_bit(C, sms, world, variant):
    for seg_vec, mb, k, m in _cases(variant, world, sms):
        alltoall_call(C, E.World(world, sms), variant, seg_vec, mb, ["staged", "buffer"][(k + m) % 2],
                      seed=23000 * world + 100 * variant + k)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_reduce_scatter_equals_the_all_reduce_slice_on_the_same_inputs(C, sms, world):
    """Every dtype and op, pull and LL: segment r of the reduce-scatter is bit for bit slice r of the all-reduce kernels'
    result (one-shot, two-shot and LL) of the same inputs, NaN payloads included."""
    for d, dtype in enumerate(RS.DTYPES):
        for op in OPS:
            epv = RS.elems_per_vec(dtype)
            seg_vec = 300
            n = world * seg_vec * epv
            xs = [RM.as_bytes(x).cuda().view(dtype) for x in RS.make_inputs(op, dtype, world, n, 41 * d + op)]
            kop, code = RM.kernel_op(op, dtype), RM.CODES[dtype]
            for ar_variant in (M.ONESHOT, M.TWOSHOT, M.LL):
                W = E.World(world, sms)
                ar_bufs = [x.clone() for x in xs]
                ptrs = [b.data_ptr() for b in ar_bufs]
                inbox, cap = E._inbox(W, ar_variant)
                W.launch(M.grid_blocks(ar_variant, world * seg_vec, world, 3),
                         lambda r: C.allreduce(ar_variant, dtype == torch.bfloat16, ptrs, W.sig_ptrs, 0, None, None,
                                               world * seg_vec, 1.0, r, world, 3, inbox, cap, kop, -1, dtype=code))
                for variant in VARIANTS:
                    bufs = [torch.zeros_like(x) for x in xs]
                    outs = [torch.zeros(seg_vec * epv, dtype=dtype, device="cuda") for _ in range(world)]
                    bptrs = [b.data_ptr() for b in bufs]
                    inbox, cap = E._inbox(W, variant)
                    W.launch(_grid(variant, seg_vec, 3),
                             lambda r: C.reduce_scatter(variant, bptrs, W.sig_ptrs, xs[r], outs[r], world * seg_vec, r, world,
                                                        3, inbox, cap, kop, code))
                    want = [RM.as_bytes(RS.segment(ar_bufs[r], r, world)).cpu() for r in range(world)]
                    RM.assert_bits_equal(f"{RS.NAMES[dtype]} op {op} all-reduce {M.VARIANT_NAMES[ar_variant]} vs "
                                         f"reduce-scatter {M.VARIANT_NAMES[variant]} world {world}", _bytes_cpu(outs), want)


# ---------------------------------------------------------------------------------------------------------- sequences
@pytest.mark.parametrize("world", range(1, 9))
def test_new_calls_share_pads_and_inboxes_with_every_kind_through_the_epoch_wrap(C, sms, world):
    """One set of pads and inboxes, starting 5 before the uint32 wrap: reduce-scatters and all-to-alls in both variants and
    modes between all-reduces, broadcasts, all-gathers, scatters, gathers and barriers; every call matches its model and
    the per-block epochs agree on every rank at the end."""
    W = E.World(world, sms, pad_start=E.WRAP)
    f32, b16 = torch.float32, torch.bfloat16
    last, mid = world - 1, world // 2
    calls = [("rs", M.LL, torch.int64, CM.SUM, 1000, 3, "inplace"), ("a2a", M.LL, 700, 1, "staged"),
             ("ar", M.LL, CM.MAX, 1000, 3, f32, "inplace", -1), ("rs", M.ONESHOT, torch.float32, CM.SUM, 3000, 3, "staged"),
             ("sc", M.LL, 1000, 3, "inplace", last), "barrier", ("a2a", M.ONESHOT, 2000, 2, "buffer"),
             ("rs", M.LL, torch.bool, CM.SUM, 4096, 1, "staged"), ("ga", M.TWOSHOT, 600, 2, "staged", 0),
             ("ag", M.LL, 513, 2, "inplace"), ("a2a", M.LL, 4096, 3, "buffer"), ("bc", M.LL, 700, 1, "staged", last),
             ("rs", M.ONESHOT, torch.bfloat16, CM.MIN, 5000, 2, "inplace"), ("ar", M.TWOSHOT, CM.SUM, world * 900, 3, b16,
                                                                              "staged", mid),
             ("a2a", M.ONESHOT, 513, 3, "staged"), ("ga", M.LL, 513, 3, "inplace", 0), "barrier",
             ("rs", M.LL, torch.float16, CM.PRODUCT, 513, 3, "staged"), ("sc", M.ONESHOT, 3000, 2, "staged", mid),
             ("a2a", M.LL, 1, 1, "staged"), ("rs", M.ONESHOT, torch.uint8, CM.MAX, 700, 1, "inplace")]
    for k, c in enumerate(calls):
        seed = 151 * world + k
        if c == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
        elif c[0] == "rs":
            _, variant, dtype, op, seg_vec, mb, mode = c
            reduce_scatter_call(C, W, variant, dtype, op, seg_vec, mb, mode, seed)
        elif c[0] == "a2a":
            _, variant, seg_vec, mb, mode = c
            alltoall_call(C, W, variant, seg_vec, mb, mode, seed)
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
            (E.scatter_call if kind == "sc" else E.gather_call)(C, W, variant, seg_vec, mb, mode, root, seed)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 100


# ---------------------------------------------------------------------------------------------------------- SymmWorld
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_reduce_scatter_routes_stages_and_copies_out(C, sms, world):
    """``reduce_scatter_`` of every dtype with tensor and list inputs (one block, separate tensors), ragged segments,
    unaligned tensors, an output that aliases the input's own slice or another whole slice (written in the kernel) or lies
    inside the input at half a segment's offset (through the staging buffer), on both sides of the LL / pull threshold; the
    group's global ranks are not 0..W-1.  Every rank's output is checked bit for bit against the model's segment r."""
    worlds, keep = E.symm_worlds(world, sms, [10 + 3 * r for r in range(world)])
    for k, numel in enumerate([5, 1024, 3001, 12288, 40000]):
        for d, dtype in enumerate(RS.DTYPES):
            op = OPS[(k + d) % 4]
            form = ["tensor", "block", "list", "alias", "shifted", "other_slice"][(k + d) % 6]
            if form == "shifted" and world == 1:
                form = "tensor"                         # one segment: no room for an output at half a segment's offset
            unaligned = (k + d) % 3 == 1 and form in ("tensor", "block", "list")
            xs = RS.make_inputs(op, dtype, world, world * numel, 300 * world + 10 * k + d)
            # a world of 1 launches nothing (as all_reduce_): the output is a copy of the input, NaN payloads included
            want = [RM.as_bytes(xs[0] if world == 1 else RS.reduce_scatter_result(op, xs, r)) for r in range(world)]
            ins = [RM.as_bytes(x).cuda().view(dtype) for x in xs]
            if unaligned:
                ins = [_unaligned(x) for x in ins]
            if form == "alias":
                outs = [x.view(world, numel)[r] for r, x in enumerate(ins)]
            elif form == "other_slice":
                outs = [x.view(world, numel)[(r + 1) % world] for r, x in enumerate(ins)]
            elif form == "shifted":
                outs = [x[numel // 2:numel // 2 + numel] for x in ins]
            else:
                outs = [torch.zeros(numel, dtype=dtype, device="cuda") for _ in range(world)]
                if unaligned:
                    outs = [_unaligned(o) for o in outs]
            if form == "block":
                args = [list(x.view(world, numel).unbind(0)) for x in ins]
            elif form == "list":
                args = [[s.clone() for s in x.view(world, numel).unbind(0)] for x in ins]
            else:
                args = ins
            E.on_ranks(worlds, lambda r, w: w.reduce_scatter_(outs[r], args[r], op))
            RM.assert_bits_equal(f"reduce_scatter_ {RS.NAMES[dtype]} {CM.OP_NAMES[op]} {numel} {form} unaligned {unaligned}",
                                 _bytes_cpu(outs), want, _any_nan(op, dtype))
    w0 = worlds[0]
    t = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="SUM, PRODUCT, MAX and MIN"):
        w0.reduce_scatter_(t, t.repeat(world), torch.distributed.ReduceOp.AVG)
    with pytest.raises(TypeError):
        w0.reduce_scatter_(torch.zeros(4, dtype=torch.int16, device="cuda"), torch.zeros(4 * world, dtype=torch.int16,
                                                                                         device="cuda"))
    with pytest.raises(ValueError, match="world x the output's"):
        w0.reduce_scatter_(t, t.repeat(world + 1))
    with pytest.raises(ValueError, match=f"needs {world} input tensors"):
        w0.reduce_scatter_(t, [t] * (world + 1))
    with pytest.raises(ValueError, match="output's dtype and size"):
        w0.reduce_scatter_(t, [torch.zeros(5, dtype=torch.int32, device="cuda")] * world)
    del keep


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_all_to_all_routes_stages_and_copies_out(C, sms, world):
    """``all_to_all_`` of int64 / bf16 / uint8 payloads at ragged sizes, aligned and unaligned, an output that is the input
    (ragged through the staging buffer; aligned in place in the kernel, pull and LL), and segments of LL_CAP_VEC and
    LL_CAP_VEC + 1 vectors (the last one LL can take, the first it cannot)."""
    worlds, keep = E.symm_worlds(world, sms, [10 + 3 * r for r in range(world)])
    for k, numel in enumerate([5, 1024, 3001, 12288, 40000, 16 * M.LL_CAP_VEC, 16 * (M.LL_CAP_VEC + 1), 512]):
        dtype = [torch.int64, torch.bfloat16, torch.uint8][k % 3] if k < 5 else torch.uint8
        unaligned = k % 3 == 1 and k < 5
        same = k in (2, 3, 7)
        xs = [_raw(dtype, world * numel, 1000 * world + 10 * k + r) for r in range(world)]
        want = [torch.cat([x.view(world, numel)[r] for x in xs]) for r in range(world)]
        ins = [x.cuda() for x in xs]
        outs = ins if same else [torch.zeros_like(x) for x in ins]
        if unaligned:
            ins = [_unaligned(x) for x in ins]
            outs = [_unaligned(o) for o in outs]
        E.on_ranks(worlds, lambda r, w: w.all_to_all_(outs[r], ins[r]))
        for r in range(world):
            assert E._bits_equal(outs[r], want[r]), ("all_to_all_", dtype, numel, unaligned, same, r)
            if not same:
                assert E._bits_equal(ins[r], xs[r]), ("all_to_all_: input changed", numel, r)
    w0 = worlds[0]
    if world > 1:
        with pytest.raises(ValueError, match="multiple of world"):
            w0.all_to_all_(torch.zeros(world + 1, device="cuda"), torch.zeros(world + 1, device="cuda"))
    with pytest.raises(ValueError, match="one dtype and size"):
        w0.all_to_all_(torch.zeros(world, device="cuda"), torch.zeros(world, dtype=torch.int32, device="cuda"))
    del keep
