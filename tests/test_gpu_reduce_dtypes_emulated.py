"""The all-reduce and reduce of fp16, fp64, int8, uint8, int32, int64 and bool (csrc/allreduce.cu lane types) on ONE GPU with
W emulated ranks, bit for bit against tests/reduce_dtypes_model.py.

The harness is tests/emulated_ranks.py's: each rank has its own buffers, signal pad, LL inbox and stream, the W
launches go out back to back, and no case runs more CTAs than the GPU has SMs (every CTA spins on its peers).  Outputs,
symmetric buffers and the sentinels behind them are compared whole.  The last tests drive ``SymmWorld.all_reduce_`` /
``reduce_`` for W ranks built over the emulated buffers, one rank per stream.
"""
import pytest
import torch

import collectives_model as CM
import comm_model as M
import emulated_ranks as E
import reduce_dtypes_model as RM
from emulated_ranks import C, VARIANT_IDS, VARIANTS, _bits_equal, _byte_sentinel, pytestmark, sms  # noqa: F401

OPS = [CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN]


def reduce_call(C, W, variant, dtype, op, n_vec, mb, mode, root, seed):
    world = W.world
    epv = RM.elems_per_vec(dtype)
    n = n_vec * epv
    xs = RM.make_inputs(op, dtype, world, n, seed)
    tail = E.SENT_VECS * epv
    bufs = [_byte_sentinel(n + tail, dtype) for _ in range(world)]
    src = dst = [None] * world
    if mode == "inplace":
        for r in range(world):
            bufs[r][:n].copy_(xs[r])
        outs = bufs
    else:
        src = [torch.cat([RM.as_bytes(xs[r]), RM.as_bytes(_byte_sentinel(tail, dtype, "cpu"))]).cuda().view(dtype)
               for r in range(world)]
        dst = src if mode == "alias" else [_byte_sentinel(n + tail, dtype) for _ in range(world)]
        outs = dst
    want = RM.reduce_model(variant, op, xs, mode, root, [RM.as_bytes(o).cpu() for o in outs],
                           [RM.as_bytes(b).cpu() for b in bufs])
    ptrs = [b.data_ptr() for b in bufs]
    inbox, cap = E._inbox(W, variant)
    kop = RM.kernel_op(op, dtype)
    W.launch(M.grid_blocks(variant, n_vec, world, mb),
             lambda r: C.allreduce(variant, False, ptrs, W.sig_ptrs, 0, src[r], dst[r], n_vec, 1.0, r, world, mb, inbox, cap,
                                   kop, root, dtype=RM.CODES[dtype]))
    what = (f"{RM.NAMES[dtype]} {CM.OP_NAMES[op]} root {root} {M.VARIANT_NAMES[variant]} world {world} n_vec {n_vec} "
            f"max_blocks {mb} {mode}")
    any_nan = RM.nan_any(op, dtype)
    RM.assert_bits_equal(what + ": output", [RM.as_bytes(o).cpu() for o in outs], want["out"], any_nan)
    RM.assert_bits_equal(what + ": symmetric buffers", [RM.as_bytes(b).cpu() for b in bufs], want["buf"], any_nan)


def dtype_cases(variant, world, sms):
    """(n_vec, max_blocks, dtype, op, root, mode) per case over comm_model's sizes (every grid and unroll tail at max_blocks
    1, 3 and SMs // world), each size once per dtype; ops, roots (all, 0, last, middle) and modes cycle independently."""
    roots = [-1, 0, world - 1, world // 2]
    modes = ["inplace", "staged", "alias"]
    out = []
    for k, (n_vec, mb, _, _) in enumerate(E.allreduce_cases(variant, world, sms)):
        for d, dtype in enumerate(RM.DTYPES):
            j = k * len(RM.DTYPES) + d
            out.append((n_vec, mb, dtype, OPS[(k + d) % 4], roots[(j // 4) % 4], modes[(k + 2 * d) % 3]))
    return out


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("world", range(1, 9))
def test_reductions_of_every_dtype_match_the_model_bit_for_bit(C, sms, world, variant):
    for k, (n_vec, mb, dtype, op, root, mode) in enumerate(dtype_cases(variant, world, sms)):
        reduce_call(C, E.World(world, sms), variant, dtype, op, n_vec, mb, mode, root, seed=9000 * world + 100 * variant + k)


@pytest.mark.parametrize("dtype", RM.DTYPES, ids=[RM.NAMES[d] for d in RM.DTYPES])
def test_every_op_and_root_of_each_dtype(C, sms, dtype):
    """Each (dtype, op, root) at one size per variant at world 4: the cycling above meets every combination somewhere, this
    meets each in one place."""
    world = 4
    for variant in VARIANTS:
        n_vec = 1000 if variant != M.TWOSHOT else world * 700
        for op in OPS:
            for root in (-1, 0, world - 1, world // 2):
                for mode in ("inplace", "staged"):
                    reduce_call(C, E.World(world, sms), variant, dtype, op, n_vec, 3, mode, root,
                                seed=17 * variant + 5 * op + root)


@pytest.mark.parametrize("world", range(1, 9))
def test_new_dtypes_share_pads_and_inboxes_with_every_call_through_the_epoch_wrap(C, sms, world):
    """One set of pads and inboxes, starting 5 before the uint32 wrap: new-dtype reductions interleaved with fp32 / bf16
    all-reduces, broadcasts, all-gathers and barriers in every variant; every call matches its model and the per-block
    epochs agree at the end."""
    W = E.World(world, sms, pad_start=E.WRAP)
    f32, b16 = torch.float32, torch.bfloat16
    last, mid = world - 1, world // 2
    calls = [("nd", M.LL, torch.int64, CM.SUM, 1000, 3, "inplace", -1), ("ar", M.LL, CM.MAX, 1000, 3, f32, "inplace", -1),
             ("nd", M.ONESHOT, torch.float16, CM.PRODUCT, 3000, 3, "staged", mid), ("bc", M.LL, 700, 1, "staged", last),
             ("nd", M.TWOSHOT, torch.uint8, CM.MAX, world * 300, 2, "inplace", 0), "barrier",
             ("nd", M.LL, torch.bool, CM.SUM, 4096, 1, "alias", -1), ("ag", M.LL, 4096, 1, "staged"),
             ("ar", M.TWOSHOT, CM.SUM, world * 900, 3, b16, "staged", mid), ("nd", M.LL, torch.float64, CM.MIN, 513, 3,
                                                                              "inplace", last),
             ("nd", M.ONESHOT, torch.int8, CM.SUM, 5000, 2, "alias", -1), ("bc", M.ONESHOT, 5000, 2, "inplace", 0),
             ("nd", M.TWOSHOT, torch.int32, CM.PRODUCT, world * 1500, 3, "staged", -1), "barrier",
             ("nd", M.LL, torch.float16, CM.MAX, 2000, 3, "inplace", mid), ("ag", M.TWOSHOT, 300, 2, "inplace"),
             ("ar", M.LL, CM.SUM, 4096, 3, f32, "alias", -1), ("nd", M.LL, torch.int64, CM.MIN, 4096, 3, "staged", 0)]
    for k, c in enumerate(calls):
        seed = 131 * world + k
        if c == "barrier":
            W.launch(1, lambda r: C.barrier(W.sig_ptrs, r, world))
        elif c[0] == "nd":
            _, variant, dtype, op, n_vec, mb, mode, root = c
            reduce_call(C, W, variant, dtype, op, n_vec, mb, mode, root, seed)
        elif c[0] == "ar":
            _, variant, op, n_vec, mb, wire, mode, root = c
            E.reduce_call(C, W, variant, op, n_vec, mb, wire, mode, wire, root, seed)
        elif c[0] == "bc":
            _, variant, n_vec, mb, mode, root = c
            E.broadcast_call(C, W, variant, n_vec, mb, mode, root, seed)
        else:
            _, variant, seg_vec, mb, mode = c
            E.allgather_call(C, W, variant, seg_vec, mb, mode, seed)
    ep = torch.stack([p[M.EPOCH_WORD0:M.EPOCH_WORD0 + M.MAX_BLOCKS] for p in W.pads]).cpu()
    assert bool((ep == ep[0]).all())
    assert 0 < int(ep[0, 0]) < 100


def test_nan_results_have_the_pinned_bit_patterns(C, sms):
    """fp16: a NaN result is 0x7FFF (the fp32 accumulator's NaN rounded to fp16), for SUM as for MAX; fp64 MAX / MIN return
    0x7FFFFFFFFFFFFFFF.  The model pins both; this confirms them on the device once."""
    world = 2
    for dtype, op, want in ((torch.float16, CM.SUM, RM.F16_NAN), (torch.float16, CM.MAX, RM.F16_NAN),
                            (torch.float16, CM.PRODUCT, RM.F16_NAN), (torch.float64, CM.MAX, RM.F64_NAN),
                            (torch.float64, CM.MIN, RM.F64_NAN)):
        epv = RM.elems_per_vec(dtype)
        xs = [torch.zeros(epv, dtype=dtype) for _ in range(world)]
        xs[1][0] = float("nan")
        xs[0][1] = float("inf")
        xs[1][1] = float("-inf") if op == CM.SUM else 0.0       # Inf - Inf (SUM) and Inf x 0 (PRODUCT) make NaN too
        bufs = [x.cuda() for x in xs]
        ptrs = [b.data_ptr() for b in bufs]
        W = E.World(world, sms)
        W.launch(1, lambda r: C.allreduce(M.ONESHOT, False, ptrs, W.sig_ptrs, 0, None, None, 1, 1.0, r, world, 1, [], 0, op,
                                          -1, dtype=RM.CODES[dtype]))
        got = RM.bits(bufs[0].cpu())
        mask = (1 << (8 * got.element_size())) - 1
        assert int(got[0]) & mask == want, (dtype, op, hex(int(got[0]) & mask))
        if op in (CM.SUM, CM.PRODUCT) and dtype == torch.float16:
            assert int(got[1]) & mask == want, (dtype, op, hex(int(got[1]) & mask))


# ---------------------------------------------------------------------------------------------------------- SymmWorld
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_symm_world_reduces_every_dtype_with_ragged_and_unaligned_tensors(C, sms, world):
    """``all_reduce_`` and ``reduce_`` of every new dtype on both sides of the LL / one-shot / two-shot thresholds, ragged
    sizes, and views that start one element into their storage (not 16-byte aligned); a bool SUM is a MAX; roots are global
    ranks of a group whose ranks are not 0..W-1."""
    globals_ = [10 + 3 * r for r in range(world)]
    worlds, keep = E.symm_worlds(world, sms, globals_)
    for k, numel in enumerate([5, 1024, 3001, 12288, 40000, 200003]):
        for d, dtype in enumerate(RM.DTYPES):
            op = OPS[(k + d) % 4]
            xs = RM.make_inputs(op, dtype, world, numel, 100 * world + 10 * k + d)
            want = xs[0] if world == 1 else RM.fold(op, xs)     # a world of 1 launches nothing: t is left as it is
            any_nan = RM.nan_any(op, dtype)
            unaligned = (k + d) % 2 == 1
            bases = [torch.cat([x[:1], x]).cuda() if unaligned else x.cuda() for x in xs]
            ts = [b[1:] if unaligned else b for b in bases]
            E.on_ranks(worlds, lambda r, w: w.all_reduce_(ts[r], op=op))
            RM.assert_bits_equal(f"all_reduce_ {RM.NAMES[dtype]} {CM.OP_NAMES[op]} {numel}", [t.cpu() for t in ts],
                                 [want] * world, any_nan)
            root_local = [0, world - 1, world // 2][(k + d) % 3]
            ts = [x.cuda() for x in xs]
            E.on_ranks(worlds, lambda r, w: w.reduce_(ts[r], globals_[root_local], op))
            for r in range(world):
                if r == root_local:
                    RM.assert_bits_equal(f"reduce_ {RM.NAMES[dtype]} {numel}", [ts[r].cpu()], [want], any_nan)
                else:
                    assert _bits_equal(ts[r], xs[r]), ("reduce_: a non-root changed its tensor", dtype, numel, r)
    with pytest.raises(ValueError, match="fp32 / bf16 SUM only"):
        worlds[0].all_reduce_(torch.zeros(4, dtype=torch.int32, device="cuda"), scale=0.5)
    with pytest.raises(TypeError, match="wire dtype conversion"):
        worlds[0].all_reduce_(torch.zeros(4, dtype=torch.float16, device="cuda"), wire=torch.bfloat16)
    with pytest.raises(TypeError):
        worlds[0].all_reduce_(torch.zeros(4, dtype=torch.int16, device="cuda"))
    del keep


@pytest.mark.parametrize("world", [2, 3, 8])
def test_evaluate_sums_its_float64_totals_on_the_fp64_kernels(C, sms, world, monkeypatch):
    """``evaluate()``'s ``[loss, correct, n]`` float64 sum (``convnet_eval._group_sum``) on a process group whose CUDA backend
    is NCCL and which has a symmetric world (``backend="b200"``): the tensor stays on the device, goes through
    ``SymmWorld.all_reduce_`` over the emulated ranks, never reaches torch.distributed, and every rank gets the rank-order
    fp64 sum."""
    from dist_tuto.pth_b200 import comm
    from dist_tuto.pth_b200.ops import convnet_eval
    worlds, keep = E.symm_worlds(world, sms, list(range(world)))
    current = {}
    monkeypatch.setattr(comm, "is_initialized", lambda: True)
    monkeypatch.setattr(comm, "get_world_size", lambda group=None: world)
    monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: current["w"] if tensor.is_cuda else None)
    monkeypatch.setattr(convnet_eval.dist, "get_backend", lambda group=None: "cpu:gloo,cuda:nccl")

    def refuse(*a, **k):
        raise AssertionError("evaluate()'s sum reached torch.distributed on a symmetric world")
    monkeypatch.setattr(comm.dist, "all_reduce", refuse)
    g = torch.Generator().manual_seed(world)
    totals = [torch.tensor([float(torch.rand(1, generator=g)) * 1000.0, 37.0 + r, 125.0 + r], dtype=torch.float64)
              for r in range(world)]
    want = torch.zeros(3, dtype=torch.float64)
    for t in totals:
        want = want + t
    ts = [t.cuda() for t in totals]
    got = [None] * world

    def one(r, w):
        current["w"] = w
        got[r] = convnet_eval._group_sum(ts[r], None)
    E.on_ranks(worlds, one)
    for r in range(world):
        assert got[r].is_cuda and got[r].data_ptr() == ts[r].data_ptr(), "the sum left the device"
        assert torch.equal(got[r].cpu().view(torch.int64), want.view(torch.int64)), (r, got[r], want)
    del keep
