"""CPU checks of tests/collectives_model.py (against fp64 and torch, and that its checker catches planted faults), of the
variant plan of parallel/symm.py, of the bindings' refusals for the new collectives, and of docs/api.md."""
import os

import pytest
import torch

import collectives_model as CM
import comm_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, B16 = torch.float32, torch.bfloat16


def _stack(xs):
    return torch.stack([x.float() for x in xs])


# ---------------------------------------------------------------------------------------------------------- the model
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", [F32, B16])
def test_max_and_min_folds_match_torch_and_ieee_754_2019(world, dtype):
    xs = CM.make_reduce_inputs(CM.MAX, world, 4096, dtype, seed=world)
    s = _stack(xs)
    for op, ref in ((CM.MAX, s.amax(0)), (CM.MIN, s.amin(0))):
        got = CM.fold(op, [x.float() for x in xs])
        nan = torch.isnan(s).any(0)
        assert torch.equal(torch.isnan(got), nan)                       # any NaN term gives NaN
        assert bool((got[~nan] == ref[~nan]).all())
        zero = (got == 0) & ~nan
        neg = s.signbit() & (s == 0)
        pos = ~s.signbit() & (s == 0)
        if op == CM.MAX:                                                # -0 < +0: -0 only if no term is >= +0
            want_neg = ~(pos | (s > 0)).any(0)
        else:
            want_neg = (neg | (s < 0)).any(0)
        assert torch.equal(got.signbit()[zero], want_neg[zero])


@pytest.mark.parametrize("world", [1, 2, 5, 8])
def test_product_fold_is_within_the_fp64_bound(world):
    xs = CM.make_reduce_inputs(CM.PRODUCT, world, 8192, F32, seed=world)
    got = CM.fold(CM.PRODUCT, xs).double()
    ref = torch.ones(8192, dtype=torch.float64)
    for x in xs:
        ref = ref * x.double()
    fin = torch.isfinite(ref)
    assert bool(((got[fin] - ref[fin]).abs() <= ref[fin].abs() * world * 2.0 ** -24 * 1.01).all())
    assert torch.equal(got[~fin].nan_to_num(), ref[~fin].nan_to_num())
    small = ref[fin & (ref != 0)].abs().min()
    assert small > 2.0 ** -120                                         # far from the subnormal range the kernels flush


def test_sum_fold_is_comm_models_sum():
    xs = M.make_inputs(4, 1024, F32, seed=3)
    assert torch.equal(CM.fold(CM.SUM, xs, 0.25), M.reduce_scaled(xs, 0.25))


@pytest.mark.parametrize("variant", [M.ONESHOT, M.TWOSHOT, M.LL])
@pytest.mark.parametrize("mode", ["inplace", "staged", "alias"])
def test_reduce_model_leaves_non_roots_alone(variant, mode):
    world, n, root = 4, 256, 2
    xs = CM.make_reduce_inputs(CM.MAX, world, n, F32, seed=1)
    outs = [torch.full((n + 8,), 7.0) for _ in range(world)] if mode == "staged" else \
        [torch.cat([x, torch.full((8,), 7.0)]) for x in xs]
    bufs = [torch.cat([x, torch.full((8,), 7.0)]) for x in xs] if mode == "inplace" else \
        [torch.full((n + 8,), 7.0) for _ in range(world)]
    if mode == "inplace":
        outs = bufs
    want = CM.reduce_model(variant, CM.MAX, xs, F32, 1.0, mode, root, outs, bufs)
    full = CM.reduce_model(variant, CM.MAX, xs, F32, 1.0, mode, -1, outs, bufs)
    for r in range(world):
        if r == root:
            assert M.first_mismatch([want["out"][r]], [full["out"][r]], 4) is None
        else:
            assert torch.equal(want["out"][r].view(torch.int32), outs[r].view(torch.int32))
        assert torch.equal(want["out"][r][n:], outs[r][n:])            # sentinels


def test_raw_models_move_every_bit():
    world, n = 3, 64
    xs = CM.make_raw_inputs(world, n, seed=4)
    outs = [torch.zeros(n, dtype=torch.int32) for _ in range(world)]
    bufs = [torch.zeros(world * n, dtype=torch.int32) for _ in range(world)]
    for variant in (M.ONESHOT, M.TWOSHOT, M.LL):
        b = CM.broadcast_model(variant, xs, 1, "staged", outs, bufs[:1] * world)
        assert all(torch.equal(o, xs[1]) for o in b["out"])
        g = CM.allgather_model(variant, xs, "staged", [torch.zeros(world * n, dtype=torch.int32)] * world, bufs)
        assert all(torch.equal(o, torch.cat(xs)) for o in g["out"])
    specials = set(int(v) & 0xFFFFFFFF for x in xs for v in x.tolist())
    assert {0x80000000, 0x7FC01234, 0x00000001} <= specials            # -0, a NaN payload and a subnormal are moved


# ---------------------------------------------------------------------------------------------------------- planted faults
def test_a_max_that_drops_nan_is_caught():
    xs = CM.make_reduce_inputs(CM.MAX, 4, 2048, F32, seed=7)
    want = CM.fold(CM.MAX, xs)
    dropped = xs[0].clone()
    for x in xs[1:]:
        dropped = torch.fmax(dropped, x)                                # fmaxf: a NaN term is ignored
    nan = torch.isnan(want)
    assert bool(nan.any()) and M.first_mismatch([dropped[nan]], [want[nan]], 4) is not None


def test_a_broadcast_through_a_float_add_is_caught():
    xs = CM.make_raw_inputs(2, 1024, seed=8)
    want = CM.broadcast_model(M.ONESHOT, xs, 0, "staged", [torch.zeros(1024, dtype=torch.int32)] * 2,
                              [torch.zeros(1024, dtype=torch.int32)] * 2)["out"]
    through_add = (torch.zeros(1024) + xs[0].view(F32)).view(torch.int32)   # 0 + -0 = +0; NaN payloads may change
    m = M.first_mismatch([through_add, through_add], want, 4)
    assert m is not None and m[4] == 0x80000000 and m[3] == 0


def test_a_non_root_that_writes_its_output_is_caught():
    world, n, root = 3, 512, 0
    xs = CM.make_reduce_inputs(CM.MIN, world, n, F32, seed=9)
    outs = [torch.full((n,), 7.0) for _ in range(world)]
    want = CM.reduce_model(M.ONESHOT, CM.MIN, xs, F32, 1.0, "staged", root, outs, [torch.zeros(n)] * world)["out"]
    leaky = CM.reduce_model(M.ONESHOT, CM.MIN, xs, F32, 1.0, "staged", -1, outs, [torch.zeros(n)] * world)["out"]
    m = M.first_mismatch(leaky, want, 4)
    assert m is not None and m[0] == 1 and m[1] == 0


# ---------------------------------------------------------------------------------------------------------- variant plan
def test_plan_variant_picks_by_size_and_keeps_nvls_for_the_sum_all_reduce():
    from dist_tuto.pth_b200.parallel.symm import plan_variant
    th = dict(ll_max=32 << 10, oneshot_max=64 << 10, nvls_min=128 << 10)

    def plan(c, op, nbytes, world=4, mc=True, forced=None):
        return plan_variant(c, op, nbytes, world, th["ll_max"], th["oneshot_max"], th["nvls_min"], mc, forced)
    for c in ("allreduce", "reduce", "broadcast"):
        assert [plan(c, 0, b) for b in (16, 32 << 10, (32 << 10) + 16, 64 << 10, 100 << 10)] == [3, 3, 0, 0, 1]
        assert plan(c, 0, 128 << 10) == (2 if c == "allreduce" else 1)
    for op in (1, 2, 3):
        assert plan("allreduce", op, 1 << 20) == 1
        assert plan("allreduce", op, 1 << 20, forced="nvls") == 1      # NVLS cannot MAX / MIN / multiply f32 in the switch
    assert plan("allreduce", 0, 1 << 20, forced="nvls") == 2
    assert plan("allreduce", 0, 1 << 20, mc=False, forced="nvls") == 1
    assert plan("allreduce", 0, 16, forced="twoshot") == 1
    # all-gather: LL by one rank's input, one-shot by the whole output
    assert plan("allgather", 0, 32 << 10) == 3
    assert plan("allgather", 0, 32 << 10, world=2) == 3
    assert plan_variant("allgather", 0, (32 << 10) + 16, 2, 32 << 10, 128 << 10, 1 << 62, True) == 0
    assert plan_variant("allgather", 0, (32 << 10) + 16, 4, 32 << 10, 128 << 10, 1 << 62, True) == 1
    assert plan("allgather", 0, 1 << 30, world=1) == 0
    with pytest.raises(ValueError):
        plan("scatter", 0, 16)


def test_op_code_maps_reduce_ops():
    import torch.distributed as dist
    from dist_tuto.pth_b200.parallel.symm import op_code
    assert [op_code(o) for o in (dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT, dist.ReduceOp.MAX, dist.ReduceOp.MIN)] == [0, 1, 2, 3]
    assert op_code(dist.ReduceOp.AVG) is None and op_code(4) is None and op_code(True) is None


# ---------------------------------------------------------------------------------------------------------- bindings
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def _ptrs(world, base):
    return [base * (i + 1) for i in range(world)]


def test_allreduce_binding_refuses_bad_ops_roots_scales_and_wires():
    C = _C()
    b, s = _ptrs(2, 0x1000), _ptrs(2, 0x2000)
    with pytest.raises(RuntimeError, match="op must be 0"):
        C.allreduce(0, False, b, s, 0, None, None, 64, 1.0, 0, 2, 1, [], 0, 4, -1)
    with pytest.raises(RuntimeError, match="root must be -1"):
        C.allreduce(0, False, b, s, 0, None, None, 64, 1.0, 0, 2, 1, [], 0, 2, 2)
    with pytest.raises(RuntimeError, match="scale applies to SUM only"):
        C.allreduce(0, False, b, s, 0, None, None, 64, 0.5, 0, 2, 1, [], 0, 2, -1)
    with pytest.raises(RuntimeError, match="NVLS runs the SUM all-reduce only"):
        C.allreduce(2, False, b, s, 0x4000, None, None, 64, 1.0, 0, 2, 1, [], 0, 3, -1)
    with pytest.raises(RuntimeError, match="NVLS runs the SUM all-reduce only"):
        C.allreduce(2, False, b, s, 0x4000, None, None, 64, 1.0, 0, 2, 1, [], 0, 0, 1)


def test_raw_move_bindings_refuse_bad_roots_and_ll_overflow():
    C = _C()
    b, s, ib = _ptrs(4, 0x1000), _ptrs(4, 0x2000), _ptrs(4, 0x3000)
    with pytest.raises(RuntimeError, match="broadcast: root must be in"):
        C.broadcast(0, b, s, None, None, 64, -1, 0, 4)
    with pytest.raises(RuntimeError, match="root must be -1"):
        C.broadcast(0, b, s, None, None, 64, 4, 0, 4)
    with pytest.raises(RuntimeError, match="more than the inbox holds"):
        C.allgather(3, b, s, None, None, 4 * (M.LL_CAP_VEC + 1), 0, 4, 0, ib, M.LL_CAP_VEC)
    with pytest.raises(RuntimeError, match="more than the inbox holds"):
        C.broadcast(3, b, s, None, None, M.LL_CAP_VEC + 1, 0, 0, 4, 0, ib, M.LL_CAP_VEC)
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.allgather(0, b, s, None, None, 4 * 100 + 1, 0, 4)


def test_fp32_over_a_bf16_wire_is_for_sum_only():
    C = _C()
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA tensor to pass the dtype")
    t = torch.zeros(64, device="cuda")
    with pytest.raises(RuntimeError, match="bf16 wire for fp32 tensors is for SUM only"):
        C.allreduce(0, True, [0x1000], [0x2000], 0, t, t, 8, 1.0, 0, 1, 1, [], 0, 2, -1)


# ---------------------------------------------------------------------------------------------------------- docs
def test_api_reference_lists_the_new_collectives():
    text = open(os.path.join(ROOT, "docs", "api.md")).read()
    for name in ("reduce_", "broadcast_", "all_gather_", "plan_variant", "op_code", "supports_op", "supports_raw"):
        assert f"`{name}" in text, name
