"""CPU checks of the reductions beyond fp32 / bf16: the model of tests/reduce_dtypes_model.py against torch, planted faults
the checker catches, the launcher's and the binding's refusals, the NVLS fall-back of ``SymmWorld._launch``, and how
``comm`` routes each dtype and op."""
import ctypes
import math

import pytest
import torch

import collectives_model as CM
import comm_model as M
import reduce_dtypes_model as RM

INTS = [torch.int8, torch.uint8, torch.int32, torch.int64]


def _fold_torch(op, xs):
    s = torch.stack(xs)
    if op == CM.SUM:
        return s.sum(0, dtype=torch.int64).to(xs[0].dtype) if xs[0].dtype != torch.int64 else s.sum(0)
    if op == CM.PRODUCT:
        return s.prod(0, dtype=torch.int64).to(xs[0].dtype) if xs[0].dtype != torch.int64 else s.prod(0)
    return s.amax(0) if op == CM.MAX else s.amin(0)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", INTS + [torch.bool], ids=["int8", "uint8", "int32", "int64", "bool"])
def test_integer_and_bool_results_are_torch_with_wrap(dtype, world):
    for op in (CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN):
        xs = RM.make_inputs(op, dtype, world, 4000, 7 * world + op)
        got = RM.fold(op, xs)
        if dtype == torch.bool:
            want = _fold_torch(RM.kernel_op(op, dtype), [x.to(torch.uint8) for x in xs]).bool()
        else:
            want = _fold_torch(op, xs)
        assert got.dtype == dtype and torch.equal(RM.bits(got), RM.bits(want)), (dtype, op)


def test_overflow_wraps_and_signedness_decides_max():
    i8 = [torch.tensor([127, -1], dtype=torch.int8), torch.tensor([1, 1], dtype=torch.int8)]
    assert RM.fold(CM.SUM, i8).tolist() == [-128, 0]
    u8 = [torch.tensor([255, 1], dtype=torch.uint8), torch.tensor([1, 2], dtype=torch.uint8)]
    assert RM.fold(CM.MAX, u8).tolist() == [255, 2]
    assert RM.fold(CM.MAX, [t.view(torch.int8) for t in u8]).tolist() == [1, 2]
    i64 = [torch.tensor([2 ** 63 - 1], dtype=torch.int64), torch.tensor([1], dtype=torch.int64)]
    assert RM.fold(CM.SUM, i64).tolist() == [-2 ** 63]
    b = [torch.tensor([True, False, True]), torch.tensor([True, False, False])]
    assert RM.fold(CM.SUM, b).tolist() == [True, False, True]                   # SUM is MAX
    assert RM.fold(CM.PRODUCT, b).tolist() == [True, False, False]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_fp64_sum_is_the_rank_order_fold_and_fp16_rounds_once(world):
    xs = RM.make_inputs(CM.SUM, torch.float64, world, 5000, world)
    acc = torch.zeros(5000, dtype=torch.float64)
    for x in xs:
        acc = acc + x
    assert torch.equal(RM.fold(CM.SUM, xs).nan_to_num(), acc.nan_to_num())
    hs = RM.make_inputs(CM.SUM, torch.float16, world, 5000, world)
    f = torch.zeros(5000)
    for h in hs:
        f = f + h.float()
    want = torch.where(f.isnan(), torch.tensor(RM.F16_NAN, dtype=torch.int16).view(torch.float16), f.half())
    assert torch.equal(RM.bits(RM.fold(CM.SUM, hs)), RM.bits(want))
    if world >= 3:                               # 1 + (world - 1) 2^-11: exact once, but 1 when rounded per term
        assert float(RM.fold(CM.SUM, hs)[3]) == float(torch.tensor(1 + (world - 1) * 2 ** -11).half()) > 1.0
        assert float(RM.fold(CM.SUM, hs, fault="f16_every_term")[3]) == 1.0


def test_fp16_and_fp64_specials():
    h = [torch.tensor([60000.0, -0.0, math.nan], dtype=torch.float16), torch.tensor([60000.0, 0.0, 1.0], dtype=torch.float16)]
    got = RM.fold(CM.SUM, h)
    assert got[0] == math.inf and RM.bits(got)[2] == RM.F16_NAN
    assert RM.bits(RM.fold(CM.MAX, h))[1] == 0 and RM.bits(RM.fold(CM.MIN, h))[1] == RM.bits(torch.tensor([-0.0], dtype=torch.float16))[0]
    d = [torch.tensor([-0.0, math.nan, math.inf]), torch.tensor([0.0, 1.0, -math.inf])]
    d = [x.double() for x in d]
    mx, mn = RM.fold(CM.MAX, d), RM.fold(CM.MIN, d)
    assert RM.bits(mx)[0] == 0 and RM.bits(mn)[0] == -2 ** 63
    assert RM.bits(mx)[1] == RM.F64_NAN and RM.bits(mn)[1] == RM.F64_NAN
    assert mx[2] == math.inf and mn[2] == -math.inf


# ------------------------------------------------------------------------------------------------------ planted faults
@pytest.mark.parametrize("fault,dtype,op", [("minmax_sign", torch.uint8, CM.MAX), ("minmax_sign", torch.int8, CM.MIN),
                                            ("saturate", torch.int8, CM.SUM), ("f16_every_term", torch.float16, CM.SUM),
                                            ("f64_via_f32", torch.float64, CM.SUM), ("bool_wrap", torch.bool, CM.SUM),
                                            ("lost_nan", torch.float16, CM.MAX), ("lost_nan", torch.float64, CM.MIN)])
def test_the_checker_catches_planted_faults(fault, dtype, op):
    world, n = 4, 2000
    xs = RM.make_inputs(op, dtype, world, n, 3)
    outs = [RM.as_bytes(torch.zeros(n, dtype=dtype)) for _ in range(world)]
    bufs = [RM.as_bytes(torch.zeros(n, dtype=dtype)) for _ in range(world)]
    good = RM.reduce_model(M.ONESHOT, op, xs, "staged", -1, outs, bufs)
    bad = RM.reduce_model(M.ONESHOT, op, xs, "staged", -1, outs, bufs, fault=fault)
    assert RM.first_mismatch(good["out"], good["out"]) is None
    with pytest.raises(AssertionError):
        RM.assert_bits_equal(fault, bad["out"], good["out"], RM.nan_any(op, dtype))


def test_reduce_model_leaves_non_roots_and_keeps_staging():
    world, n = 3, 16
    xs = RM.make_inputs(CM.SUM, torch.int32, world, n, 1)
    before = [torch.full((n + 4,), 7, dtype=torch.int32) for _ in range(world)]
    got = RM.reduce_model(M.TWOSHOT, CM.SUM, xs, "staged", 1, before, before)
    for r in range(world):
        assert torch.equal(got["out"][r][n:], before[r][n:])
        if r != 1:
            assert torch.equal(got["out"][r], before[r]) and torch.equal(got["buf"][r][:n], xs[r])
    assert torch.equal(got["out"][1][:n], got["result"]) and torch.equal(got["buf"][1][:n], got["result"])


# ---------------------------------------------------------------------------------------------------------- refusals
def _C():
    from dist_tuto.pth_b200.ops import _ext
    return _ext.C()


def _ptrs(world, base):
    return [base + 0x100000 * r for r in range(world)]


def _dtype_launcher():
    from dist_tuto.pth_b200.ops import _ext
    _C()
    fn = ctypes.CDLL(_ext.so_path()).b2_allreduce_dtype_launch
    fn.restype = ctypes.c_int
    i, p, z = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
    fn.argtypes = [i, i, p, p, p, p, i, p, i, z, ctypes.c_float, i, i, i, p, z, i, i, p]
    return fn


def test_launcher_refuses_bad_dtype_calls_without_a_launch():
    """b2_allreduce_dtype_launch returns cudaErrorInvalidValue (1) before any CUDA call for each of these (without a GPU, a
    launch would return another error)."""
    fn = _dtype_launcher()
    bufs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x1000))
    sigs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x2000))

    def call(variant, dtype, op=0, scale=1.0, src_f32=0, dst_f32=0, root=-1):
        return fn(variant, dtype, bufs, sigs, ctypes.c_void_p(0x900000), None, src_f32, None, dst_f32, 64, scale, 0, 4, 0,
                  None, 0, op, root, None)
    for dtype in (-1, 9, 100):
        assert call(0, dtype) == 1                                          # unknown dtype
    for dtype in range(2, 8):                                               # SUM: the only op the fp32 / bf16 rules allow
        assert call(0, dtype, op=0, scale=0.5) == 1                         # a scale
        assert call(0, dtype, op=0, src_f32=1) == 1                         # fp32 locals
        assert call(0, dtype, op=0, dst_f32=1) == 1
        assert call(2, dtype, op=0) == 1                                    # NVLS
    assert call(0, 8, op=0) == 1                                            # bool SUM (the caller maps it to MAX)
    for op in (4, 5, 6):
        assert call(0, 3, op=op, root=0) == 1                               # a dtype for the raw moves
    assert call(0, 3, op=7) == 1                                            # the existing refusals stay: unknown op


def test_binding_refuses_bad_dtype_calls():
    C = _C()
    b, s = _ptrs(4, 0x1000), _ptrs(4, 0x2000)

    def f(dtype, bf16=False, scale=1.0, variant=0, op=2, src=None):
        C.allreduce(variant, bf16, b, s, 0, src, None, 64, scale, 0, 4, 0, [], 0, op, -1, dtype=dtype)
    with pytest.raises(RuntimeError, match="dtype must be"):
        f(9)
    with pytest.raises(RuntimeError, match="contradicts the bf16 flag"):
        f(0, bf16=True)
    with pytest.raises(RuntimeError, match="bf16 wire is for fp32 / bf16"):
        f(3, bf16=True)
    with pytest.raises(RuntimeError, match="scale applies to fp32 / bf16 SUM only"):
        f(6, scale=0.5, op=0)
    with pytest.raises(RuntimeError, match="NVLS reduces fp32 / bf16 only"):
        f(7, variant=2, op=0)
    with pytest.raises(RuntimeError, match="bool SUM is a MAX"):
        f(8, op=0)
    with pytest.raises(RuntimeError, match="src is"):
        f(6, src=torch.zeros(256, dtype=torch.int64))


# ---------------------------------------------------------------------------------------------------------- variants
class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda variant, *a, **k: self.calls.append((name, variant, a, k))


def _planning_world(world, staging=True):
    from dist_tuto.pth_b200.parallel import symm
    w = object.__new__(symm.SymmWorld)
    w.C, w.world, w.rank, w.ranks = _Recorder(), world, 0, list(range(world))
    w.global_rank, w.device = 0, torch.device("cpu")
    w.multicast, w.max_blocks = True, 132
    w.ll_max, w.oneshot_max, w.nvls_min = 32 << 10, 128 << 10, 1
    hd = symm.SymmHandle(w, 1 << 30, 1 << 30, [0x10000 * (r + 1) for r in range(world)], 0x900000, [], 0, "vmm")
    hd.ll = symm.SymmHandle(w, 0, 0, [0x20000 * (r + 1) for r in range(world)], 0, [], 0, "vmm")
    return w, hd


def test_launch_falls_back_from_nvls_for_the_new_dtypes(monkeypatch):
    from dist_tuto.pth_b200.parallel import symm
    monkeypatch.delenv("B200DIST_AR_VARIANT", raising=False)
    w, hd = _planning_world(8)
    big = (1 << 20) // 16
    assert w._launch(hd, False, big, 1.0, None, None, None) == 2                        # fp32 SUM: NVLS
    for code in range(2, 9):
        op = 2 if code == 8 else 0
        assert w._launch(hd, False, big, 1.0, None, None, None, None, "allreduce", op, -1, dtype=code) == 1
        assert w.C.calls[-1][3] == {"dtype": code}
        assert w._launch(hd, False, 64, 1.0, None, None, None, None, "allreduce", op, -1, dtype=code) == 3
    monkeypatch.setenv("B200DIST_AR_VARIANT", "nvls")
    assert w._launch(hd, False, big, 1.0, None, None, None, None, "allreduce", 0, -1, dtype=3) == 1
    assert w._launch(hd, False, big, 1.0, None, None, None) == 2
    assert "dtype" not in w.C.calls[-1][3]                                   # fp32 / bf16 calls are as before
    assert symm.DTYPE_CODES[torch.bool] == RM.CODES[torch.bool] and symm.DTYPE_CODES == RM.CODES


def test_symm_reduce_refuses_bad_combinations_at_every_world_size(monkeypatch):
    """A scale or a wire conversion with a new dtype, and a dtype outside the table, raise before any launch -- at world 1
    too, where nothing would be launched anyway."""
    for world in (1, 4):
        w, hd = _planning_world(world)
        monkeypatch.setattr(type(w), "supports_reduction", lambda self, t: t.dtype in RM.CODES)
        monkeypatch.setattr(type(w), "supports", lambda self, t: t.dtype in (torch.float32, torch.bfloat16))
        with pytest.raises(ValueError, match="fp32 / bf16 SUM only"):
            w.all_reduce_(torch.zeros(4, dtype=torch.int64), scale=0.25)
        with pytest.raises(ValueError, match="scale applies to SUM only"):
            w.all_reduce_(torch.zeros(4, dtype=torch.int64), scale=0.25, op=CM.MAX)
        with pytest.raises(TypeError, match="wire dtype conversion"):
            w.all_reduce_(torch.zeros(4, dtype=torch.float16), wire=torch.bfloat16)
        with pytest.raises(TypeError, match="int16"):
            w.all_reduce_(torch.zeros(4, dtype=torch.int16))
        assert w.C.calls == []


def test_bool_sum_runs_as_max_through_symm(monkeypatch):
    from dist_tuto.pth_b200.parallel import symm
    w, hd = _planning_world(4)
    monkeypatch.setattr(type(w), "supports_reduction", lambda self, t: t.dtype in RM.CODES)
    monkeypatch.setattr(type(w), "supports", lambda self, t: t.dtype in (torch.float32, torch.bfloat16))
    got = []
    monkeypatch.setattr(type(w), "_launch", lambda self, hd, bf16, n_vec, scale, src, dst, variant, mb, kind, op, root, dtype=None:
                        got.append((kind, op, root, dtype)))
    monkeypatch.setattr(type(w), "_staging_for", lambda self, dt, nbytes: hd)
    t = torch.zeros(64, dtype=torch.bool)
    w.all_reduce_(t)
    w.reduce_(torch.zeros(64, dtype=torch.int8), 2, CM.SUM)
    assert got == [("allreduce", CM.MAX, -1, 8), ("reduce", CM.SUM, 2, 4)]
    assert symm.op_code(torch.distributed.ReduceOp.AVG) is None


# ---------------------------------------------------------------------------------------------------------- routing
class _StandInWorld:
    """A symmetric world as comm.py sees it: CUDA-only checks replaced by dtype checks, records which method it ran."""

    def __init__(self, with_reduction=True):
        self.calls = []
        if with_reduction:
            self.supports_reduction = lambda t: t.dtype in RM.CODES

    def supports(self, t):
        return t.dtype in (torch.float32, torch.bfloat16)

    def supports_op(self, op):
        from dist_tuto.pth_b200.parallel.symm import op_code
        return op_code(op) is not None

    def all_reduce_(self, t, scale=1.0, op=None):
        self.calls.append(("all_reduce_", t.dtype))

    def reduce_(self, t, root, op):
        self.calls.append(("reduce_", t.dtype, root))


def _route(monkeypatch, w, call):
    from dist_tuto.pth_b200 import comm
    nccl = []
    monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: w)
    monkeypatch.setattr(comm.dist, "all_reduce", lambda t, **k: nccl.append(("nccl_all_reduce", t.dtype)))
    monkeypatch.setattr(comm.dist, "reduce", lambda t, **k: nccl.append(("nccl_reduce", t.dtype)))
    call(comm)
    return w.calls + nccl


@pytest.mark.parametrize("dtype", RM.DTYPES, ids=[RM.NAMES[d] for d in RM.DTYPES])
def test_comm_routes_new_dtypes_to_the_kernels(monkeypatch, dtype):
    from dist_tuto.pth_b200 import comm
    for rank_root in (0, 3):
        for op in (comm.reduce_op.SUM, comm.reduce_op.PRODUCT, comm.reduce_op.MAX, comm.reduce_op.MIN):
            t = torch.zeros(8, dtype=dtype)
            assert _route(monkeypatch, _StandInWorld(), lambda c: c.all_reduce(t, op=op)) == [("all_reduce_", dtype)]
            assert _route(monkeypatch, _StandInWorld(), lambda c: c.reduce(t, rank_root, op=op)) == \
                [("reduce_", dtype, rank_root)]
            # the two-level world (no supports_reduction) keeps them on torch
            assert _route(monkeypatch, _StandInWorld(False), lambda c: c.all_reduce(t, op=op)) == [("nccl_all_reduce", dtype)]
            assert _route(monkeypatch, _StandInWorld(False), lambda c: c.reduce(t, rank_root, op=op)) == \
                [("nccl_reduce", dtype)]


def test_comm_keeps_int16_complex_and_avg_on_torch(monkeypatch):
    from dist_tuto.pth_b200 import comm
    for t in (torch.zeros(8, dtype=torch.int16), torch.zeros(8, dtype=torch.complex64), torch.zeros(8, dtype=torch.uint16)):
        assert _route(monkeypatch, _StandInWorld(), lambda c: c.all_reduce(t)) == [("nccl_all_reduce", t.dtype)]
    for dt in (torch.float64, torch.int32):
        t = torch.zeros(8, dtype=dt)
        assert _route(monkeypatch, _StandInWorld(), lambda c: c.all_reduce(t, op=torch.distributed.ReduceOp.AVG)) == \
            [("nccl_all_reduce", dt)]
        assert _route(monkeypatch, _StandInWorld(), lambda c: c.all_reduce(t, async_op=True)) == [("nccl_all_reduce", dt)]


def test_average_gradients_of_fp16_keeps_the_torch_path(monkeypatch):
    """``supports`` still means fp32 / bf16: average_gradients of fp16 gradients takes torch's all-reduce and ``div_`` even
    on a world that reduces fp16, while fp32 gradients take the fused kernel with the 1 / world scale."""
    from dist_tuto.pth_b200 import comm
    from dist_tuto.pth_b200.parallel import ddp
    w = _StandInWorld()
    fused = []
    w.all_reduce_ = lambda t, scale=1.0, op=None: fused.append((t.dtype, scale))
    torched = []

    def torch_all_reduce(t, op=None, group=None):
        torched.append(t.dtype)
        t.mul_(2)                                            # two ranks with the same gradients
    monkeypatch.setattr(comm, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(ddp, "_symm_world", lambda group, dev: w)
    monkeypatch.setattr(ddp.dist, "all_reduce", torch_all_reduce)
    for dtype in (torch.float16, torch.float32):
        model = torch.nn.Linear(3, 2).to(dtype)
        for p in model.parameters():
            p.grad = torch.full_like(p, 0.75)
        ddp.average_gradients(model)
        if dtype == torch.float16:
            assert torched == [torch.float16] and fused == []
            assert all(bool((p.grad == 0.75).all()) for p in model.parameters())   # summed by torch, then div_
        else:
            assert torched == [torch.float16] and fused == [(torch.float32, 0.5)]
