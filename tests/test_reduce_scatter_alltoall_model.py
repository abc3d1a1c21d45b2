"""CPU checks of the reduce-scatter and all-to-all: the model (tests/reduce_scatter_alltoall_model.py) against torch folds and
against the all-reduce model, the planted faults its checker must catch, the bindings' and the launchers' refusals (no
launch), the variant plan, the routing of comm.py, and the four calls on gloo at world 2 and 3 through ``b2.launch``."""
import ctypes
import functools
import os

import pytest
import torch

import collectives_model as CM
import comm_model as M
import reduce_dtypes_model as RM
import reduce_scatter_alltoall_model as RS

OPS = [CM.SUM, CM.PRODUCT, CM.MAX, CM.MIN]
VARIANTS = [M.ONESHOT, M.LL]


def _torch_fold(op, terms):
    """The reduction by torch ops, identity first, in rank order (integers wrap in their dtype, bool SUM is MAX)."""
    dtype = terms[0].dtype
    if dtype == torch.bool:
        op = CM.MAX if op == CM.SUM else op
        terms = [t.view(torch.uint8) for t in terms]
    if op in (CM.MAX, CM.MIN):
        f = torch.maximum if op == CM.MAX else torch.minimum
        out = functools.reduce(f, terms)
    else:
        ident = torch.zeros_like(terms[0]) if op == CM.SUM else torch.ones_like(terms[0])
        out = functools.reduce(torch.add if op == CM.SUM else torch.mul, terms, ident)
    return out.view(torch.bool) if dtype == torch.bool else out


@pytest.mark.parametrize("dtype", [torch.float64, torch.int8, torch.uint8, torch.int32, torch.int64, torch.bool],
                         ids=lambda d: RS.NAMES[d])
@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_reduce_scatter_model_agrees_with_torch_folds(dtype, world):
    """The model's segment r is torch's fold of segment r: bit for bit for the integers and bool, by value for fp64 without
    NaNs (torch pins neither NaN payloads nor the sign of max(-0, +0))."""
    for op in OPS:
        xs = RS.make_inputs(op, dtype, world, world * 40, 7 * world + op)
        if dtype.is_floating_point:
            xs = [torch.nan_to_num(x, nan=1.0) for x in xs]
        for r in range(world):
            want = _torch_fold(op, [RS.segment(x, r, world) for x in xs])
            got = RS.reduce_scatter_result(op, xs, r)
            if dtype.is_floating_point:
                assert torch.equal(got, want), (dtype, op, r)
            else:
                assert torch.equal(RM.bits(RM.as_bytes(got)), RM.bits(RM.as_bytes(want))), (dtype, op, r)


@pytest.mark.parametrize("dtype", RS.DTYPES, ids=lambda d: RS.NAMES[d])
def test_reduce_scatter_model_is_slice_r_of_the_all_reduce_model(dtype):
    for world in (1, 2, 3, 8):
        for op in OPS:
            n = world * 64
            xs = RS.make_inputs(op, dtype, world, n, 3 * world + op)
            before = [torch.zeros(n, dtype=RM.as_bytes(xs[0]).dtype) for _ in range(world)]
            if dtype in (torch.float32, torch.bfloat16):
                ar = CM.reduce_model(M.ONESHOT, op, xs, dtype, 1.0, "staged", -1, before, before)["out"]
            else:
                ar = RM.reduce_model(M.ONESHOT, op, xs, "staged", -1, before, before)["out"]
            got = RS.reduce_scatter_model(M.ONESHOT, op, xs, "staged", before, before)["result"]
            for r in range(world):
                RM.assert_bits_equal(f"{RS.NAMES[dtype]} op {op} rank {r}", [got[r]], [RS.segment(ar[r], r, world)],
                                     RM.nan_any(op, dtype))


def test_alltoall_model_is_a_transpose_of_segments():
    for world in (1, 2, 3, 8):
        xs = CM.make_raw_inputs(world, world * 12, world)
        for variant in VARIANTS:
            before = [torch.full((world * 12 + 4,), 5, dtype=torch.int32) for _ in range(world)]
            got = RS.alltoall_model(variant, xs, "staged", before, before)
            for r in range(world):
                want = torch.cat([x.view(world, 12)[r] for x in xs])
                assert torch.equal(got["out"][r][:world * 12], want) and torch.equal(got["out"][r][world * 12:], before[r][world * 12:])
            if variant == M.LL:                                          # LL leaves the buffers alone
                assert all(torch.equal(a, b) for a, b in zip(got["buf"], before))
                if world > 1:
                    assert torch.equal(got["lines"][0][world - 1], xs[0].view(world, 12)[world - 1])


def test_the_in_place_model_leaves_the_other_segments_alone():
    world, n = 4, 4 * 8
    xs = RS.make_inputs(CM.SUM, torch.int32, world, n, 1)
    before = [torch.cat([x, torch.full((4,), 7, dtype=torch.int32)]) for x in xs]
    got = RS.reduce_scatter_model(M.LL, CM.SUM, xs, "inplace", before, before)
    for r in range(world):
        for s in range(world):
            want = got["result"][r] if s == r else RS.segment(xs[r], s, world)
            assert torch.equal(got["buf"][r][s * 8:(s + 1) * 8], want)
        assert torch.equal(got["buf"][r][n:], before[r][n:])


# ---------------------------------------------------------------------------------------------------------- planted faults
def _caught(want, wrong, any_nan=False):
    return RM.first_mismatch(wrong, want, any_nan) is not None


@pytest.mark.parametrize("fault", ["swap", "next_slice"])
def test_a_reduce_scatter_that_delivers_another_segment_is_caught(fault):
    world, n = 4, 4 * 16
    xs = RS.make_inputs(CM.SUM, torch.int32, world, n, 2)
    before = [torch.zeros(n, dtype=torch.int32) for _ in range(world)]
    want = RS.reduce_scatter_model(M.ONESHOT, CM.SUM, xs, "staged", before, before)["out"]
    wrong = RS.reduce_scatter_model(M.ONESHOT, CM.SUM, xs, "staged", before, before, fault=fault)["out"]
    assert all(_caught([want[r]], [wrong[r]]) for r in range(world))


def test_a_reduce_scatter_that_combines_in_another_rank_order_is_caught_in_fp32_bits():
    world, n = 4, 4 * 256
    xs = RS.make_inputs(CM.SUM, torch.float32, world, n, 3)
    before = [torch.zeros(n, dtype=torch.float32) for _ in range(world)]
    want = RS.reduce_scatter_model(M.LL, CM.SUM, xs, "staged", before, before)["out"]
    wrong = RS.reduce_scatter_model(M.LL, CM.SUM, xs, "staged", before, before, fault="order")["out"]
    assert _caught(want, wrong)


def test_a_missing_bool_sum_to_max_mapping_is_caught():
    world, n = 3, 3 * 64
    xs = RS.make_inputs(CM.SUM, torch.bool, world, n, 4)
    before = [torch.zeros(n, dtype=torch.uint8) for _ in range(world)]
    want = RS.reduce_scatter_model(M.ONESHOT, CM.SUM, xs, "staged", before, before)["out"]
    wrong = RS.reduce_scatter_model(M.ONESHOT, CM.SUM, xs, "staged", before, before, fault="bool_wrap")["out"]
    assert _caught(want, wrong)


def test_an_ll_alltoall_that_keeps_the_line_of_the_wrong_source_is_caught():
    world, seg = 4, 8
    xs = CM.make_raw_inputs(world, world * seg, 5)
    before = [torch.zeros(world * seg, dtype=torch.int32) for _ in range(world)]
    want = RS.alltoall_model(M.LL, xs, "staged", before, before)["out"]
    wrong = RS.alltoall_model(M.LL, xs, "staged", before, before, keep=lambda r, p: (p + 1) % world if p != r else p)["out"]
    m = M.first_mismatch(wrong, want, 4)
    assert m is not None and m[0] == 0
    assert all(M.first_mismatch([wrong[r]], [want[r]], 4) is not None for r in range(world))


@pytest.mark.parametrize("dtype", [torch.int32, torch.float16, torch.uint8], ids=["int32", "fp16", "uint8"])
def test_a_dropped_last_segment_at_a_ragged_size_is_caught(dtype):
    """Ragged segments (not a multiple of 16 bytes) go through 16-byte slots of the staging buffer; a staging loop that
    leaves out the last segment gives the last rank a reduction of stale bytes."""
    world, seg = 3, 5
    xs = RS.make_inputs(CM.MAX, dtype, world, world * seg, 6)
    stale = [torch.full((1024,), 0x41, dtype=torch.uint8) for _ in range(world)]
    want = [RS.fold(CM.MAX, [RS.segment(x, r, world) for x in xs]) for r in range(world)]
    good = RS.ragged_reduce_scatter(CM.MAX, xs, dtype, stale)
    RM.assert_bits_equal("ragged", good, want)
    bad = RS.ragged_reduce_scatter(CM.MAX, xs, dtype, stale, fault="drop_last")
    m = RM.first_mismatch(bad, want)
    assert m is not None and m[0] == world - 1


# ---------------------------------------------------------------------------------------------------------- refusals
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def _ptrs(world, base):
    return [base * (i + 1) for i in range(world)]


def test_bindings_refuse_bad_variants_ops_dtypes_sizes_and_ll_overflow():
    C = _C()
    b, s, ib = _ptrs(4, 0x1000), _ptrs(4, 0x2000), _ptrs(4, 0x3000)
    rs = lambda variant=0, n_vec=64, op=0, dtype=0, inbox=(), cap=0, src=None: C.reduce_scatter(  # noqa: E731
        variant, b, s, src, None, n_vec, 0, 4, 0, list(inbox), cap, op, dtype)
    with pytest.raises(RuntimeError, match="variant must be 0 .pull. or 3 .LL."):
        rs(variant=1)
    with pytest.raises(RuntimeError, match="op must be"):
        rs(op=4)
    with pytest.raises(RuntimeError, match="dtype must be"):
        rs(dtype=9)
    with pytest.raises(RuntimeError, match="bool SUM is a MAX"):
        rs(dtype=8, op=0)
    with pytest.raises(RuntimeError, match="multiple of world"):
        rs(n_vec=65)
    with pytest.raises(RuntimeError, match="more than the inbox holds"):
        rs(variant=3, n_vec=4 * (M.LL_CAP_VEC + 1), inbox=ib, cap=M.LL_CAP_VEC)
    with pytest.raises(RuntimeError, match="src is"):
        rs(dtype=6, src=torch.zeros(256, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="variant must be 0 .pull. or 3 .LL."):
        C.alltoall(2, b, s, None, torch.zeros(1), 64, 0, 4)
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.alltoall(0, b, s, None, torch.zeros(1), 66, 0, 4)


def _segment_launchers():
    from dist_tuto.pth_b200.ops import _ext
    _C()
    lib = ctypes.CDLL(_ext.so_path())
    i, p, z = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
    rs, a2a = lib.b2_reduce_scatter_launch, lib.b2_alltoall_launch
    rs.restype = a2a.restype = ctypes.c_int
    rs.argtypes = [i, i, i, p, p, p, p, z, i, i, i, p, z, p]
    a2a.argtypes = [i, p, p, p, p, z, i, i, i, p, z, p]
    return rs, a2a


def test_launchers_refuse_bad_calls_without_a_launch():
    """b2_reduce_scatter_launch and b2_alltoall_launch return cudaErrorInvalidValue (1) before any CUDA call for each of
    these (without a GPU, a launch would return another error)."""
    rs, a2a = _segment_launchers()
    bufs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x1000))
    sigs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x2000))
    inbox = (ctypes.c_void_p * 8)(*_ptrs(4, 0x3000))
    dst = ctypes.c_void_p(0x800000)

    def r(variant=0, dtype=0, op=0, n_vec=64, rank=0, world=4, ll_cap=0):
        return rs(variant, dtype, op, bufs, sigs, None, dst, n_vec, rank, world, 0, inbox if variant == 3 else None,
                  ll_cap, None)

    def t(variant=0, n_vec=64, rank=0, world=4, ll_cap=0, out=dst):
        return a2a(variant, bufs, sigs, None, out, n_vec, rank, world, 0, inbox if variant == 3 else None, ll_cap, None)
    for variant in (-1, 1, 2, 4):
        assert r(variant=variant) == 1 and t(variant=variant) == 1       # pull and LL only
    for op in (-1, 4, 7):
        assert r(op=op) == 1                                             # unknown op
    for dtype in (-1, 9):
        assert r(dtype=dtype) == 1                                       # unknown dtype
    assert r(dtype=8, op=0) == 1                                         # bool SUM (the caller maps it to MAX)
    assert r(n_vec=65) == 1 and t(n_vec=65) == 1                         # not world segments
    assert r(world=9) == 1 and t(world=0) == 1 and r(rank=4) == 1 and t(rank=-1) == 1
    assert r(variant=3, n_vec=4 * (M.LL_CAP_VEC + 1), ll_cap=M.LL_CAP_VEC) == 1
    assert t(variant=3, n_vec=4 * (M.LL_CAP_VEC + 1), ll_cap=M.LL_CAP_VEC) == 1
    assert rs(3, 0, 0, bufs, sigs, None, dst, 64, 0, 4, 0, None, M.LL_CAP_VEC, None) == 1     # LL without an inbox
    assert t(out=None) == 1                                              # all-to-all in place


# ---------------------------------------------------------------------------------------------------------- variant plan
class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda variant, *a: self.calls.append((name, variant, a))


def _planning_world(world):
    from dist_tuto.pth_b200.parallel import symm
    w = object.__new__(symm.SymmWorld)
    w.C, w.world, w.rank, w.ranks = _Recorder(), world, 0, list(range(world))
    w.multicast, w.max_blocks = True, 132
    w.ll_max, w.oneshot_max, w.nvls_min = 32 << 10, 128 << 10, 1
    hd = symm.SymmHandle(w, 1 << 30, 1 << 30, [0x10000 * (r + 1) for r in range(world)], 0x900000, [], 0, "vmm")
    hd.ll = symm.SymmHandle(w, 0, 0, [0x20000 * (r + 1) for r in range(world)], 0, [], 0, "vmm")
    return w, hd


@pytest.mark.parametrize("kind,binding", [("reducescatter", "reduce_scatter"), ("alltoall", "alltoall")])
def test_reduce_scatter_and_alltoall_plan_ll_or_pull(kind, binding, monkeypatch):
    from dist_tuto.pth_b200.parallel.symm import plan_variant
    monkeypatch.delenv("B200DIST_AR_VARIANT", raising=False)
    for world in (2, 4, 8):
        w, hd = _planning_world(world)
        for seg_bytes, want in ((16, 3), (32 << 10, 3), ((32 << 10) + 16, 0), (1 << 20, 0)):
            assert plan_variant(kind, 0, seg_bytes, world, w.ll_max, w.oneshot_max, w.nvls_min, True) == want
            assert w._launch_segments(kind, hd, None, None, seg_bytes // 16, None, None) == want
            assert w.C.calls[-1][:2] == (binding, want)
        for forced, want in (("nvls", 0), ("twoshot", 0), ("oneshot", 0), ("ll", 3)):
            monkeypatch.setenv("B200DIST_AR_VARIANT", forced)
            assert plan_variant(kind, 0, 1 << 20, world, w.ll_max, w.oneshot_max, w.nvls_min, True, forced) == want
            assert w._launch_segments(kind, hd, None, None, 64, None, None) == want
        monkeypatch.setenv("B200DIST_AR_VARIANT", "ll")                  # a segment larger than the inbox: pull
        assert w._launch_segments(kind, hd, None, None, M.LL_CAP_VEC + 1, None, None) == 0
        hd.ll = None                                                     # no inbox: pull
        assert w._launch_segments(kind, hd, None, None, 64, None, None) == 0
        monkeypatch.delenv("B200DIST_AR_VARIANT")
    assert plan_variant(kind, 0, 16, 1, 1 << 20, 1, 1, True) == 0        # world 1


# ---------------------------------------------------------------------------------------------------------- routing
class _StandInWorld:
    """A symmetric world as comm.py sees it: records which method it was asked to run."""

    def __init__(self, world, with_methods=True):
        from dist_tuto.pth_b200.parallel import symm
        self.world, self.calls, self._symm = world, [], symm
        if with_methods:
            self.reduce_scatter_ = lambda out, inp, op: self.calls.append("reduce_scatter_")
            self.all_to_all_ = lambda out, inp: self.calls.append("all_to_all_")
        self.all_gather_ = lambda outs, t: self.calls.append("all_gather_")

    def supports_raw(self, t):
        return True

    def supports_reduction(self, t):
        return t.dtype in self._symm.DTYPE_CODES

    def supports_op(self, op):
        return self._symm.op_code(op) is not None


def _route(monkeypatch, with_methods, call):
    """comm.py with the stand-in world for device tensors ("meta" stands in for CUDA here) and none for CPU tensors."""
    from dist_tuto.pth_b200 import comm
    w = _StandInWorld(4, with_methods)
    torch_calls = []
    monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: w if tensor.device.type == "meta" else None)
    for name in ("reduce_scatter", "reduce_scatter_tensor", "all_to_all_single", "all_gather_into_tensor"):
        monkeypatch.setattr(comm.dist, name, lambda *a, _n=name, **k: torch_calls.append(_n))
    call(comm)
    return w.calls + torch_calls


def test_comm_routes_the_new_calls(monkeypatch):
    """Equal-split device calls of the supported ops and dtypes reach the world's methods (a malformed list too: it raises
    there, on its own rank); AVG, async_op=True, int16, given split sizes, CPU tensors and a world without the methods reach
    torch.distributed."""
    from dist_tuto.pth_b200 import comm
    dev = lambda n, dtype=torch.float32: torch.empty(n, dtype=dtype, device="meta")  # noqa: E731
    # (call, route on a world with the methods, route on one without reduce_scatter_ / all_to_all_)
    cases = [
        (lambda c: c.reduce_scatter_tensor(dev(4), dev(16)), "reduce_scatter_", "reduce_scatter_tensor"),
        (lambda c: c.reduce_scatter_tensor(dev(4, torch.bool), dev(16, torch.bool)), "reduce_scatter_",
         "reduce_scatter_tensor"),
        (lambda c: c.reduce_scatter(dev(4, torch.int64), [dev(4, torch.int64)] * 4, op=comm.reduce_op.MIN),
         "reduce_scatter_", "reduce_scatter"),
        (lambda c: c.reduce_scatter(dev(4), [dev(5)] * 3), "reduce_scatter_", "reduce_scatter"),
        (lambda c: c.all_to_all_single(dev(16, torch.uint8), dev(16, torch.uint8)), "all_to_all_", "all_to_all_single"),
        (lambda c: c.all_gather_into_tensor(dev(16), dev(4)), "all_gather_", "all_gather_"),
        (lambda c: c.reduce_scatter_tensor(dev(4), dev(16), op=torch.distributed.ReduceOp.AVG), "reduce_scatter_tensor",
         "reduce_scatter_tensor"),
        (lambda c: c.reduce_scatter_tensor(dev(4), dev(16), async_op=True), "reduce_scatter_tensor", "reduce_scatter_tensor"),
        (lambda c: c.reduce_scatter_tensor(dev(4, torch.int16), dev(16, torch.int16)), "reduce_scatter_tensor",
         "reduce_scatter_tensor"),
        (lambda c: c.reduce_scatter(torch.zeros(4), [torch.zeros(4)] * 4), "reduce_scatter", "reduce_scatter"),
        (lambda c: c.all_to_all_single(dev(16), dev(16), [4] * 4, [4] * 4), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_to_all_single(dev(16), dev(16), async_op=True), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_to_all_single(torch.zeros(16), torch.zeros(16)), "all_to_all_single", "all_to_all_single"),
        (lambda c: c.all_gather_into_tensor(dev(15), dev(4)), "all_gather_into_tensor", "all_gather_into_tensor"),
        (lambda c: c.all_gather_into_tensor(dev(16), dev(4), async_op=True), "all_gather_into_tensor",
         "all_gather_into_tensor"),
        (lambda c: c.all_gather_into_tensor(torch.zeros(16), torch.zeros(4)), "all_gather_into_tensor",
         "all_gather_into_tensor"),
    ]
    for k, (call, symm_route, plain_route) in enumerate(cases):
        assert _route(monkeypatch, True, call) == [symm_route], k
        assert _route(monkeypatch, False, call) == [plain_route], k


@pytest.mark.timeout(240)
@pytest.mark.parametrize("world", [2, 3])
def test_the_four_calls_on_gloo_give_torchs_results(world):
    import dist_tuto.pth_b200 as b2
    import reduce_scatter_alltoall_workers as W
    b2.launch(W.w_gloo, size=world, backend="gloo", join_timeout_s=200)


def test_the_new_calls_are_exported_from_the_package_root():
    import dist_tuto.pth_b200 as b2
    for name in ("reduce_scatter", "reduce_scatter_tensor", "all_to_all_single", "all_gather_into_tensor"):
        assert callable(getattr(b2, name))
