"""CPU checks of scatter and gather: the models of tests/scatter_gather_model.py against plain torch, planted faults the checker
must catch, the bindings' and the launcher's refusals (no launch), the variant plan of ``SymmWorld`` for the two calls, and
that ``comm.scatter`` / ``comm.gather`` take the same route on the root and on the other ranks."""
import ctypes
import os

import pytest
import torch

import collectives_model as CM
import comm_model as M
import scatter_gather_model as SG

VARIANTS = [M.ONESHOT, M.TWOSHOT, M.LL]


def _zeros(n):
    return torch.zeros(n, dtype=torch.int32)


def _sentinel(n):
    return torch.full((n,), 0x5EADBEEF, dtype=torch.int32)


# ---------------------------------------------------------------------------------------------------------- the models
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", ["inplace", "staged"])
@pytest.mark.parametrize("world,root", [(1, 0), (2, 1), (3, 0), (5, 2), (8, 7)])
def test_gather_model_is_torch_cat_on_the_root_only(variant, mode, world, root):
    seg = 24
    xs = CM.make_raw_inputs(world, seg, seed=world)
    outs = [_sentinel(world * seg + 8) for _ in range(world)]
    bufs = [_sentinel(world * seg + 8) for _ in range(world)]
    g = SG.gather_model(variant, xs, root, mode, outs, bufs)
    for r in range(world):
        if r == root:
            assert torch.equal(g["out"][r][:world * seg], torch.cat(xs))
        elif mode == "staged":
            assert torch.equal(g["out"][r], outs[r])                    # a non-root's output is left alone
        assert torch.equal(g["buf"][r][world * seg:], bufs[r][world * seg:])      # sentinels
        assert torch.equal(g["buf"][r][r * seg:(r + 1) * seg], xs[r]) or (mode == "staged" and variant == M.LL)
        if r != root and (mode == "inplace" or variant != M.LL):      # nothing else lands in a non-root's buffer
            rest = torch.cat([g["buf"][r][:r * seg], g["buf"][r][(r + 1) * seg:]])
            assert bool((rest == 0x5EADBEEF).all())


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", ["inplace", "staged"])
@pytest.mark.parametrize("world,root", [(1, 0), (2, 0), (3, 2), (5, 2), (8, 3)])
def test_scatter_model_is_torch_chunk(variant, mode, world, root):
    seg = 24
    xs = CM.make_raw_inputs(world, seg, seed=10 + world)
    whole = torch.cat(xs)
    outs = [_sentinel(seg + 8) for _ in range(world)]
    bufs = [_sentinel(world * seg + 8) for _ in range(world)]
    s = SG.scatter_model(variant, xs, root, mode, outs, bufs)
    chunks = whole.chunk(world)
    for r in range(world):
        got = s["out"][r][r * seg:(r + 1) * seg] if mode == "inplace" else s["out"][r][:seg]
        assert torch.equal(got, chunks[r])
        if mode == "staged":
            assert torch.equal(s["out"][r][seg:], outs[r][seg:])
        assert torch.equal(s["buf"][r][world * seg:], bufs[r][world * seg:])
    if mode == "staged" and variant == M.LL:
        assert all(torch.equal(b, b0) for b, b0 in zip(s["buf"], bufs))      # LL staged: no symmetric buffer is written


def test_raw_moves_of_scatter_and_gather_keep_every_bit():
    world, seg = 4, 64
    xs = CM.make_raw_inputs(world, seg, seed=4)
    specials = {int(v) & 0xFFFFFFFF for x in xs for v in x.tolist()}
    assert {0x80000000, 0x7FC01234, 0x00000001} <= specials
    for variant in VARIANTS:
        g = SG.gather_model(variant, xs, 1, "staged", [_zeros(world * seg)] * world, [_zeros(world * seg)] * world)
        assert torch.equal(g["out"][1], torch.cat(xs))
        s = SG.scatter_model(variant, xs, 2, "staged", [_zeros(seg)] * world, [_zeros(world * seg)] * world)
        assert all(torch.equal(s["out"][r], xs[r]) for r in range(world))


# ---------------------------------------------------------------------------------------------------------- planted faults
def test_a_non_root_gather_that_writes_its_output_is_caught():
    world, seg, root = 4, 64, 2
    xs = CM.make_raw_inputs(world, seg, seed=5)
    outs = [_sentinel(world * seg) for _ in range(world)]
    bufs = [_sentinel(world * seg) for _ in range(world)]
    want = SG.gather_model(M.ONESHOT, xs, root, "staged", outs, bufs)["out"]
    leaky = CM.allgather_model(M.ONESHOT, xs, "staged", outs, bufs)["out"]     # every rank stores
    m = M.first_mismatch(leaky, want, 4)
    assert m is not None and m[0] == 0 and m[1] == 0


def test_a_scatter_that_delivers_the_wrong_segment_is_caught():
    world, seg, root = 3, 64, 1
    xs = CM.make_raw_inputs(world, seg, seed=6)
    outs = [_sentinel(seg) for _ in range(world)]
    bufs = [_sentinel(world * seg) for _ in range(world)]
    want = SG.scatter_model(M.TWOSHOT, xs, root, "staged", outs, bufs)["out"]
    shifted = [xs[(r + 1) % world] for r in range(world)]                     # rank r receives segment r + 1
    m = M.first_mismatch(shifted, want, 4)
    assert m is not None and m[0] == 0


def test_an_ll_scatter_that_keeps_an_acknowledgement_line_is_caught():
    world, seg, root = 4, 64, 0
    xs = CM.make_raw_inputs(world, seg, seed=7)
    outs = [_sentinel(seg) for _ in range(world)]
    bufs = [_sentinel(world * seg) for _ in range(world)]
    want = SG.scatter_model(M.LL, xs, root, "staged", outs, bufs)["out"]
    wrong = SG.scatter_model(M.LL, xs, root, "staged", outs, bufs, keep=lambda r: 3 if r != 3 else 2)["out"]
    m = M.first_mismatch(wrong, want, 4)
    assert m is not None and m[0] == 0 and m[3] == 0                         # rank 0 kept rank 3's zeros
    assert all(M.first_mismatch([wrong[r]], [want[r]], 4) is not None for r in range(world))


# ---------------------------------------------------------------------------------------------------------- bindings
def _C():
    from dist_tuto.pth_b200.ops import _ext
    if not os.path.isfile(_ext.so_path()):
        pytest.skip("native extension not built")
    return _ext.C()


def _ptrs(world, base):
    return [base * (i + 1) for i in range(world)]


def test_scatter_and_gather_bindings_refuse_bad_roots_sizes_nvls_and_ll_overflow():
    C = _C()
    b, s, ib = _ptrs(4, 0x1000), _ptrs(4, 0x2000), _ptrs(4, 0x3000)
    for name in ("scatter", "gather"):
        f = getattr(C, name)
        with pytest.raises(RuntimeError, match=f"{name}: root must be in"):
            f(0, b, s, None, None, 64, -1, 0, 4)
        with pytest.raises(RuntimeError, match="root must be -1"):
            f(0, b, s, None, None, 64, 4, 0, 4)
        with pytest.raises(RuntimeError, match="multiple of world"):
            f(0, b, s, None, None, 4 * 100 + 1, 0, 0, 4)
        with pytest.raises(RuntimeError, match="NVLS runs the SUM all-reduce only"):
            f(2, b, s, None, None, 64, 0, 0, 4)
        with pytest.raises(RuntimeError, match="more than the inbox holds"):
            f(3, b, s, None, None, 4 * (M.LL_CAP_VEC + 1), 0, 0, 4, 0, ib, M.LL_CAP_VEC)


def _launcher():
    from dist_tuto.pth_b200.ops import _ext
    _C()
    fn = ctypes.CDLL(_ext.so_path()).b2_allreduce_launch
    fn.restype = ctypes.c_int
    i, p, z = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
    fn.argtypes = [i, i, p, p, p, p, i, p, i, z, ctypes.c_float, i, i, i, p, z, i, i, p]
    return fn


def test_launcher_refuses_bad_scatter_and_gather_calls_without_a_launch():
    """b2_allreduce_launch returns cudaErrorInvalidValue (1) before any CUDA call for each of these (on a machine without a
    GPU, a launch would return another error)."""
    fn = _launcher()
    bufs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x1000))
    sigs = (ctypes.c_void_p * 8)(*_ptrs(4, 0x2000))
    inbox = (ctypes.c_void_p * 8)(*_ptrs(4, 0x3000))

    def call(variant, bf16, n_vec, op, root, ll_cap=0):
        return fn(variant, bf16, bufs, sigs, None, None, 0, None, 0, n_vec, 1.0, 0, 4, 0,
                  inbox if variant == 3 else None, ll_cap, op, root, None)
    GATHER, SCATTER = 5, 6
    for op in (GATHER, SCATTER):
        assert call(0, 1, 64, op, 0) == 1                                  # a bf16 wire
        assert call(2, 0, 64, op, 0) == 1                                  # NVLS
        assert call(0, 0, 65, op, 0) == 1                                  # n_vec not a multiple of world
        assert call(3, 0, 4 * (M.LL_CAP_VEC + 1), op, 0, M.LL_CAP_VEC) == 1  # LL segment larger than the inbox
        assert call(0, 0, 64, op, 4) == 1                                  # root out of range
    assert call(0, 0, 64, SCATTER, -1) == 1                                # a scatter needs a root
    assert call(0, 0, 64, 7, 0) == 1                                       # unknown op


# ---------------------------------------------------------------------------------------------------------- variant plan
class _Recorder:
    """Stands in for the extension: records the variant each collective binding is called with."""

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


@pytest.mark.parametrize("collective", ["scatter", "gather"])
def test_scatter_and_gather_are_planned_like_an_all_gather_on_one_segment(collective, monkeypatch):
    from dist_tuto.pth_b200.parallel.symm import plan_variant
    monkeypatch.delenv("B200DIST_AR_VARIANT", raising=False)
    for world in (2, 4, 8):
        w, hd = _planning_world(world)
        for seg_bytes in (16, 32 << 10, (32 << 10) + 16, (128 << 10) // world, (128 << 10) // world + 16, 1 << 20):
            n_vec = seg_bytes // 16 * world
            got = w._launch(hd, False, n_vec, 1.0, None, None, None, None, collective, 0, world - 1)
            assert got == plan_variant("allgather", 0, seg_bytes, world, w.ll_max, w.oneshot_max, w.nvls_min, True)
            assert w.C.calls[-1][:2] == (collective, got)
        for forced, want in (("nvls", 1), ("ll", 3), ("oneshot", 0), ("twoshot", 1)):
            monkeypatch.setenv("B200DIST_AR_VARIANT", forced)
            assert w._launch(hd, False, 64 * world, 1.0, None, None, None, None, collective, 0, 0) == want
        monkeypatch.setenv("B200DIST_AR_VARIANT", "ll")                     # a segment larger than the inbox: one-shot
        assert w._launch(hd, False, (M.LL_CAP_VEC + 1) * world, 1.0, None, None, None, None, collective, 0, 0) == 0
        monkeypatch.delenv("B200DIST_AR_VARIANT")
    assert plan_variant("allgather", 0, 16, 1, 1, 1, 1, True) == 0
    with pytest.raises(ValueError):
        plan_variant("gather", 0, 16, 4, 1, 1, 1, True)                  # not a name of plan_variant's


# ---------------------------------------------------------------------------------------------------------- routing
class _StandInWorld:
    """A symmetric world as comm.py sees it: takes every tensor, records which method it was asked to run."""

    def __init__(self, world, with_methods=True):
        self.world, self.calls = world, []
        if with_methods:
            self.scatter_ = lambda t, lst, root: self.calls.append("scatter_")
            self.gather_ = lambda t, lst, root: self.calls.append("gather_")

    def supports_raw(self, t):
        return True


def _route(monkeypatch, world, rank, with_methods, call):
    from dist_tuto.pth_b200 import comm
    w = _StandInWorld(world, with_methods)
    nccl = []
    monkeypatch.setattr(comm, "_symm_world_for", lambda tensor, group: w)
    monkeypatch.setattr(comm.dist, "get_rank", lambda group=None: rank)
    monkeypatch.setattr(comm.dist, "scatter", lambda *a, **k: nccl.append("scatter"))
    monkeypatch.setattr(comm.dist, "gather", lambda *a, **k: nccl.append("gather"))
    call(comm)
    return w.calls + nccl


@pytest.mark.parametrize("with_methods", [True, False], ids=["symm", "hier"])
def test_comm_routes_scatter_and_gather_alike_on_root_and_peers(monkeypatch, with_methods):
    """The route depends on the tensor and the world only: lists that are missing, short, of another dtype, or separate
    tensors rather than one block give every rank the same route (a world without scatter_ / gather_ keeps NCCL)."""
    world, root = 4, 1
    t = torch.zeros(6, dtype=torch.int64)
    block = torch.zeros(world * 6, dtype=torch.int64)
    lists = [None, [], [torch.zeros(6)] * 2, list(block.view(world, 6).unbind(0)),
             [torch.zeros(6, dtype=torch.int64) for _ in range(world)], [torch.zeros(7, dtype=torch.int8)] * world]
    routes = set()
    for rank in range(world):
        for lst in lists:
            got = _route(monkeypatch, world, rank, with_methods,
                         lambda comm: comm.scatter(t, src=root, scatter_list=lst))
            got += _route(monkeypatch, world, rank, with_methods,
                          lambda comm: comm.gather(t, dst=root, gather_list=lst and [x.clone() for x in lst]))
            routes.add(tuple(got))
    assert routes == ({("scatter_", "gather_")} if with_methods else {("scatter", "gather")})
